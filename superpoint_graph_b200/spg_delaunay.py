"""The exact 3D Delaunay triangulation of a point cloud on the device: the simplices compute_sp_graph needs (ref:
partition/graphs.py:82, scipy.spatial.Delaunay(xyz).simplices).

    from superpoint_graph_b200.spg_delaunay import delaunay
    simplices = delaunay(xyz)                                            # int32 CUDA tensor [T, 4]
    graph_sp = compute_sp_graph(xyz, d_max, in_component, components, labels, n_labels, simplices=simplices)

xyz is float32 [n, 3], a numpy array or a tensor.  The output is the Delaunay triangulation of the unique points:
every tetrahedron has exact positive orientation, the tetrahedra tile the convex hull, and no point is strictly
inside a tetrahedron's circumsphere.  Of a group of exact duplicates (-0 equal to +0) only the smallest index appears.
Cospherical and coplanar points are resolved by a symbolic perturbation (Devillers and Teillaud's, as CGAL implements
it), so the triangulation is unique.  Each row is rotated by an even permutation to (smallest id, second smallest,
...) and the rows are sorted, so two runs give identical tensors and the output compares with oracle/delaunay_ref.py
as arrays.  DESIGN.md §4 states these conventions; the kernels are in csrc/delaunay.cu.
"""
import numpy as np
import torch

from . import ops
from ._inputs import check_dtype, device_of, n_points, on_device

__all__ = ["delaunay", "to_numpy", "last_stats"]

_STATS = {}
_MAX_CAP = 2 ** 29  # tetrahedra in the store: csrc/delaunay.cu packs tet * 4 + face into int32


def last_stats():
    """Counters of the last delaunay() call: rounds, tetrahedra, largest cavity, store capacity, growths."""
    return dict(_STATS)


def _initial_cap(u):
    return min(max(64, 7 * u + 64), _MAX_CAP)


def delaunay(xyz, capacity=None):
    """The Delaunay triangulation of xyz's unique points, int32 [T, 4] on the device (see the module docstring).

    ValueError: a non-finite coordinate, fewer than 4 affinely independent unique points, n >= 2^31 - 1, a shape
    other than [n, 3], a triangulation of more than 2^29 tetrahedra (the store's limit; about 7.7 10^7 points in
    general position), a capacity outside [8, 2^29].  TypeError: xyz not float32.  capacity: the initial store of tetrahedra (it grows as needed)."""
    n = n_points(check_dtype(xyz, "xyz", "float32"))
    if torch.is_tensor(xyz):
        ops._need_cuda(xyz)
    if n < 4:
        raise ValueError("fewer than 4 affinely independent points (%d points)" % n)
    cap = int(capacity) if capacity is not None else _initial_cap(n)
    if not 8 <= cap <= _MAX_CAP:
        raise ValueError("capacity must be in [8, 2^29] (got %d)" % cap)
    dev = device_of(xyz)
    with torch.cuda.device(dev):
        x = on_device(xyz, dev)
        store = ops.DelaunayStore(n, cap, dev)
        status, unique = store.setup(x)
        if status & 1:
            raise ValueError("Input contains NaN or infinity.")
        if unique < 4:
            raise ValueError("fewer than 4 affinely independent points (%d unique)" % unique)
        status = store.init()
        if status & 2:
            raise ValueError("fewer than 4 affinely independent points")
        if status:
            raise RuntimeError("delaunay: point location did not end (status %d)" % status)
        rounds = grows = 0
        big = -1
        max_cav = 0
        while True:
            nom, win, new, over, min_over, free, top, max_cav = store.cavities(big)
            if nom == 0:
                break
            if win == 0:
                if over == 0 or big >= 0:
                    raise RuntimeError("delaunay: a round inserted no point")
                big = min_over
                continue
            short, status = store.commit()
            if short:
                if top + new > _MAX_CAP:
                    raise ValueError("the triangulation needs more than 2^29 tetrahedra, the store's limit")
                store.grow(min(max(2 * store.cap, top + new + 64), _MAX_CAP))
                grows += 1
                continue
            if status:
                raise RuntimeError("delaunay: inconsistent triangulation (status %d)" % status)
            rounds += 1
            big = -1
            if rounds > 4 * n + 16:
                raise RuntimeError("delaunay: too many rounds")
        simplices = store.output()
    _STATS.clear()
    _STATS.update(rounds=rounds, tetrahedra=int(simplices.shape[0]), max_cavity=max_cav, capacity=store.cap,
                  grows=grows, unique=unique)
    return simplices


def to_numpy(simplices):
    """The simplices as int64 numpy."""
    return simplices.cpu().numpy().astype(np.int64)
