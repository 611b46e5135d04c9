"""A point cloud's k-nearest-neighbour graphs and geometric features on the device: the first phase of both
partition pipelines (ref: partition/partition.py:146-152, supervized_partition/graph_processing.py:146,176).

    from superpoint_graph_b200.spg_geometry import compute_graph_nn, compute_graph_nn_2, compute_geof

    graph_nn, target_fea = compute_graph_nn_2(xyz, 10, 45)        # partition/graphs.py:26-70
    geof = compute_geof(xyz, target_fea, 45)                       # partition/ply_c/ply_c.cpp:384-462
    geof[:, 3] = 2. * geof[:, 3]                                   # as the callers do

Same names, argument order and return structure as the reference; every array returned is a CUDA tensor:
source / target / target2 int64 (the reference: uint32), distances and geof float32.  xyz is float32 [n, 3], a
numpy array or a tensor.  The kernels are in csrc/geometry.cu.

Neighbours are ranked as the reference's kd-tree ranks them: by d2 = (dx dx + dy dy) + dz dz in float64 from the
float32 coordinates, then by the smaller index, the vertex itself excluded (sklearn returns it first and the
reference drops that column), so the distances are the reference's bit for bit and the ids are its ids wherever the
distances are untied.  With duplicate points the reference may list the vertex itself and drop a duplicate; here a
vertex never appears in its own list.  compute_geof solves the covariance's eigenproblem in fp64 (the reference: a
general float32 EigenSolver, whose bits cannot be reproduced); where the largest eigenvalue is 0 (k + 1 coincident
points) all four features are NaN, as the reference's 0 / 0.  DESIGN.md §4 lists these choices.
"""
import math

import numpy as np
import torch

from . import ops
from ._inputs import check_dtype, check_ints, device_of, n_points, on_device

__all__ = ["compute_graph_nn", "compute_graph_nn_2", "compute_geof"]

_GRID_DIM = 2 ** 21 - 1  # cells per axis (21 bits of the 63-bit cell key)


def _check_k(k, n, what):
    if isinstance(k, bool) or int(k) != k or k < 1:
        raise ValueError("%s must be a positive integer (got %r)" % (what, k))
    k = int(k)
    cap = ops.knn_max_k()
    if k > cap:
        raise ValueError("%s = %d is above the k-NN kernel's cap of %d neighbours" % (what, k, cap))
    if n < k + 1:  # sklearn's message for n_neighbors = k + 1
        raise ValueError("Expected n_neighbors <= n_samples_fit, but n_neighbors = %d, n_samples_fit = %d, "
                         "n_samples = %d" % (k + 1, n, n))
    return k


def _decode(words):
    """Floats from the order-preserving uint32 keys of spg_knn_bounds."""
    w = np.asarray(words, dtype=np.int64) & 0xFFFFFFFF
    bits = np.where(w & 0x80000000, w & 0x7FFFFFFF, ~w & 0xFFFFFFFF).astype(np.uint32)
    return bits.view(np.float32).astype(np.float64)


def _grid(lo, hi, cell):
    ext = hi - lo
    cell = max(cell, float(ext.max()) / (_GRID_DIM - 1), 1e-30)
    dims = [int(math.floor(e / cell)) + 1 for e in ext]
    while max(dims) > _GRID_DIM:  # rounding at the edge
        cell *= 1.0 + 1e-9
        dims = [int(math.floor(e / cell)) + 1 for e in ext]
    return (float(lo[0]), float(lo[1]), float(lo[2]), float(cell), dims[0], dims[1], dims[2])


def build_grid(xyz, k):
    """The sorted cloud and its cell table for k-neighbour queries: (grid, workspace), grid = (ox, oy, oz, cell,
    dim_x, dim_y, dim_z).  ValueError for a non-finite coordinate (the one read-back of the status word).

    The cell size sets only the work of the query.  Aim: about max(4, (k + 1) / 2) points per occupied cell, so that
    the query's first ring of cells usually holds its k neighbours.  The first guess spreads the points over the
    box's volume.  Real scans are surfaces, and a few stray points can inflate the box by orders of magnitude, so the
    grid is rebuilt from the measured occupancy (one 4-byte read-back each, at most four builds): the cell size is
    scaled by (target / occupancy)^(1 / D), with D = 2 at first and then the dimension two measurements imply,
    kept within [2, 3] so that a step never shrinks the cells further than a surface or a volume would need.  The
    grid whose occupancy came closest to the aim is the one kept."""
    n = xyz.shape[0]
    words = ops.knn_bounds(xyz).cpu().numpy()
    if words[6] & 1:
        raise ValueError("Input contains NaN or infinity.")
    lo, hi = _decode(words[0:3]), _decode(words[3:6])
    target = max(4.0, (k + 1) / 2.0)
    ext = hi - lo
    pos = ext[ext > 0]
    cell = (float(np.prod(pos)) * target / n) ** (1.0 / pos.size) if pos.size else 1.0
    ws = ops.knn_workspace(n, xyz.device)
    tried = []  # (|log(occupancy / target)|, grid, occupied cells)
    for attempt in range(4):
        grid = _grid(lo, hi, cell)
        cells = int(ops.knn_grid(xyz, grid, ws).item())
        occ = n / cells
        tried.append((abs(math.log(occ / target)), grid, cells))
        if target / 2 <= occ <= 2 * target or attempt == 3:
            break
        dim = 2.0
        if len(tried) > 1 and tried[-2][2] != cells and tried[-2][1][3] != grid[3]:
            dim = math.log(cells / tried[-2][2]) / math.log(tried[-2][1][3] / grid[3])
            dim = min(max(dim, 2.0), 3.0)
        cell = grid[3] * (target / occ) ** (1.0 / dim)
    best = min(tried, key=lambda t: t[0])
    if best[1] != grid:
        grid = best[1]
        ops.knn_grid(xyz, grid, ws)
    return grid, ws


def _knn(xyz, k, k1, want_target2):
    grid, ws = build_grid(xyz, k)
    return ops.knn_query(xyz.shape[0], k, k1, grid, ws, want_target2)


def compute_graph_nn(xyz, k_nn):
    """The k-NN graph (ref: partition/graphs.py:11-24): dict is_nn=True, source = repeat(arange(n), k_nn),
    target (int64 [n k_nn], row-major) and distances (float32 [n k_nn])."""
    n = n_points(np.shape(xyz))
    k_nn = _check_k(k_nn, n, "k_nn")
    check_dtype(xyz, "xyz", "float32")
    dev = device_of(xyz)
    xyz = on_device(xyz, dev)
    with torch.cuda.device(dev):
        source, target, distances, _ = _knn(xyz, k_nn, k_nn, False)
    return {"is_nn": True, "source": source, "target": target, "distances": distances}


def compute_graph_nn_2(xyz, k_nn1, k_nn2, voronoi=0.0):
    """The k_nn1 graph and the k_nn2 neighbour list from one query (ref: partition/graphs.py:26-70):
    (graph, target2) with graph as compute_graph_nn's for the first k_nn1 neighbours and target2 int64 [n k_nn2].
    The Delaunay edges of voronoi > 0 are spg_structure.compute_graph_nn_2's."""
    assert k_nn1 <= k_nn2, "knn1 must be smaller than knn2"
    if voronoi > 0:
        raise NotImplementedError("voronoi > 0 (Delaunay edges) is not computed here; use "
                                  "spg_structure.compute_graph_nn_2")
    n = n_points(np.shape(xyz))
    k_nn1 = _check_k(k_nn1, n, "k_nn1")
    k_nn2 = _check_k(k_nn2, n, "k_nn2")
    check_dtype(xyz, "xyz", "float32")
    dev = device_of(xyz)
    xyz = on_device(xyz, dev)
    with torch.cuda.device(dev):
        source, target, distances, target2 = _knn(xyz, k_nn2, k_nn1, True)
    return {"is_nn": True, "source": source, "target": target, "distances": distances}, target2


def compute_geof(xyz, target, k_nn):
    """Linearity, planarity, scattering and verticality of every vertex and its k_nn neighbours
    target[k_nn i : k_nn i + k_nn] (ref: partition/ply_c/ply_c.cpp:384-462), float32 [n, 4], unscaled (the callers
    double column 3).  IndexError for an id outside [0, n) (one read-back), ValueError for a short target."""
    n = n_points(np.shape(xyz))
    if isinstance(k_nn, bool) or int(k_nn) != k_nn or k_nn < 1:
        raise ValueError("k_nn must be a positive integer (got %r)" % (k_nn,))
    k_nn = int(k_nn)
    n_ids = math.prod(check_ints(target, "target"))
    if n_ids < n * k_nn:
        raise ValueError("target has %d ids for %d vertices of %d neighbours" % (n_ids, n, k_nn))
    check_dtype(xyz, "xyz", "float32")
    dev = device_of(xyz, target)
    t = target.reshape(-1) if torch.is_tensor(target) else np.asarray(target).reshape(-1)
    t = on_device(t[:n * k_nn], dev, int64=True)
    xyz = on_device(xyz, dev)
    with torch.cuda.device(dev):
        out, status = ops.geof(xyz, t, k_nn)
        if int(status.item()) & 2:
            raise IndexError("target holds an id outside [0, %d)" % n)
    return out
