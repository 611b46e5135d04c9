"""Voxel pruning of a point cloud on the device: the step before the first phase of both partition pipelines (ref:
partition/ply_c/ply_c.cpp:149-380 `prune`, called at partition/partition.py:124 and
supervized_partition/graph_processing.py:124,142).

    from superpoint_graph_b200.spg_prune import prune, to_numpy

    xyz, rgb, labels, objects = prune(xyz, voxel_width, rgb, labels, objects, n_labels, n_objects)
    xyz, rgb, labels, objects = to_numpy((xyz, rgb, labels, objects))      # the reference's dtypes, if wanted

Same name, argument order and return tuple as the reference; every array returned is a CUDA tensor: xyz float32
[m, 3], rgb uint8 [m, 3], labels int64 [m, n_labels + 1] and objects int64 [m, n_objects + 1] (the reference: uint32).
to_numpy gives the reference's numpy dtypes.  The kernels are in csrc/prune.cu.

Row i is the i-th voxel touched in point order (the reference's insertion order).  A voxel's position is the fp32 sum
of its points in point order divided by float(count), its colour the uint32 channel sums over float(count) truncated
to uint8, its labels and objects the histograms of the values: every output is the reference's bit for bit.  Labels
are counted when n_labels > 0, objects only when n_labels > 0 and n_objects > 0, as ply_c.cpp:343-354 does.

chunk_rows > 0 prunes every chunk of chunk_rows consecutive points on its own and stacks the results in chunk order,
which is what partition/provider.py:250-303 (`read_semantic3d_format`) computes with ver_batch = chunk_rows.

xyz is float32 [n, 3] and rgb uint8 [n, 3]; labels and objects hold integers, [n] (or [n, 1]); numpy arrays or
tensors.  The reference reinterprets the memory of other dtypes; here they are refused (TypeError).  Its undefined
behaviour raises ValueError: an empty cloud, a non-finite coordinate, voxel_size <= 0 or a bin of 2^32 or more.  A
label above n_labels or an object above n_objects raises IndexError, as the reference's .at() does.  DESIGN.md §4 lists
these choices.
"""
import numpy as np
import torch

from . import ops
from ._inputs import check_dtype, check_ints, device_of, n_points, on_device

__all__ = ["prune", "to_numpy"]

_MAX_COLS = 2 ** 31 - 2
_MAX_CHUNKS = 65535  # one grid row of the bounds pass per chunk


def _count(v, name):
    if isinstance(v, bool) or int(v) != v or not 0 <= v <= _MAX_COLS:
        raise ValueError("%s must be an integer in [0, %d] (got %r)" % (name, _MAX_COLS, v))
    return int(v)


def _check_ids(a, name, n):
    """A label or object array read by the reference: integers, one per point."""
    shape = check_ints(a, name)
    if len(shape) == 0 or shape[0] != n or int(np.prod(shape)) != n:
        raise ValueError("%s has shape %s for %d points" % (name, tuple(shape), n))


def prune(xyz, voxel_size, rgb, labels, objects, n_labels, n_objects, chunk_rows=0):
    """The cloud pruned on a regular voxel grid of side voxel_size (ref: partition/ply_c/ply_c.cpp:288-380); with
    chunk_rows > 0, every chunk of chunk_rows points pruned on its own and the results stacked (ref:
    partition/provider.py:265-297).

    ValueError: an empty cloud, a non-finite coordinate, voxel_size not finite and > 0, a bin of 2^32 or more,
    negative n_labels / n_objects / chunk_rows, row-count mismatches of the arrays read.  TypeError: xyz not float32,
    rgb not uint8, non-integer labels or objects.  IndexError: a label outside [0, n_labels] or an object outside
    [0, n_objects]."""
    n = n_points(np.shape(xyz))
    if n == 0:
        raise ValueError("prune needs at least one point")
    check_dtype(xyz, "xyz", "float32")
    n_labels = _count(n_labels, "n_labels")
    n_objects = _count(n_objects, "n_objects")
    chunk_rows = _count(chunk_rows, "chunk_rows")
    if chunk_rows and -(-n // chunk_rows) > _MAX_CHUNKS:
        raise ValueError("%d chunks of %d rows; at most %d chunks are supported" % (-(-n // chunk_rows), chunk_rows,
                                                                                     _MAX_CHUNKS))
    voxel = np.float32(voxel_size)  # the reference's C++ float
    if not (np.isfinite(voxel) and voxel > 0):
        raise ValueError("voxel_size must be finite and > 0 (got %r)" % (voxel_size,))
    with_labels = n_labels > 0
    with_objects = with_labels and n_objects > 0
    rgb_shape = check_dtype(rgb, "rgb", "uint8")
    if rgb_shape != (n, 3):
        raise ValueError("rgb has shape %s for %d points (want [n, 3])" % (rgb_shape, n))
    if with_labels:
        _check_ids(labels, "labels", n)
    if with_objects:
        _check_ids(objects, "objects", n)
    dev = device_of(xyz, rgb, labels, objects)
    xyz = on_device(xyz, dev)
    rgb = on_device(rgb, dev)
    lab = on_device(labels, dev, int64=True).reshape(-1) if with_labels else None
    obj = on_device(objects, dev, int64=True).reshape(-1) if with_objects else None
    with torch.cuda.device(dev):
        ws = ops.prune_workspace(n, chunk_rows, dev)
        words = [int(v) for v in ops.prune_bounds(xyz, chunk_rows, voxel, lab, n_labels, obj, n_objects, ws).cpu()]
        status = words[0]
        if status & 1:
            raise ValueError("Input contains NaN or infinity.")
        if status & 2:
            raise ValueError("a voxel bin of 2^32 or more: voxel_size %r is too small for the cloud's extent"
                             % float(voxel))
        if status & 4:
            raise IndexError("labels hold a value outside [0, n_labels = %d]" % n_labels)
        if status & 8:
            raise IndexError("objects hold a value outside [0, n_objects = %d]" % n_objects)
        m = int(ops.prune_voxels(xyz, chunk_rows, voxel, words[1:], ws).item())
        return ops.prune_reduce(xyz, rgb, lab, n_labels, obj, n_objects, chunk_rows, ws, m)


_NUMPY_DTYPES = ("float32", "uint8", "uint32", "uint32")


def to_numpy(pruned):
    """The pruned cloud with the reference's numpy dtypes (float32 xyz, uint8 rgb, uint32 histograms)."""
    return tuple(t.cpu().numpy().astype(d) for t, d in zip(pruned, _NUMPY_DTYPES))
