"""The superpoint graph of a partition on the device: the third phase of both partition pipelines (ref:
partition/partition.py:184, supervized_partition/supervized_partition.py:346, generate_partition.py:109).

    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph, to_numpy

    graph_sp = compute_sp_graph(xyz, d_max, in_component, components, labels, n_labels)   # graphs.py:75-210
    write_spg(spg_file, to_numpy(graph_sp), components, in_component)                    # provider.py:558

Same name, argument order and dict keys as the reference (is_nn False, sp_*, source, target, se_*); every array
returned is a CUDA tensor: the features float32, source / target [n_sedg, 1], sp_point_count [n_com, 1] and
sp_labels [n_com, n_labels + 1] int64 (sp_labels is [] without labels).  to_numpy gives the reference's numpy dtypes.
The kernels are in csrc/sp_graph.cu.

xyz is float32 [n, 3] and in_component integer [n], numpy arrays or tensors.  in_component is the only source of
membership; `components` is checked only for its length.  The Delaunay triangulation stays on the host: with
simplices=None it is scipy.spatial.Delaunay(xyz).simplices, and a caller can compute it while cut pursuit runs and
pass it as simplices (int [T, 4]).

The centroids, the point counts, the labels, the lengths of components of at most two unique points, the superedge
ids and the ratios are the reference's bit for bit.  The eigenvalues and the offset statistics are computed in fp64
and rounded once.  The superedge keys are exact 64-bit (source, target) pairs, and a cloud of one component has no
superedge (the reference raises IndexError there).  DESIGN.md §4 lists these choices.
"""
import numpy as np
import torch

from . import ops
from ._inputs import check_dtype, check_ints, device_of, n_points, on_device, simplices_on

__all__ = ["compute_sp_graph", "to_numpy"]


def _label_mode(labels, n, n_labels):
    """graphs.py:79-80: 0 (no labels) unless len(labels) > 1; 2 (sum of the label rows) when labels is 2-D with
    more than one column; else 1 (the histogram of the values 0..n_labels)."""
    if len(labels) <= 1:
        return 0
    shape = check_ints(labels, "labels")
    if shape[0] != n:
        raise ValueError("labels has %d rows for %d points" % (shape[0], n))
    if len(shape) > 1 and shape[1] > 1:
        if len(shape) != 2 or shape[1] != n_labels + 1:
            raise ValueError("a label histogram must be [n, n_labels + 1] = [%d, %d] (got shape %s)"
                             % (n, n_labels + 1, shape))
        return 2
    return 1


def compute_sp_graph(xyz, d_max, in_component, components, labels, n_labels, simplices=None):
    """The superpoint graph with its superpoint and superedge features (ref: partition/graphs.py:75-210).

    ValueError: a non-finite coordinate, a negative or empty component id below max + 1, len(components) other than
    max(in_component) + 1, a label histogram without n_labels + 1 columns.  TypeError: xyz not float32, non-integer
    ids, labels or simplices.  IndexError: a simplex id outside [0, n)."""
    n = n_points(np.shape(xyz))
    if n == 0:
        raise ValueError("compute_sp_graph needs at least one point")
    check_dtype(xyz, "xyz", "float32")
    n_labels = int(n_labels)
    shape = check_ints(in_component, "in_component")
    if len(shape) != 1 or shape[0] != n:
        raise ValueError("in_component has shape %s for %d points" % (shape, n))
    label_mode = _label_mode(labels, n, n_labels)
    dev = device_of(xyz, in_component, simplices)
    host_xyz = xyz
    xyz = on_device(xyz, dev)
    comp = on_device(in_component, dev, int64=True)
    lab = None
    if label_mode:
        lab = on_device(labels, dev, int64=True)
        lab = lab.reshape(-1) if label_mode == 1 else lab
    with torch.cuda.device(dev):
        n_com, status = (int(v) for v in ops.sp_scan(xyz, comp).cpu())
        if status & 1:
            raise ValueError("Input contains NaN or infinity.")
        if status & 4:
            raise ValueError("in_component holds a negative id")
        if n_com > n:
            raise ValueError("%d components for %d points: some component holds no point" % (n_com, n))
        if len(components) != n_com:
            raise ValueError("components has %d entries for max(in_component) + 1 = %d" % (len(components), n_com))
        if simplices is None:
            from scipy.spatial import Delaunay  # host triangulation; scipy is imported only when it is needed

            host = host_xyz.cpu().numpy() if torch.is_tensor(host_xyz) else np.asarray(host_xyz)
            simplices = Delaunay(host).simplices
        tets = simplices_on(simplices, dev)
        sp, sp_status = ops.sp_points(xyz, comp, n_com, lab, label_mode, n_labels)
        offsets, e_status = ops.sp_edges_count(comp, tets)
        if int(sp_status.item()) & 8:
            raise ValueError("a component below max(in_component) + 1 holds no point")
        if int(e_status.item()) & 2:
            raise IndexError("simplices hold an id outside [0, %d)" % n)
        n_cand = int(offsets[-1].item())
        ws, n_sedg = ops.sp_edges_build(xyz, comp, tets, offsets, n_cand, d_max)
        se = ops.sp_edges_features(xyz, tets.shape[0], n_cand, ws, int(n_sedg.item()), sp[:5])
    graph = {"is_nn": False, "sp_centroids": sp[0], "sp_length": sp[1], "sp_surface": sp[2], "sp_volume": sp[3],
             "sp_point_count": sp[4], "sp_labels": sp[5] if label_mode else []}
    graph.update(se)
    return graph


_NUMPY_DTYPES = {"source": "uint32", "target": "uint32", "sp_labels": "uint32", "sp_point_count": "uint64"}


def to_numpy(graph_sp):
    """The graph with the reference's numpy dtypes (uint32 ids and labels, uint64 counts, float32 features), as
    provider.write_spg consumes it."""
    out = {}
    for k, v in graph_sp.items():
        if torch.is_tensor(v):
            v = v.cpu().numpy().astype(_NUMPY_DTYPES.get(k, "float32"))
        out[k] = v
    return out
