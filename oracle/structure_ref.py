"""numpy restatement of the learned partition's graph structure (ref: partition/graphs.py:42-64 on given simplices,
supervized_partition/graph_processing.py:124-126,144-190): the oracle of superpoint_graph_b200.spg_structure.

The k-NN lists are inputs (`neighbors` [n, k_nn2], each vertex's neighbours nearest first, the vertex itself
excluded), as are the simplices, so the oracle can be fed the reference's captured arrays or the device's own."""
import numpy as np

from .partition_ref import connected_comp as _cc_scipy

_PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def voronoi_graph(xyz, simplices, neighbors, k_nn1, voronoi):
    """graphs.py:42-64: (source, target int64 sorted by (target, source), distances float32 of the kept
    candidates in candidate order)."""
    xyz = np.asarray(xyz, dtype=np.float32)
    simp = np.asarray(simplices).astype(np.int64)
    n = xyz.shape[0]
    src = np.concatenate([simp[:, a] for a, _ in _PAIRS])
    tgt = np.concatenate([simp[:, b] for _, b in _PAIRS])
    d = xyz[src] - xyz[tgt]                                  # float32, each op rounded
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = d2 < np.float32(voronoi)
    src = np.concatenate([src[keep], np.repeat(np.arange(n, dtype=np.int64), k_nn1)])
    tgt = np.concatenate([tgt[keep], np.asarray(neighbors)[:, :k_nn1].reshape(-1).astype(np.int64)])
    _, first = np.unique(src + n * tgt, return_index=True)
    return src[first], tgt[first], d2[keep]


def connected_comp(n_ver, source, target, active):
    """libply_c.connected_comp with cutoff 0, the mask byte read as a signed char: (list of member arrays,
    in_component)."""
    act = np.ascontiguousarray(np.asarray(active).reshape(-1)).astype(np.uint8).view(np.int8)
    return _cc_scipy(n_ver, np.asarray(source), np.asarray(target), act, 0)


def inpainting_problem(labels, source, target):
    """graph_processing.py:152-162: (hard_labels, edg_source, edg_target, edge_weight, node_weight), with :155's
    operator precedence."""
    labels = np.asarray(labels)
    hard = np.argmax(labels[:, 1:], 1) + 1
    no_labels = (labels[:, 1:].sum(1) == 0).nonzero()
    hard[no_labels] = 0
    hs, ht = hard[source], hard[target]
    is_tr = hs != ht * (hs != 0) * (ht != 0)
    keep = (is_tr == 0).nonzero()
    node_weight = np.ones((len(hard),), dtype="f4")
    node_weight[no_labels] = 0
    return (hard.astype(np.int64), np.asarray(source)[keep].astype(np.int64),
            np.asarray(target)[keep].astype(np.int64), np.ones(len(keep[0]), dtype="f4"), node_weight)


def plane_elevation(xyz, coef, intercept):
    """float32(z - (x c0 + y c1 + b)) in float64."""
    x = np.asarray(xyz, dtype=np.float64)
    return (x[:, 2] - ((x[:, 0] * coef[0] + x[:, 1] * coef[1]) + intercept)).astype(np.float32)


def structure(dataset, xyz, labels, objects, neighbors, k_nn_adj, k_nn_local, voronoi=0.0, simplices=None,
              pruned=True, plane=None):
    """graph_processing.py:124-126,144-190 with compute_geof = 0: dict of source, target, distances,
    target_local_geometry, is_transition, labels, objects, elevation, xyn.  plane: (coef, intercept) of the RANSAC
    fit, or None for z - min z."""
    xyz = np.asarray(xyz, dtype=np.float32)
    n = xyz.shape[0]
    nb = np.asarray(neighbors).astype(np.int64)
    if voronoi > 0:
        src, tgt, dist = voronoi_graph(xyz, simplices, nb, k_nn_adj, voronoi)
    else:
        src = np.repeat(np.arange(n, dtype=np.int64), k_nn_adj)
        tgt = nb[:, :k_nn_adj].reshape(-1)
        dist = None
    if dataset == "s3dis":
        if pruned:
            objects = np.asarray(objects)[:, 1:].argmax(axis=1) + 1
        objects = np.asarray(objects).reshape(-1)
        is_tr = objects[src] != objects[tgt]
    elif dataset == "vkitti":
        hard = np.argmax(labels, 1)
        is_tr = hard[src] != hard[tgt]
        objects = connected_comp(n, src, tgt, (is_tr == 0).astype("uint8"))[1]
    elif dataset == "sema3d" and labels is None:
        labels, objects, is_tr = np.array([0]), np.array([0]), np.array(False)
    else:
        objects = np.asarray(objects).reshape(-1)
        is_tr = objects[src] != objects[tgt]
    if plane is None:
        elevation = xyz[:, 2] - xyz[:, 2].min()
    else:
        elevation = plane_elevation(xyz, *plane)
    ma, mi = np.max(xyz[:, :2], axis=0, keepdims=True), np.min(xyz[:, :2], axis=0, keepdims=True)
    xyn = (xyz[:, :2] - mi) / (ma - mi + np.float32(1e-8))
    return dict(source=src, target=tgt, distances=dist, target_local_geometry=nb[:, :k_nn_local],
                is_transition=np.asarray(is_tr), labels=np.asarray(labels), objects=np.asarray(objects),
                elevation=elevation.astype(np.float32), xyn=xyn.astype(np.float32))


def low_points(xyz):
    """graph_processing.py:182: the ids with z - min z < 0.5 in float32."""
    xyz = np.asarray(xyz, dtype=np.float32)
    return ((xyz[:, 2] - xyz[:, 2].min()) < 0.5).nonzero()[0]
