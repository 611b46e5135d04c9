"""The learned partition's graph structure on the device: the Voronoi adjacency, label transitions and label-constant
objects of graph_processing (ref: supervized_partition/graph_processing.py:124-126,144-193), the step between a
pruned cloud and read_structure -> PartitionStore.add -> load_batch.

    from superpoint_graph_b200.spg_structure import compute_structure, as_read_structure

    structure = compute_structure(args, "vkitti", xyz, rgb, labels)       # dict of write_structure's arguments
    store.add(name, *as_read_structure(structure, args.learned_embeddings_geof))

    graph_nn, target2 = compute_graph_nn_2(xyz, 5, 20, voronoi=0.3)      # partition/graphs.py:26-70
    components, in_component = connected_comp(n, source, target, active, 0)   # libply_c.connected_comp

Every array returned is a CUDA tensor; to_numpy gives write_structure's dtypes.  The kernels are in
csrc/structure.cu; the k-NN and geometric features are spg_geometry's, the triangulation spg_delaunay's.

compute_graph_nn_2(voronoi > 0) mirrors graphs.py:42-64.  The 6 T directed candidates (v0,v1), (v0,v2), (v0,v3),
(v1,v2), (v1,v3), (v2,v3) of every simplex come in column-block order, each in the orientation its row gives.  A
candidate is kept when d2 = (dx dx + dy dy) + dz dz in float32 is < float32(voronoi) (numpy 2 casts the Python float
to float32 before comparing).  graph["distances"] is d2 of the kept candidates, squared, in candidate order and not
deduplicated, so its length differs from that of source: the reference's quirk, kept.  The kept candidates and the
n k_nn1 k-NN edges are deduplicated as np.unique(source + n target) does, so the edges are sorted by (target,
source).  Given scipy's simplices the output is the reference's bit for bit; given the device's canonical rows it is
the same formula applied to those rows.  DESIGN.md §4 lists these choices.
"""
import numpy as np
import torch

from . import ops, spg_delaunay, spg_geometry
from ._inputs import check_dtype, check_ints, device_of, n_points, on_device, simplices_on
from .spg_cut_pursuit import Components, cutpursuit2

__all__ = ["compute_graph_nn_2", "connected_comp", "compute_structure", "inpainting_problem", "to_numpy",
           "as_read_structure"]

_DATASETS = ("s3dis", "sema3d", "vkitti")


def _raise_ids(status, what):
    if int(status.item()) & 2:
        raise IndexError("%s holds an id outside [0, n)" % what)


def compute_graph_nn_2(xyz, k_nn1, k_nn2, voronoi=0.0, simplices=None):
    """(graph, target2) of graphs.py:26-70.  voronoi == 0: spg_geometry.compute_graph_nn_2.  voronoi > 0: the
    Delaunay edges of `simplices` (int [T, 4], numpy or CUDA; spg_delaunay.delaunay(xyz) when None) with
    d2 < float32(voronoi), joined with the k_nn1 graph and deduplicated (see the module docstring): source, target
    int64 sorted by (target, source), distances float32 = d2 of the kept candidates, target2 int64 [n k_nn2].
    IndexError for a simplex id outside [0, n)."""
    if not voronoi > 0:
        return spg_geometry.compute_graph_nn_2(xyz, k_nn1, k_nn2, voronoi)
    graph, target2 = spg_geometry.compute_graph_nn_2(xyz, k_nn1, k_nn2)  # validates xyz, k_nn1 <= k_nn2
    k_nn1 = int(k_nn1)
    dev = graph["target"].device
    vor = float(np.float32(voronoi))
    with torch.cuda.device(dev):
        x = on_device(xyz, dev)
        if simplices is None:
            simplices = spg_delaunay.delaunay(x)
        simp = simplices_on(simplices, dev)
        counts, status = ops.st_vor_count(x, simp, vor)
        _raise_ids(status, "simplices")
        n_kept = int(counts[-1].item())
        distances, source, target, n_edges, status = ops.st_vor_build(x, simp, vor, counts, graph["target"], k_nn1,
                                                                      n_kept)
        m = int(n_edges.item())
    return {"is_nn": True, "source": source[:m], "target": target[:m], "distances": distances}, target2


def _edge_ids(a, name, dev):
    if len(check_ints(a, name)) != 1:
        raise ValueError("%s must be 1-D" % name)
    return on_device(a, dev, int64=True)


def connected_comp(n_ver, source, target, active_edg, cutoff=0):
    """libply_c.connected_comp (ref: partition/ply_c/connected_components.cpp:17-110, ply_c.cpp:465-478):
    (components, in_component) of the graph of the edges whose active_edg byte, read as a signed char as on x86-64,
    is > 0 (so bytes 128-255 are inactive).  components is a Components CSR (members ascending, as boost pushes
    them), in_component int64, components numbered by their smallest vertex (boost's numbering).

    active_edg: uint8, int8 or bool [E]; source, target: integers [E] in [0, n_ver) (IndexError otherwise).
    cutoff > 0 raises NotImplementedError: its fusion pass is sequential and order-dependent, it never fuses into
    component 0 (largest_neigh_comp_index > 0), and no reference caller passes it (graph_processing.py:171,
    losses.py:134)."""
    if isinstance(n_ver, bool) or int(n_ver) != n_ver or not 1 <= n_ver < 2 ** 31 - 1:
        raise ValueError("n_ver must be an integer in [1, 2^31 - 1) (got %r)" % (n_ver,))
    if int(cutoff) != cutoff or cutoff < 0:
        raise ValueError("cutoff must be a non-negative integer (got %r)" % (cutoff,))
    if cutoff > 0:
        raise NotImplementedError("connected_comp with cutoff > 0 is not computed on the device")
    n_ver = int(n_ver)
    dt = active_edg.dtype if torch.is_tensor(active_edg) else np.asarray(active_edg).dtype
    if dt not in (torch.uint8, torch.int8, torch.bool, np.uint8, np.int8, np.bool_):
        raise TypeError("active_edg must be uint8, int8 or bool (got %s)" % dt)
    dev = device_of(source, target, active_edg)
    with torch.cuda.device(dev):
        src = _edge_ids(source, "source", dev)
        tgt = _edge_ids(target, "target", dev)
        if torch.is_tensor(active_edg):
            act = active_edg.reshape(-1).to(dev).contiguous()
            act = act.view(torch.uint8) if act.dtype == torch.int8 else act.to(torch.uint8)
        else:
            a = np.ascontiguousarray(np.asarray(active_edg).reshape(-1))
            act = torch.from_numpy(a.view(np.uint8) if a.dtype != np.bool_ else a.astype(np.uint8)).to(dev)
        if not src.shape[0] == tgt.shape[0] == act.shape[0]:
            raise ValueError("source, target and active_edg have %d, %d and %d entries"
                             % (src.shape[0], tgt.shape[0], act.shape[0]))
        in_comp, offsets, members, n_comp, status = ops.st_cc(src, tgt, act, n_ver)
        _raise_ids(status, "source or target")
        c = int(n_comp.item())
    return Components(offsets[:c + 1], members), in_comp


def _field(args, name):
    if not hasattr(args, name):
        raise ValueError("args has no field %r" % name)
    return getattr(args, name)


def _histogram(a, name, n, dev):
    shape = check_ints(a, name)
    if len(shape) != 2 or shape[0] != n or shape[1] < 1:
        raise ValueError("%s must be a [%d, C] histogram (got shape %s)" % (name, n, tuple(shape)))
    return on_device(a, dev, int64=True)


def _per_vertex(a, name, n, dev):
    shape = check_ints(a, name)
    if tuple(shape) not in ((n,), (n, 1)):
        raise ValueError("%s must hold one integer per vertex (got shape %s)" % (name, tuple(shape)))
    return on_device(a, dev, int64=True).reshape(-1)


def _transitions(lab, graph_nn, mode=ops.ST_DIFFERENT):
    tr, status = ops.st_transitions(lab, graph_nn["source"], graph_nn["target"], mode)
    _raise_ids(status, "the graph")
    return tr


def inpainting_problem(labels, graph_nn):
    """The node-weighted problem graph_processing.py:152-162 hands to libcp.cutpursuit2 for sema3d
    (spg_cut_pursuit.cutpursuit2 solves it): (hard_labels int64 [n], edg_source, edg_target int64 (the
    non-transition edges, in edge order), edge_weight float32 ones, node_weight float32 (0 where the label row
    labels[:, 1:] is empty, else 1)).  The transitions keep :155's operator precedence,
    hard[s] != (hard[t] * (hard[s] != 0) * (hard[t] != 0))."""
    src = graph_nn["source"]
    dev = src.device
    with torch.cuda.device(dev):
        check_ints(labels, "labels")
        lab = on_device(labels, dev, int64=True)
        if lab.dim() != 2 or lab.shape[1] < 2:
            raise ValueError("labels must be a [n, C] histogram with C >= 2 (got shape %s)" % (tuple(lab.shape),))
        hard, node_weight = ops.st_argmax(lab, 1, 1, zero_empty=True, want_weight=True)
        is_tr = _transitions(hard, graph_nn, ops.ST_INPAINT)
        index, count = ops.st_select(is_tr, False) if is_tr.numel() else (None, torch.zeros(1, dtype=torch.int64))
        m = int(count.item())
        if m:
            s = ops.st_gather_rows(src, index, m)[0]
            t = ops.st_gather_rows(graph_nn["target"], index, m)[0]
        else:
            s = t = torch.empty(0, dtype=torch.int64, device=dev)
        edge_weight = torch.ones(m, dtype=torch.float32, device=dev)
    return hard, s, t, edge_weight, node_weight


def _plane(xyz, bounds, low):
    """The RANSAC plane of the low points (graph_processing.py:182-183): (coef_x, coef_y, intercept) as floats.  The
    low points are compacted on the device; the fit is sklearn's, on the host."""
    from sklearn.linear_model import RANSACRegressor  # imported only when a plane model is asked for

    index, count = ops.st_select(low, True)
    pts, _ = ops.st_gather_rows(xyz, index, int(count.item()))
    pts = pts.cpu().numpy()
    reg = RANSACRegressor(random_state=0).fit(pts[:, :2], pts[:, 2])
    coef = np.asarray(reg.estimator_.coef_, dtype=np.float64).reshape(-1)
    return float(coef[0]), float(coef[1]), float(np.float64(reg.estimator_.intercept_))


def compute_structure(args, dataset, xyz, rgb, labels, objects=None, pruned=True, simplices=None, inpaint=False,
                      seed=0):
    """graph_processing.py:124-126 and :144-193 on the device: a dict of write_structure's arguments, xyz, rgb,
    graph_nn, target_local_geometry (int64 [n, k_nn_local]), is_transition (uint8), labels, objects (int64), geof
    (float32 [n, 4], column 3 doubled, or None), elevation (float32 [n]) and xyn (float32 [n, 2]).

    args: k_nn_adj, k_nn_local, use_voronoi, compute_geof, plane_model.  simplices: the triangulation of
    use_voronoi > 0 (spg_delaunay.delaunay(xyz) when None).  dataset:
      s3dis   objects: the pruned [n, n_objects + 1] histogram (pruned=True: first argmax of objects[:, 1:] plus 1,
              :126) or one id per vertex; is_transition = objects[s] != objects[t].
      vkitti  labels: the [n, C] histogram; objects = connected_comp of the edges whose hard labels (first argmax)
              agree, is_transition = hard[s] != hard[t].
      sema3d  labels None: labels = objects = [0], is_transition = False (:136-138).  With labels the objects come
              from libcp.cutpursuit2 on inpainting_problem(labels, graph_nn) (:150-165): inpaint=True computes them
              with spg_cut_pursuit.cutpursuit2 (lambda 0.01, k-means draws keyed by seed, so they equal libcp's
              only up to those draws), or pass them as objects= (else NotImplementedError); is_transition =
              objects[source] != objects[target] over every edge (:165).
    inpaint=True anywhere else (another dataset, no labels, objects given) raises ValueError.  Other datasets raise
    ValueError.  The reference's geof = 0 without compute_geof makes write_structure's len(geof)
    raise; here geof is None.  With plane_model the low points are fitted by sklearn's RANSACRegressor(random_state=0)
    on the host and elevation = float32(z - (x c0 + y c1 + b)) in fp64 on the device."""
    if dataset not in _DATASETS:
        raise ValueError("%s is an unknown data set" % dataset)
    k_adj, k_local = _field(args, "k_nn_adj"), _field(args, "k_nn_local")
    voronoi, want_geof, plane_model = (_field(args, "use_voronoi"), _field(args, "compute_geof"),
                                       _field(args, "plane_model"))
    n = n_points(np.shape(xyz))
    if inpaint and (dataset != "sema3d" or labels is None or objects is not None):
        raise ValueError("inpaint=True makes the objects of sema3d from its labels: it needs dataset 'sema3d', labels "
                         "and no objects")
    if dataset == "sema3d" and labels is not None and objects is None and not inpaint:
        raise NotImplementedError("sema3d with labels needs the objects of libcp.cutpursuit2 (node-weighted cut "
                                  "pursuit): pass inpaint=True to compute them on the device, or pass them as objects=")
    if dataset == "s3dis" and objects is None:
        raise ValueError("s3dis needs objects")
    if dataset == "vkitti" and labels is None:
        raise ValueError("vkitti needs labels")
    dev = device_of(xyz, rgb, labels, objects)
    with torch.cuda.device(dev):
        check_dtype(xyz, "xyz", "float32")
        x = on_device(xyz, dev)
        rgb_d = on_device(rgb, dev)
        if dataset == "s3dis":
            check_ints(labels, "labels")
            lab = on_device(labels, dev, int64=True)
            obj = (ops.st_argmax(_histogram(objects, "objects", n, dev), 1, 1)[0] if pruned
                   else _per_vertex(objects, "objects", n, dev))
        elif dataset == "vkitti":
            lab = _histogram(labels, "labels", n, dev)
        elif labels is None:
            lab = torch.zeros(1, dtype=torch.int64, device=dev)
            obj = torch.zeros(1, dtype=torch.int64, device=dev)
        else:
            check_ints(labels, "labels")
            lab = on_device(labels, dev, int64=True)
            obj = None if inpaint else _per_vertex(objects, "objects", n, dev)
        graph_nn, target2 = compute_graph_nn_2(x, k_adj, k_local, voronoi=voronoi, simplices=simplices)
        if inpaint:
            hard, s, t, edge_weight, node_weight = inpainting_problem(lab, graph_nn)
            obj = cutpursuit2(hard.to(torch.float32).reshape(n, 1), s, t, edge_weight, node_weight, 0.01,
                              seed=seed)[1]
        if dataset == "vkitti":
            hard = ops.st_argmax(lab, 0, 0)[0]
            is_tr = _transitions(hard, graph_nn)
            obj = connected_comp(n, graph_nn["source"], graph_nn["target"],
                                 _transitions(hard, graph_nn, ops.ST_EQUAL), 0)[1]
        elif dataset == "sema3d" and labels is None:
            is_tr = torch.zeros((), dtype=torch.uint8, device=dev)
        else:
            is_tr = _transitions(obj, graph_nn)
        geof = None
        if want_geof:
            geof = spg_geometry.compute_geof(x, target2, k_local)
        bounds = ops.knn_bounds(x)
        elevation = torch.empty(n, dtype=torch.float32, device=dev)
        xyn = torch.empty((n, 2), dtype=torch.float32, device=dev)
        low = torch.empty(n, dtype=torch.uint8, device=dev) if plane_model else None
        ops.st_points(x, bounds, elevation=elevation, xyn=xyn, low=low, geof=geof)
        if plane_model:
            ops.st_points(x, bounds, plane=_plane(x, bounds, low), elevation=elevation)
    return {"xyz": x, "rgb": rgb_d, "graph_nn": graph_nn, "target_local_geometry": target2.reshape(n, int(k_local)),
            "is_transition": is_tr, "labels": lab, "objects": obj, "geof": geof, "elevation": elevation, "xyn": xyn}


def _labels_numpy(labels):
    a = labels.cpu().numpy()
    if len(a) > 0 and a.ndim > 1 and a.shape[1] > 1:  # write_structure's choice of dtype (:218-221)
        return a.astype(np.int32)
    return a.astype(np.uint8)


def to_numpy(structure):
    """The structure with write_structure's dtypes (graph_processing.py:207-221): float32 xyz, rgb, elevation, xyn
    and geof (None when not computed), int64 source / target, uint8 is_transition, uint32 target_local_geometry and
    objects, labels int32 when a histogram, else uint8; graph_nn keeps its distances (float32)."""
    s = structure
    g = s["graph_nn"]
    return {"xyz": s["xyz"].cpu().numpy().astype(np.float32), "rgb": s["rgb"].cpu().numpy().astype(np.float32),
            "graph_nn": {"is_nn": True, "source": g["source"].cpu().numpy().astype(np.int64),
                         "target": g["target"].cpu().numpy().astype(np.int64),
                         "distances": g["distances"].cpu().numpy().astype(np.float32)},
            "target_local_geometry": s["target_local_geometry"].cpu().numpy().astype(np.uint32),
            "is_transition": s["is_transition"].cpu().numpy().astype(np.uint8),
            "labels": _labels_numpy(s["labels"]), "objects": s["objects"].cpu().numpy().astype(np.uint32),
            "geof": None if s["geof"] is None else s["geof"].cpu().numpy().astype(np.float32),
            "elevation": s["elevation"].cpu().numpy().astype(np.float32),
            "xyn": s["xyn"].cpu().numpy().astype(np.float32)}


def as_read_structure(structure, read_geof):
    """read_structure's tuple (graph_processing.py:224-247) of what write_structure would store, as numpy: (xyz, rgb,
    edg_source, edg_target, is_transition, local_geometry, labels, objects, elevation, xyn), ready for
    PartitionStore.add.  local_geometry is geof when read_geof, else target_local_geometry."""
    s = to_numpy(structure)
    labels = s["labels"].squeeze()
    if labels.ndim == 0:
        labels = np.array([0])
    is_tr = s["is_transition"]
    if is_tr.ndim == 0:
        is_tr = np.array([0])
    if read_geof:
        if s["geof"] is None:
            raise ValueError("the structure has no geof (compute_geof = 0)")
        local = s["geof"]
    else:
        local = s["target_local_geometry"]
    return (s["xyz"], s["rgb"], s["graph_nn"]["source"].squeeze(), s["graph_nn"]["target"].squeeze(), is_tr, local,
            labels, s["objects"], s["elevation"], s["xyn"])
