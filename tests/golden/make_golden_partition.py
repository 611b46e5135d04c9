"""Generates tests/golden/partition.npz by running the UNMODIFIED learned-partition objective of the reference on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_partition.py

supervized_partition/losses.py does not import here (libcp, libply_c and partition.provider are not built), so,
as make_golden.py::upsampling does, the SOURCE TEXT of its functions (zhang, compute_dist, compute_loss,
compute_partition, compute_weight_loss, compute_weights_SEAL, compute_weights_XPART, mode, relax_edge_binary),
of provider.py's perfect_prediction and of metrics.py's compute_boundary_recall / compute_boundary_precision is
read from the checkout and executed unmodified, on CPU tensors, in a namespace holding:
  * `libply_c.connected_comp`: a STAND-IN on scipy.sparse.csgraph.connected_components with the cutoff-0
    semantics of partition/ply_c/connected_components.cpp (no component is fused; components numbered by their
    smallest vertex, as boost's connected_components numbers them);
  * `libcp.cutpursuit`: a STAND-IN that records the edge weights it is handed and returns a fixed partition
    (cut pursuit itself is not part of what is pinned).

Cases: two batches of a synthetic graph (object blobs, 5 neighbours per vertex, edges in both directions,
duplicate edges, isolated vertices), "main" with transitions and "flat" with none.  For each: the distances of
every dist_type, loss1 / loss2 and their embedding gradient for every dist_type x loss, the weights of every
scheme, cut pursuit's edge weights for edge_weight_threshold -0.5 and 2, relax_edge_binary at tolerance 1 and 2
of both masks, the boundary recall / precision, and perfect_prediction.
"""
import json
import os
import types

import numpy as np
import torch

REF = os.environ["SPG_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))

DIST_TYPES = ["euclidian", "intrinsic", "scalar"]
LOSSES = ["tv_zhang", "laplacian_zhang", "TVH_zhang", "tv_TVminus", "laplacian_TVminus", "TVH_TVminus"]
SCHEMES = ["none", "proportional", "seal", "crosspartition"]


def grab(path, name):
    lines = open(os.path.join(REF, path)).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.startswith("def %s(" % name))
    end = start + 1
    while end < len(lines) and not (lines[end].startswith("def ") or lines[end].startswith("#")):
        end += 1
    return "\n".join(lines[start:end])


def connected_comp_standin(n_ver, edg_source, edg_target, active, cutoff):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    assert cutoff == 0
    act = active > 0
    g = coo_matrix((np.ones(int(act.sum()), dtype=np.int8), (edg_source[act], edg_target[act])), shape=(n_ver, n_ver))
    n, lab = connected_components(g, directed=False)
    return [np.nonzero(lab == c)[0].astype(np.uint32) for c in range(n)], lab.astype(np.uint32)


def reference_namespace(partition, seen):
    def cutpursuit(ver_value, s, t, edge_weight, *a, **k):
        seen.append(np.array(edge_weight))
        return partition

    ns = {"np": np, "torch": torch, "libply_c": types.SimpleNamespace(connected_comp=connected_comp_standin),
          "libcp": types.SimpleNamespace(cutpursuit=cutpursuit)}
    for name in ("zhang", "compute_dist", "compute_loss", "compute_partition", "compute_weight_loss",
                 "compute_weights_SEAL", "compute_weights_XPART", "mode", "relax_edge_binary"):
        exec(grab("supervized_partition/losses.py", name), ns)
    exec(grab("partition/provider.py", "perfect_prediction"), ns)
    for name in ("compute_boundary_recall", "compute_boundary_precision"):
        exec(grab("learning/metrics.py", name), ns)
    return ns


def make_graph(rng, n_ver, n_iso, n_obj, flat):
    """Points in object blobs; 5 nearest neighbours of every non-isolated vertex, both directions, a few
    duplicates; the predicted partition cuts space into voxels (so it only partly follows the objects)."""
    centres = rng.uniform(0, 10, size=(n_obj, 3))
    obj = rng.integers(0, n_obj, size=n_ver)
    xyz = centres[obj] + rng.normal(0, 0.8, size=(n_ver, 3))
    if flat:
        obj[:] = 0
    m = n_ver - n_iso
    d = ((xyz[:m, None, :] - xyz[None, :m, :]) ** 2).sum(-1)
    np.fill_diagonal(d, np.inf)
    nn = np.argsort(d, 1, kind="stable")[:, :5]
    s = np.repeat(np.arange(m), 5)
    t = nn.reshape(-1)
    src, tgt = np.concatenate([s, t]), np.concatenate([t, s])
    dup = rng.integers(0, len(src), size=40)
    src, tgt = np.concatenate([src, src[dup]]), np.concatenate([tgt, tgt[dup]])
    vox = np.floor(xyz / 2.5).astype(np.int64)
    _, pic = np.unique(vox[:, 0] * 10000 + vox[:, 1] * 100 + vox[:, 2], return_inverse=True)
    pic = pic.astype(np.uint32)
    comps = [np.nonzero(pic == c)[0].astype(np.uint32) for c in range(int(pic.max()) + 1)]
    is_tr = torch.from_numpy((obj[src] != obj[tgt]).astype(np.uint8))
    labels = np.zeros((n_ver, 14), dtype=np.uint32)
    labels[np.arange(n_ver), 1 + obj % 13] = rng.integers(1, 6, size=n_ver)
    labels[:, 1:] += rng.integers(0, 3, size=(n_ver, 13)).astype(np.uint32)
    labels[:, 0] = rng.integers(0, 2, size=n_ver)
    return dict(src=src.astype(np.int64), tgt=tgt.astype(np.int64), is_tr=is_tr, obj=obj.astype(np.int64),
                xyz=xyz.astype(np.float32), pic=pic, comps=comps, labels=labels)


def run_case(tag, gph, rng, arrs):
    n_ver = gph["xyz"].shape[0]
    partition = (gph["comps"], gph["pic"])
    seen = []
    ns = reference_namespace(partition, seen)
    src, tgt, is_tr = gph["src"], gph["tgt"], gph["is_tr"]
    D = 4
    emb0 = torch.nn.functional.normalize(torch.from_numpy(
        (np.eye(D)[gph["obj"] % D] + rng.normal(0, 0.4, size=(n_ver, D))).astype(np.float32)))
    arrs.update({tag + k: v for k, v in (("src", src), ("tgt", tgt), ("is_tr", is_tr.numpy()), ("obj", gph["obj"]),
                                          ("pic", gph["pic"].astype(np.int64)), ("labels", gph["labels"]),
                                          ("emb", emb0.numpy()))})
    args = types.SimpleNamespace(loss_weight="crosspartition", loss="TVH_zhang", dist_type="euclidian",
                                 transition_factor=5.0, k_nn_adj=5, edge_weight_threshold=-0.5, spatial_emb=0,
                                 reg_strength=1.0, CP_cutoff=10, cuda=0)
    for dt in DIST_TYPES:
        args.dist_type = dt
        diff = ns["compute_dist"](emb0, src, tgt, dt)
        arrs[tag + "diff.%s" % dt] = diff.numpy()
        # weights of every scheme (the partition comes from the cut-pursuit stand-in; they do not depend on
        # dist_type), and cut pursuit's edge weights
        for scheme in SCHEMES if dt == "euclidian" else []:
            args.loss_weight = scheme
            for thr in (-0.5, 2.0):
                args.edge_weight_threshold = thr
                del seen[:]
                try:
                    w = ns["compute_weight_loss"](args, emb0, torch.from_numpy(gph["obj"]), src, tgt, is_tr, diff,
                                                  True, gph["xyz"])[0].numpy()
                except ZeroDivisionError as e:  # 'proportional' without transitions
                    w = np.array("ZeroDivisionError: %s" % e)
                arrs[tag + "edge_weight.%g" % thr] = seen[0]
            arrs[tag + "w.%s" % scheme] = w
        weights = torch.from_numpy(arrs[tag + "w.crosspartition"])
        for loss in LOSSES:
            args.loss = loss
            emb = emb0.clone().requires_grad_(True)
            diff = ns["compute_dist"](emb, src, tgt, dt)
            l1, l2 = ns["compute_loss"](args, diff, is_tr, weights)
            (l1 + l2).backward()
            key = "%s.%s" % (dt, loss)
            arrs[tag + "loss1." + key] = l1.detach().numpy()
            arrs[tag + "loss2." + key] = l2.detach().numpy()
            arrs[tag + "grad." + key] = emb.grad.numpy()
    pred_tr = gph["pic"][src] != gph["pic"][tgt]
    arrs[tag + "pred_tr"] = pred_tr
    for tol in (1, 2):
        rp = ns["relax_edge_binary"](pred_tr, src, tgt, n_ver, tol)
        rt = ns["relax_edge_binary"](is_tr, src, tgt, n_ver, tol)
        arrs[tag + "relax_pred.%d" % tol] = rp
        arrs[tag + "relax_tr.%d" % tol] = rt
        it = is_tr.numpy()
        with np.errstate(invalid="ignore", divide="ignore"):
            arrs[tag + "BR.%d" % tol] = np.float64(ns["compute_boundary_recall"](it, rp))
            arrs[tag + "BP.%d" % tol] = np.float64(ns["compute_boundary_precision"](rt, pred_tr))
    arrs[tag + "perfect"] = ns["perfect_prediction"](gph["comps"], gph["labels"])
    # crosspartition components of the stand-in (what the device numbers by smallest vertex)
    cx, inx = connected_comp_standin(n_ver, src.astype("uint32"), tgt.astype("uint32"),
                                     (is_tr.numpy() + pred_tr == 0).astype("uint8"), 0)
    arrs[tag + "in_comp_x"] = inx.astype(np.int64)
    arrs[tag + "comp_x_size"] = np.array([len(c) for c in cx], dtype=np.int64)


def main():
    torch.set_num_threads(4)
    rng = np.random.default_rng(31)
    arrs = {}
    run_case("main.", make_graph(rng, 2000, 15, 12, False), rng, arrs)
    run_case("flat.", make_graph(rng, 300, 5, 1, True), rng, arrs)
    arrs["meta"] = json.dumps({"numpy": np.__version__, "torch": torch.__version__, "dist_types": DIST_TYPES,
                               "losses": LOSSES, "schemes": SCHEMES, "cases": ["main", "flat"],
                               "transition_factor": 5.0, "k_nn_adj": 5,
                               "connected_comp": "scipy stand-in, cutoff 0"})
    np.savez_compressed(os.path.join(OUT, "partition.npz"), **arrs)
    print("wrote partition.npz", sum(a.nbytes for a in arrs.values() if hasattr(a, "nbytes")) // 1024, "KiB")


if __name__ == "__main__":
    main()
