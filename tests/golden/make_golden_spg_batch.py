"""Generates tests/golden/spg_batch.npz by running the UNMODIFIED superpoint-graph loader of the reference on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_spg_batch.py

learning/spg.py does not import here (igraph, h5py, sklearn), so the SOURCE TEXT of `spg_reader`,
`spg_edge_features`, `spg_to_igraph`, `random_neighborhoods`, `k_big_enough`, `loader`, `eccpc_collate`,
`load_superpoint`, `augment_cloud`, `cloud_edge_feats` and of the class `GraphConvInfo`
(learning/ecc/GraphConvInfo.py) is executed unmodified with compat/igraph, compat/h5py and compat/transforms3d as
stand-ins.  The graphs are spg_reader's output without scaler01 (the store takes the tuple as it is given).

Rooms, written by compat/make_fixture.write_room: 60 and 45 superpoints, and a room of 30 superpoints whose only
superedges are one pair u -> v, v -> u (rewritten after write_room), so that a sampled neighbourhood of it keeps an
edge only when a centre is u or v.  The parsed clouds keep their first 64 points and the columns xyzrgbe.  Python's `random` and numpy's global seed are set before every case; each case
records each graph's kept original ids and sub-graph edge list (the loader's, before the collate), the collated
batch or the collate's exception, and both generators' states afterwards.
"""
import io
import json
import math
import os
import random
import sys
import tempfile
import types
import zipfile
from collections import defaultdict

import numpy as np
import torch

REF = os.environ["SPG_REFERENCE"]
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "compat"))
import h5py  # noqa: E402  (compat/h5py)
import igraph  # noqa: E402  (compat/igraph)
import transforms3d  # noqa: E402  (compat/transforms3d)
from make_fixture import write_room  # noqa: E402

ROOMS = [("Area_1", "room_a", 60), ("Area_1", "room_b", 45), ("Area_2", "room_c", 30)]
ARGS = dict(edge_attribs="delta_avg,delta_std,nlength/ld,surface/ld,volume/ld,size/ld,xyz/d",
            spg_superedge_cutoff=-1, spg_augm_nneigh=100, spg_augm_order=3, spg_augm_hardcutoff=512, ptn_minpts=40,
            ptn_npts=16, pc_attribs="xyzrgbe", pc_xyznormalize=1, pc_augm_scale=0, pc_augm_rot=1,
            pc_augm_mirror_prob=0, pc_augm_jitter=1)

# name, room indices, train, args overrides, seed (Python's random and numpy's), test_seed_offset
CASES = [
    ("train_both", [0, 1], True, dict(spg_augm_nneigh=8, spg_augm_order=1, spg_augm_hardcutoff=20), 21, 0),
    ("train_nneigh", [0, 1], True, dict(spg_augm_nneigh=1, spg_augm_order=3, spg_augm_hardcutoff=0), 22, 0),
    ("train_cutoff", [0, 1], True, dict(spg_augm_nneigh=0, spg_augm_hardcutoff=15), 23, 0),
    ("train_neither", [1], True, dict(spg_augm_nneigh=0, spg_augm_hardcutoff=0, pc_augm_scale=1.2,
                                       pc_augm_mirror_prob=0.5), 24, 0),
    ("train_order0", [0], True, dict(spg_augm_nneigh=30, spg_augm_order=0, spg_augm_hardcutoff=0), 25, 0),
    ("train_nneigh_ge_n", [1], True, dict(spg_augm_nneigh=1000, spg_augm_hardcutoff=20), 26, 0),
    ("train_minpts_high", [0], True, dict(spg_augm_nneigh=6, spg_augm_order=1, spg_augm_hardcutoff=10,
                                          ptn_minpts=100000), 27, 0),
    ("train_middle_empty", [0, 2, 1], True, dict(spg_augm_nneigh=3, spg_augm_order=1, spg_augm_hardcutoff=0), 28, 0),
    ("train_first_empty", [2, 0], True, dict(spg_augm_nneigh=3, spg_augm_order=1, spg_augm_hardcutoff=0), 28, 0),
    ("eval_offset0", [0, 1], False, dict(), 29, 0),
    ("eval_offset2", [0, 1], False, dict(), 29, 2),
]


def grab(path, name, kind="def"):
    lines = open(os.path.join(REF, path)).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.startswith("%s %s(" % (kind, name)))
    end = start + 1
    while end < len(lines) and not (lines[end].startswith("def ") or lines[end].startswith("class ")
                                    or lines[end].startswith("####")):
        end += 1
    return "\n".join(lines[start:end])


def reference_namespace():
    ecc_ns = {"np": np, "torch": torch, "defaultdict": defaultdict, "igraph": igraph}
    exec(grab("learning/ecc/GraphConvInfo.py", "GraphConvInfo", "class"), ecc_ns)
    ns = {"np": np, "torch": torch, "os": os, "math": math, "random": random, "h5py": h5py, "igraph": igraph,
          "transforms3d": transforms3d, "ecc": types.SimpleNamespace(GraphConvInfo=ecc_ns["GraphConvInfo"])}
    for name in ("spg_edge_features", "spg_reader", "spg_to_igraph", "random_neighborhoods", "k_big_enough",
                 "loader", "cloud_edge_feats", "eccpc_collate", "load_superpoint", "augment_cloud"):
        exec(grab("learning/spg.py", name), ns)
    return ns


def write_rooms(root):
    rng = np.random.default_rng(53)
    for area, room, n_sp in ROOMS:
        write_room(h5py, root, int(area.split("_")[1]), room, n_sp, rng)
    # room_c: only the first superedge u -> v of the file and v -> u
    path = os.path.join(root, "superpoint_graphs", "Area_2", "room_c.h5")
    f = h5py.File(path, "r")
    data = {k: np.array(f[k][:]) for k in f.keys()}
    u, v = int(data["source"][0, 0]), int(data["target"][0, 0])
    keep = ((data["source"][:, 0] == u) & (data["target"][:, 0] == v)) | \
           ((data["source"][:, 0] == v) & (data["target"][:, 0] == u))
    assert keep.sum() == 2
    for k in ("source", "target", "se_delta_mean", "se_delta_std"):
        data[k] = data[k][keep]
    rewrite(path, data)
    # parsed clouds: the first 64 points and the 7 columns xyzrgbe read by pc_attribs, to keep the golden small
    for area, room, _ in ROOMS:
        path = os.path.join(root, "parsed", area, room + ".h5")
        f = h5py.File(path, "r")
        rewrite(path, {k: np.array(f[k][:64, :7]) for k in f.keys()})


def rewrite(path, data):
    os.remove(path)
    with h5py.File(path, "w") as g:
        for k, v in data.items():
            g.create_dataset(k, data=v)


def save_npz(path, arrs):
    """np.savez_compressed with a fixed timestamp on every member, so that a rerun gives the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for key, a in arrs.items():
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            z.writestr(info, buf.getvalue())


def states():
    py = random.getstate()
    np_state = np.random.get_state()
    return (np.array(py[1], dtype=np.int64), np.concatenate([np_state[1].astype(np.int64),
                                                              [np_state[2], np_state[3]]]).astype(np.int64))


def main():
    ns = reference_namespace()
    arrs, meta_cases = {}, []
    with tempfile.TemporaryDirectory() as root:
        write_rooms(root)
        base = types.SimpleNamespace(**ARGS)
        graphs = []
        for i, (area, room, _) in enumerate(ROOMS):
            g = ns["spg_reader"](base, os.path.join(root, "superpoint_graphs", area, room + ".h5"), True)
            graphs.append(g)
            for k, a in zip(("node_gt", "node_gt_size", "edges", "edge_feats"), g[:4]):
                arrs["room%d.%s" % (i, k)] = a
            parsed = h5py.File(os.path.join(root, "parsed", area, room + ".h5"), "r")
            for sp in range(g[0].shape[0]):
                arrs["room%d.sp%d" % (i, sp)] = np.array(parsed["%d" % sp][:])
        for tag, idx, train, over, seed, offset in CASES:
            args = dict(ARGS, **over)
            a = types.SimpleNamespace(**args)
            random.seed(seed)
            np.random.seed(seed)
            entries = [ns["spg_to_igraph"](*graphs[i]) for i in idx]
            batch = [ns["loader"](e, train, a, root, offset) for e in entries]
            p = tag + "."
            kept = []
            for b, (t, G, meta, flag, clouds, cglob) in enumerate(batch):
                kept.append(G is not None)
                if G is not None:
                    arrs[p + "ids.%d" % b] = np.array(G.vs["v"], dtype=np.int64)
                    arrs[p + "sub_edges.%d" % b] = np.array(G.get_edgelist(), dtype=np.int64).reshape(-1, 2)
            error = None
            try:
                targets, GIs, (meta, flag, clouds, cglob) = ns["eccpc_collate"](batch)
            except Exception as e:  # the collate's own exception is part of the record
                error = type(e).__name__
            py_state, np_state = states()
            arrs[p + "py_state"], arrs[p + "np_state"] = py_state, np_state
            if error is None:
                idxn, idxe, degs, degs_gpu, feats = GIs[0].get_buffers()
                arrs.update({p + "targets": targets.numpy(), p + "idxn": idxn.numpy(), p + "degs": degs.numpy(),
                             p + "edgefeats": feats.numpy(), p + "edge_index": GIs[0].get_pyg_buffers().numpy(),
                             p + "clouds_flag": flag.numpy(), p + "clouds": clouds.numpy(),
                             p + "clouds_global": cglob.numpy()})
            meta_cases.append(dict(tag=tag, rooms=idx, train=train, args=args, seed=seed, test_seed_offset=offset,
                                   kept=kept, error=error, clouds_meta=meta if error is None else None))
    assert [c for c in meta_cases if c["tag"] == "train_middle_empty"][0]["kept"] == [True, False, True]
    assert [c for c in meta_cases if c["tag"] == "train_first_empty"][0]["error"] == "TypeError"
    assert [c for c in meta_cases if c["tag"] == "train_minpts_high"][0]["error"] == "TypeError"
    arrs["meta"] = json.dumps({"numpy": np.__version__, "torch": torch.__version__, "fixture_seed": 53,
                               "rooms": [dict(name="%s/%s" % (a, r), n_sp=n) for a, r, n in ROOMS],
                               "cases": meta_cases})
    save_npz(os.path.join(OUT, "spg_batch.npz"), arrs)
    print("wrote spg_batch.npz", os.path.getsize(os.path.join(OUT, "spg_batch.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
