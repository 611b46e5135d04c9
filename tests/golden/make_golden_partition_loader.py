"""Generates tests/golden/partition_loader.npz by running the UNMODIFIED learned-partition batch loader of the
reference on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_partition_loader.py

supervized_partition/graph_processing.py does not import here (h5py files, libply_c), so the SOURCE TEXT of its
`graph_loader`, `graph_collate` and `augment_cloud_whole` is read from the checkout and executed unmodified in a
namespace holding:
  * `read_structure`: a STAND-IN serving the synthetic files below from memory (fresh copies at every call, as a
    file read gives);
  * `libply_c.random_subgraph`: a STAND-IN returning a fixed mask, a seeded breadth-first search with the vertex
    budget written here (the sampler itself is not what is pinned), edges kept when both ends are;
  * `transforms3d`: compat/transforms3d;
  * `augment_cloud_whole`: the reference's function, wrapped to record the xyz / rgb it returns.

Synthetic files: three clouds of 400, 250 and 150 vertices (800 in all, so that the golden with every case stays
under 1 MB) in blobs, a 30-wide spatial kNN (self first) as `local_geometry` with a few duplicated neighbour ids, one
blob of 25 coincident points on quarter-unit coordinates (an exact float32 mean, so their neighbourhoods have
diameter exactly 0), a 5-NN edge graph in both directions, objects numbered from 0 in every file (so the collate's
max-not-max+1 offset collides), label histograms [n, 14] uint32.  Cases (train / eval, batch 1 and 3, use_rgb,
global_feat, augmentation with and without jitter, sub-sampling) are listed in CASES; numpy's global seed is set
before every case and recorded.
"""
import io
import json
import math
import os
import sys
import types
import zipfile

import numpy as np
import torch

REF = os.environ["SPG_REFERENCE"]
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "compat"))
import transforms3d  # noqa: E402  (compat/transforms3d)

FILES = [("Area_1/f0.h5", 400, 7), ("Area_1/f1.h5", 250, 5), ("Area_2/f2.h5", 150, 3)]
K_GEOMETRY = 30

# name, file indices, train, args overrides, numpy seed
CASES = [
    ("eval_b1", [0], False, dict(use_rgb=1, global_feat="eXYrgb"), 11),
    ("eval_b3", [0, 1, 2], False, dict(use_rgb=0, global_feat="e"), 12),
    ("train_sub", [0, 1, 2], True, dict(use_rgb=1, global_feat="exy", max_ver_train=120), 13),
    ("train_jitter", [0, 1, 2], True, dict(use_rgb=1, global_feat="eXYrgb", pc_augm_jitter=1, max_ver_train=120), 14),
    ("train_jitter_b1", [1], True, dict(use_rgb=0, global_feat="", pc_augm_jitter=1, max_ver_train=0), 15),
    ("train_rot_b1", [1], True, dict(use_rgb=1, global_feat="eXYrgb", pc_augm_rot=1, pc_augm_jitter=1,
                                     max_ver_train=0), 16),
    ("train_rot_nojitter_b1", [2], True, dict(use_rgb=1, global_feat="eXYrgb", pc_augm_rot=1, pc_augm_jitter=0,
                                              max_ver_train=0), 18),
    ("train_rot_b3", [0, 1, 2], True, dict(use_rgb=0, global_feat="exy", pc_augm_rot=1, pc_augm_jitter=1,
                                           max_ver_train=120), 17),
]


def grab(path, name):
    lines = open(os.path.join(REF, path)).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.startswith("def %s(" % name))
    end = start + 1
    while end < len(lines) and not (lines[end].startswith("def ") or lines[end].startswith("#")):
        end += 1
    return "\n".join(lines[start:end])


def make_file(rng, n, n_obj):
    """xyz in object blobs (one blob of 25 coincident points), rgb 0..255, 30-NN local geometry (self first,
    stable order, a few duplicated ids), 5-NN edges both ways, objects from 0."""
    centres = rng.uniform(0, 6, size=(n_obj, 3))
    obj = np.sort(rng.integers(0, n_obj, size=n))
    xyz = (centres[obj] + rng.normal(0, 0.4, size=(n, 3))).astype(np.float32)
    # 25 coincident points on a coordinate with few mantissa bits, so that numpy's float32 mean of 20 copies is
    # exact: their 20 nearest neighbours have diameter exactly 0 and the clouds divide by 1e-10 alone
    xyz[:25] = np.round(xyz[0] * 4) / 4
    d = ((xyz[:, None, :].astype(np.float64) - xyz[None, :, :]) ** 2).sum(-1)
    d[np.arange(n), np.arange(n)] = -1.0  # self first
    order = np.argsort(d, 1, kind="stable")
    lg = order[:, :K_GEOMETRY].astype(np.uint32)
    dup = rng.integers(0, n, size=12)
    lg[dup, 3] = lg[dup, 2]  # duplicate neighbours
    nn = order[:, 1:6]
    s, t = np.repeat(np.arange(n), 5), nn.reshape(-1)
    src, tgt = np.concatenate([s, t]).astype(np.int64), np.concatenate([t, s]).astype(np.int64)
    is_tr = (obj[src] != obj[tgt]).astype(np.uint8)
    labels = np.zeros((n, 14), dtype=np.uint32)
    labels[np.arange(n), 1 + obj % 13] = rng.integers(1, 9, size=n)
    labels[:, 0] = rng.integers(0, 3, size=n)
    rgb = rng.integers(0, 256, size=(n, 3)).astype(np.float32)
    elevation = ((xyz[:, 2] - xyz[:, 2].min()) / np.ptp(xyz[:, 2]) - 0.5).astype(np.float32)
    xyn = ((xyz[:, :2] - xyz[:, :2].mean(0)) / 3).astype(np.float32)
    return (xyz, rgb, src, tgt, is_tr, lg, labels, obj.astype(np.int64), elevation, xyn)


def random_subgraph_standin(n_ver, src, tgt, max_ver):
    """Breadth-first search from seeded random starts until max_ver vertices are selected."""
    rng = np.random.default_rng(1000 + n_ver)
    adj = [[] for _ in range(n_ver)]
    for s, t in zip(src.tolist(), tgt.tolist()):
        adj[s].append(t)
    sel = np.zeros(n_ver, dtype=np.uint8)
    count = 0
    while count < max_ver:
        start = int(rng.choice(np.nonzero(sel == 0)[0]))
        queue, sel[start], count = [start], 1, count + 1
        while queue and count < max_ver:
            v = queue.pop(0)
            for u in adj[v]:
                if not sel[u] and count < max_ver:
                    sel[u], count = 1, count + 1
                    queue.append(u)
    return (sel[src] * sel[tgt]).astype(np.uint8), sel


def reference_namespace(files, record, masks):
    def read_structure(entry, read_geof):
        assert not read_geof
        return tuple(np.array(a, copy=True) for a in files[entry])

    def random_subgraph(n_ver, src, tgt, max_ver):
        e, v = random_subgraph_standin(n_ver, src, tgt, max_ver)
        masks.append(v.astype(bool))
        return e, v

    ns = {"np": np, "torch": torch, "os": os, "math": math, "transforms3d": transforms3d,
          "read_structure": read_structure, "libply_c": types.SimpleNamespace(random_subgraph=random_subgraph)}
    path = "supervized_partition/graph_processing.py"
    for name in ("graph_loader", "graph_collate", "augment_cloud_whole"):
        exec(grab(path, name), ns)
    inner = ns["augment_cloud_whole"]

    def augment_cloud_whole(args, xyz, rgb):
        out = inner(args, xyz, rgb)
        record.append((np.array(out[0]), np.array(out[1])))
        return out

    ns["augment_cloud_whole"] = augment_cloud_whole
    return ns


def save_npz(path, arrs):
    """np.savez_compressed with a fixed timestamp on every member, so that a rerun gives the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for key, a in arrs.items():
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            z.writestr(info, buf.getvalue())


def main():
    rng = np.random.default_rng(47)
    files = {name: make_file(rng, n, n_obj) for name, n, n_obj in FILES}
    arrs = {}
    keys = ("xyz", "rgb", "src", "tgt", "is_tr", "lg", "labels", "objects", "elevation", "xyn")
    for i, (name, _, _) in enumerate(FILES):
        for k, a in zip(keys, files[name]):
            arrs["file%d.%s" % (i, k)] = a
    meta_cases = []
    for tag, idx, train, over, seed in CASES:
        args = dict(ver_value="ptn", learned_embeddings=True, k_nn_local=20, use_rgb=1, global_feat="eXYrgb",
                    pc_augm_rot=0, pc_augm_jitter=0, max_ver_train=0)
        args.update(over)
        record, masks = [], []
        ns = reference_namespace(files, record, masks)
        np.random.seed(seed)
        names = [FILES[i][0] for i in idx]
        batch = ns["graph_collate"]([ns["graph_loader"](nm, train, types.SimpleNamespace(**args), "")
                                     for nm in names])
        fname, src, tgt, is_tr, labels, objects, (clouds, cglob, nei), xyz = batch
        p = tag + "."
        arrs.update({p + "edg_source": src, p + "edg_target": tgt, p + "is_transition": is_tr.numpy(),
                     p + "labels": labels, p + "objects": objects.numpy(), p + "clouds": clouds.numpy(),
                     p + "clouds_global": cglob.numpy(), p + "nei": nei, p + "xyz": xyz})
        for b, (ax, ar) in enumerate(record):
            arrs[p + "aug_xyz.%d" % b], arrs[p + "aug_rgb.%d" % b] = ax, ar
        for b, m in enumerate(masks):
            arrs[p + "mask.%d" % b] = m
        meta_cases.append(dict(tag=tag, files=idx, train=train, args=args, seed=seed, fname=list(fname),
                               subsampled=len(masks) > 0))
    arrs["meta"] = json.dumps({"numpy": np.__version__, "torch": torch.__version__, "generator_seed": 47,
                               "files": [dict(name=n, n_ver=v, n_obj=o) for n, v, o in FILES],
                               "random_subgraph": "seeded BFS stand-in", "cases": meta_cases})
    save_npz(os.path.join(OUT, "partition_loader.npz"), arrs)
    print("wrote partition_loader.npz", os.path.getsize(os.path.join(OUT, "partition_loader.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
