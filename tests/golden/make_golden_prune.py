"""Writes tests/golden/prune.npz: seeded clouds pruned by the reference's own `prune`
(partition/ply_c/ply_c.cpp:149-380), compiled by the recipe oracle/build_ref.py.

    SPG_REFERENCE=<superpoint_graph checkout> python oracle/build_ref.py
    python tests/golden/make_golden_prune.py

Cases: a room with labels and objects (supervized_partition/graph_processing.py:124), labels only
(partition/partition.py:124), neither, n_labels = 0 with objects, a cloud offset by 10^4 m, duplicated points with a
+-0 mix, coordinates on exact voxel boundaries, and a chunked cloud stored as the stack of the reference's per-chunk
results (partition/provider.py:265-297).  For every case: the inputs (<case>.xyz float32, .rgb uint8, .labels uint8,
.objects uint32) and the reference's outputs (<case>.out_xyz, .out_rgb, .out_labels, .out_objects).
"""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "prune.npz")


def _room(rng, n, lo=(0.0, 0.0, 0.0), hi=(4.0, 3.0, 2.5)):
    m = n // 3
    lo, hi = np.asarray(lo), np.asarray(hi)
    xyz = np.concatenate([np.c_[rng.uniform(lo[0], hi[0], m), rng.uniform(lo[1], hi[1], m), np.full(m, lo[2])],
                          np.c_[rng.uniform(lo[0], hi[0], m), np.full(m, lo[1]), rng.uniform(lo[2], hi[2], m)],
                          rng.uniform(lo, hi, (n - 2 * m, 3))])
    return (xyz + rng.normal(0, 0.004, xyz.shape)).astype(np.float32)


def cases():
    rng = np.random.default_rng(20261018)
    out = []

    def add(name, xyz, voxel, n_labels, n_objects, chunk_rows=0):
        n = len(xyz)
        out.append(dict(name=name, xyz=xyz, voxel=voxel, n_labels=n_labels, n_objects=n_objects,
                        chunk_rows=chunk_rows, rgb=rng.integers(0, 256, (n, 3)).astype(np.uint8),
                        labels=rng.integers(0, n_labels + 1, n).astype(np.uint8),
                        objects=rng.integers(0, n_objects + 1, n).astype(np.uint32)))

    add("room", _room(rng, 4000), 0.1, 13, 40)
    add("labels_only", _room(rng, 3000), 0.15, 8, 0)
    add("neither", _room(rng, 3000), 0.2, 0, 0)
    add("objects_no_labels", _room(rng, 2000), 0.2, 0, 6)
    add("offset", _room(rng, 3000, lo=(1e4, -1e4, 5e3), hi=(1e4 + 6, -1e4 + 4, 5e3 + 3)), 0.1, 5, 0)
    dup = _room(rng, 1500, lo=(-1, -1, -1), hi=(1, 1, 1))
    dup[::5] = dup[1::5][:len(dup[::5])]
    dup[:40, 0] = 0.0
    dup[40:80, 0] = -0.0
    dup[80:120, 2] = -0.0
    dup[120:160, 2] = 0.0
    dup[:, 1] = np.maximum(dup[:, 1], 0)  # y: the minimum is a zero of either sign
    dup[160:200, 1] = -0.0
    add("dup_zero", dup, 0.25, 4, 3)
    edge = (rng.integers(0, 40, (2000, 3)) * 0.125).astype(np.float32)  # x - x_min hits multiples of the voxel
    edge[1000:] += (rng.integers(0, 3, (1000, 3)) * 0.0625).astype(np.float32)
    add("boundary", edge, 0.25, 3, 0)
    add("chunked", _room(rng, 5000, hi=(8.0, 6.0, 3.0)), 0.2, 6, 0, chunk_rows=1500)
    return out


def main():
    ref = build_ref.load_prune()
    if ref is None:
        sys.exit("build the reference prune first: SPG_REFERENCE=<checkout> python oracle/build_ref.py")
    arrays, meta = {}, []
    for c in cases():
        name, n, rows = c["name"], len(c["xyz"]), c["chunk_rows"] or len(c["xyz"])
        parts = [ref(c["xyz"][s:s + rows], c["voxel"], c["rgb"][s:s + rows], c["labels"][s:s + rows],
                     c["objects"][s:s + rows], c["n_labels"], c["n_objects"]) for s in range(0, n, rows)]
        res = [np.vstack([p[k] for p in parts]) for k in range(4)]
        for k in ("xyz", "rgb", "labels", "objects"):
            arrays["%s.%s" % (name, k)] = c[k]
        for k, v in zip(("out_xyz", "out_rgb", "out_labels", "out_objects"), res):
            arrays["%s.%s" % (name, k)] = v
        meta.append(dict(name=name, voxel=c["voxel"], n_labels=c["n_labels"], n_objects=c["n_objects"],
                         chunk_rows=c["chunk_rows"], n=n, m=len(res[0])))
        print(name, n, "->", len(res[0]))
    gxx = subprocess.check_output(["g++", "--version"]).decode().splitlines()[0]
    arrays["meta"] = np.array(json.dumps(dict(cases=meta, numpy=np.__version__, gxx=gxx, flags=build_ref.FLAGS,
                                              extract_sha256=build_ref.SHA256)))
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes", hashlib.sha256(open(OUT, "rb").read()).hexdigest())


if __name__ == "__main__":
    main()
