"""Voxel pruning (ply_c.cpp `prune`, superpoint_graph_b200.spg_prune); prints one JSON line.

    python tools/bench_prune.py [--reps 5] [--sizes room,scan,scene,voxel] [--no-host]

Sizes (seeded):
  room   10^6 points of a room (tests/test_prune.py's generator), 0.03 m voxels, 13 labels and 50 objects
  scan   10^7 points of a LiDAR-like scan whose density falls off as 1 / range^2 (tests/test_geometry.py), 0.03 m,
         13 labels
  scene  4 10^7 points of a 200 m x 200 m x 20 m scene in chunks of 5 10^6 (read_semantic3d_format's ver_batch
         default), 0.03 m, 8 labels
  voxel  2^24 points in one voxel: the longest serial fp32 chain the reduce can meet
For each: `bounds_ms`, `voxels_ms` and `reduce_ms`, the three passes (bounds and status with its read-back; keys,
sorts, flags, scans and runs with the voxel-count read-back; gather, serial sums and histograms) timed with CUDA
events, medians over `reps`; `bounds_bytes`, the bytes the bounds kernel must read (xyz and the int64 label and
object ids it checks) and that over 3.35 TB/s; `device_ms`, a host clock around prune() from device tensors, ending in
a synchronise; `pinned_ms`, the same from pinned host tensors (the upload included).  The host arms (once):
`reference_ms`, the reference's own prune (oracle/_ref, built by oracle/build_ref.py) on this host's cores, one call
per chunk as read_semantic3d_format makes them; `oracle_ms`, the numpy restatement; `bitwise_equal_*`, whether the
device outputs equal theirs bit for bit.  The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12


def log(*a):
    print("[bench_prune]", *a, file=sys.stderr, flush=True)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e), out


def _equal(got, want):
    return all(np.asarray(a).shape == np.asarray(b).shape and
               np.array_equal(np.asarray(a).astype(b.dtype).view(np.uint8), np.asarray(b).view(np.uint8))
               for a, b in zip(got, want))


def run_size(xyz_np, rgb_np, lab_np, obj_np, voxel, n_labels, n_objects, chunk_rows, reps, host, dev):
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_prune import prune
    n = xyz_np.shape[0]
    xyz = torch.from_numpy(xyz_np).to(dev)
    rgb = torch.from_numpy(rgb_np).to(dev)
    lab = torch.from_numpy(lab_np.astype(np.int64)).to(dev) if n_labels else None
    obj = torch.from_numpy(obj_np.astype(np.int64)).to(dev) if n_labels and n_objects else None
    pinned = [torch.from_numpy(a).pin_memory() for a in (xyz_np, rgb_np, lab_np, obj_np)]
    v = np.float32(voxel)
    ms = {k: [] for k in ("bounds", "voxels", "reduce", "device", "pinned")}
    for r in range(reps + 1):  # the first round warms up every shape
        ws = ops.prune_workspace(n, chunk_rows, dev)
        t_b, words = event_ms(lambda: [int(w) for w in
                                       ops.prune_bounds(xyz, chunk_rows, v, lab, n_labels, obj, n_objects, ws).cpu()])
        t_v, m = event_ms(lambda: int(ops.prune_voxels(xyz, chunk_rows, v, words[1:], ws).item()))
        t_r, _ = event_ms(lambda: ops.prune_reduce(xyz, rgb, lab, n_labels, obj, n_objects, chunk_rows, ws, m))
        del ws
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = prune(xyz, voxel, rgb, lab, obj, n_labels, n_objects, chunk_rows=chunk_rows)
        torch.cuda.synchronize()
        t_d = 1e3 * (time.perf_counter() - t)
        t = time.perf_counter()
        prune(pinned[0], voxel, pinned[1], pinned[2], pinned[3], n_labels, n_objects, chunk_rows=chunk_rows)
        torch.cuda.synchronize()
        t_p = 1e3 * (time.perf_counter() - t)
        if r:
            for k, x in (("bounds", t_b), ("voxels", t_v), ("reduce", t_r), ("device", t_d), ("pinned", t_p)):
                ms[k].append(x)
        log("%d points: round %d, device %.1f ms, pinned %.1f ms" % (n, r, t_d, t_p))
    med = {k: float(np.median(x)) for k, x in ms.items()}
    got = [t.cpu().numpy() for t in out]
    b_bytes = n * (12 + (8 if lab is not None else 0) + (8 if obj is not None else 0))
    res = dict(points=n, voxels=int(got[0].shape[0]), voxel=voxel, chunk_rows=chunk_rows, n_labels=n_labels,
               n_objects=n_objects,
               bounds_ms=med["bounds"], voxels_ms=med["voxels"], reduce_ms=med["reduce"],
               bounds_bytes=int(b_bytes),
               bounds_fraction_of_3_35_TBps=b_bytes / HBM_BYTES_PER_S / (med["bounds"] * 1e-3),
               device_ms=med["device"], pinned_ms=med["pinned"],
               spread_device_ms=[float(min(ms["device"])), float(max(ms["device"]))])
    if not host:
        res["reference_ms"] = res["oracle_ms"] = "not run: --no-host"
        return res
    from oracle import build_ref, prune_ref
    rows = chunk_rows or n
    ref = build_ref.load_prune()
    if ref is None:
        res["reference_ms"] = "not run: oracle/_ref/libply_c_prune.so not built"
    else:
        t = time.perf_counter()
        parts = [ref(xyz_np[s:s + rows], voxel, rgb_np[s:s + rows], lab_np[s:s + rows], obj_np[s:s + rows],
                     n_labels, n_objects) for s in range(0, n, rows)]
        res["reference_ms"] = 1e3 * (time.perf_counter() - t)
        res["bitwise_equal_reference"] = _equal(got, [np.vstack([p[k] for p in parts]) for k in range(4)])
        res["speedup_device_vs_reference"] = res["reference_ms"] / res["device_ms"]
        del parts
        log("%d points: reference %.0f ms" % (n, res["reference_ms"]))
    t = time.perf_counter()
    want = prune_ref.prune_chunked(xyz_np, voxel, rgb_np, lab_np, obj_np, n_labels, n_objects, rows)
    res["oracle_ms"] = 1e3 * (time.perf_counter() - t)
    res["bitwise_equal_oracle"] = _equal(got, want)
    log("%d points: oracle %.0f ms" % (n, res["oracle_ms"]))
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--sizes", default="room,scan,scene,voxel")
    p.add_argument("--no-host", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_prune.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from superpoint_graph_b200 import _lib
    from test_geometry import falloff_cloud
    from test_prune import _room_cloud
    _lib.lib()
    res = {"bench": "prune", "card": card(), "cpu": os.uname().machine, "nproc": os.cpu_count(), "reps": a.reps}
    sizes = a.sizes.split(",")
    host = not a.no_host
    rng = np.random.default_rng(31)
    if "room" in sizes:
        xyz, rgb, lab, obj = _room_cloud(1_000_000, 11, 13, 50)
        res["room"] = run_size(xyz, rgb, lab, obj, 0.03, 13, 50, 0, a.reps, host, dev)
    if "scan" in sizes:
        n = 10_000_000
        xyz = falloff_cloud(n, 22)
        res["scan"] = run_size(xyz, rng.integers(0, 256, (n, 3)).astype(np.uint8),
                               rng.integers(0, 14, n).astype(np.uint8), np.zeros(n, np.uint32), 0.03, 13, 0, 0,
                               a.reps, host, dev)
    if "scene" in sizes:
        n = 40_000_000
        m = n // 2
        xyz = np.concatenate([np.c_[rng.uniform(0, 200, (m, 2)), rng.normal(0, 0.05, m)],
                              rng.uniform((0, 0, 0), (200, 200, 20), (n - m, 3))]).astype(np.float32)
        res["scene"] = run_size(xyz, rng.integers(0, 256, (n, 3)).astype(np.uint8),
                                rng.integers(0, 9, n).astype(np.uint8), np.zeros(n, np.uint32), 0.03, 8, 0,
                                5_000_000, a.reps, host, dev)
    if "voxel" in sizes:
        n = 1 << 24
        xyz = rng.uniform(0, 0.02, (n, 3)).astype(np.float32)
        res["voxel"] = run_size(xyz, rng.integers(0, 256, (n, 3)).astype(np.uint8),
                                rng.integers(0, 14, n).astype(np.uint8), np.zeros(n, np.uint32), 0.03, 13, 0, 0,
                                a.reps, host, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
