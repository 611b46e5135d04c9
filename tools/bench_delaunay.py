"""The device Delaunay triangulation (superpoint_graph_b200/spg_delaunay.py); prints one JSON line.

    python tools/bench_delaunay.py [--reps 3] [--sizes room,scan] [--scipy] [--no-certificate]

The default sizes take about a minute of device time in all (reps + 1 triangulations each; see README.md for the
measured times), and the --scipy arm about four minutes more.  Sizes, built as tools/bench_sp_graph.py builds them:
  room   10^6 points on the surfaces and in the volume of a room (tests/test_sp_graph.py's generator), 1 m cells
  scan   3 10^6 points of a LiDAR-like scan (tests/test_geometry.py) with 1 cm of noise, 2 m cells
  room<N>, e.g. room20000: the room generator at N points.
For each: `delaunay_ms`, delaunay(xyz) from a device xyz to the sorted simplices (host clock ending in a
synchronise, median over `reps`); `rounds`, `tetrahedra`, `max_cavity`, `capacity` and `grows` of the last run;
`certificate`, oracle/delaunay_ref.py's check of the device output; `sp_graph_ms`, compute_sp_graph end to end from
the device xyz with the device simplices (delaunay included); with --scipy, `scipy_ms`, scipy.spatial.Delaunay on the
host, once.  The card's name, power limit and maximum SM clock are read in the same run.  Without a CUDA device the
script exits.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def wall_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def run_size(xyz_np, comp_np, reps, scipy_arm, certify, dev):
    from oracle import delaunay_ref
    from superpoint_graph_b200.spg_delaunay import delaunay, last_stats
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph

    xyz = torch.from_numpy(xyz_np).to(dev)
    comp = torch.from_numpy(comp_np.astype(np.int64)).to(dev)
    n_com = int(comp.max()) + 1
    times, simplices = [], None
    for _ in range(reps):
        ms, simplices = wall_ms(lambda: delaunay(xyz))
        times.append(ms)
    out = {"n": int(xyz_np.shape[0]), "delaunay_ms": float(np.median(times))}
    out.update(last_stats())
    if certify:
        out["certificate"] = bool(delaunay_ref.certificate(xyz_np, simplices.cpu().numpy()))
    ms, _ = wall_ms(lambda: compute_sp_graph(xyz, 0.5, comp, range(n_com), [], 0, simplices=delaunay(xyz)))
    out["sp_graph_ms"] = ms
    if scipy_arm:
        from scipy.spatial import Delaunay
        t = time.perf_counter()
        Delaunay(xyz_np)
        out["scipy_ms"] = (time.perf_counter() - t) * 1e3
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--sizes", default="room,scan")
    p.add_argument("--scipy", action="store_true")
    p.add_argument("--no-certificate", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_delaunay.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from bench_sp_graph import card, voxel_partition
    from superpoint_graph_b200 import _lib
    from test_geometry import falloff_cloud
    from test_sp_graph import _big_cloud
    _lib.lib()
    res = {"bench": "delaunay", "card": card(), "cpu": os.uname().machine, "nproc": os.cpu_count(), "reps": a.reps}
    for size in a.sizes.split(","):
        if size.startswith("room"):
            n = int(size[4:]) if size[4:] else 1000000
            xyz, comp, _ = _big_cloud(n, 21)
        elif size == "scan":
            rng = np.random.default_rng(23)
            xyz = falloff_cloud(3000000, 22)
            xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)
            comp = voxel_partition(xyz, 2.0)
        else:
            sys.exit("unknown size %r" % size)
        res[size] = run_size(xyz, comp, a.reps, a.scipy, not a.no_certificate, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
