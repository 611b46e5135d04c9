"""The superpoint graph of a partition (partition/graphs.py compute_sp_graph); prints one JSON line.

    python tools/bench_sp_graph.py [--reps 5] [--sizes room,scan] [--no-host]

Sizes (seeded clouds with stand-in partitions of voxel cells, 10^3-10^4 components; cut pursuit is not part of this):
  room  10^6 points on the surfaces and in the volume of a room (the generator of tests/test_sp_graph.py), 1 m cells
  scan  3 10^6 points of a LiDAR-like scan whose density falls off as 1 / range^2 (tests/test_geometry.py) with 1 cm
        of noise, 2 m cells
For each: `delaunay_ms`, the host scipy.spatial.Delaunay the caller runs (once; it bounds the end-to-end time);
`upload_ms`, the simplices' host-to-device copy; `superpoint_ms`, the superpoint pass (sort, unique rows, centroids,
eigen-solves, labels) and `superedge_ms`, the superedge pass (tetrahedra, pair deduplication, d_max cut, grouping,
features, with its two count read-backs), each timed with CUDA events, medians over `reps`; `front_end_ms`, the
superedge pass's first kernel (the per-tetrahedron count and its scan), with its algorithmic bytes (the int32
simplices, four int64 component ids per tetrahedron, the counts written, scanned and the offsets written) over
3.35 TB/s; `largest_component`, the points of the largest component, whose serial fp32 centroid sum sets the
superpoint pass's latency; `total_ms`, a host clock around compute_sp_graph with the simplices given, ending in a
synchronise.  The host arm (once): oracle/sp_graph_ref.py, the vectorised numpy restatement, after the same Delaunay.
The card's name, power limit and maximum SM clock are read in the same run.  Without a CUDA device the script exits.
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
N_LABELS = 8


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


def voxel_partition(xyz, cell):
    _, comp = np.unique(np.floor(xyz / cell).astype(np.int64), axis=0, return_inverse=True)
    return comp.reshape(-1).astype(np.uint32)


def run_size(xyz_np, comp_np, labels_np, d_max, reps, host, dev):
    from scipy.spatial import Delaunay

    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    n = xyz_np.shape[0]
    t0 = time.perf_counter()
    simplices = Delaunay(xyz_np).simplices
    delaunay_ms = 1e3 * (time.perf_counter() - t0)
    print("[bench_sp_graph] %d points: Delaunay %.0f ms" % (xyz_np.shape[0], delaunay_ms), file=sys.stderr, flush=True)
    T = simplices.shape[0]
    n_com = int(comp_np.max()) + 1
    comps = np.split(np.argsort(comp_np, kind="stable"), np.cumsum(np.bincount(comp_np))[:-1])
    xyz = torch.from_numpy(xyz_np).to(dev)
    comp = torch.from_numpy(comp_np.astype(np.int64)).to(dev)
    labels = torch.from_numpy(labels_np.astype(np.int64)).to(dev)

    def upload():
        return torch.from_numpy(simplices).to(dev)

    tets = upload()

    def superedges(sp):
        offsets, _ = ops.sp_edges_count(comp, tets)
        n_cand = int(offsets[-1].item())
        ws, n_sedg = ops.sp_edges_build(xyz, comp, tets, offsets, n_cand, d_max)
        return ops.sp_edges_features(xyz, T, n_cand, ws, int(n_sedg.item()), sp), n_cand

    def total():
        torch.cuda.synchronize()
        t = time.perf_counter()
        g = compute_sp_graph(xyz, d_max, comp, comps, labels, N_LABELS, simplices=tets)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t), g

    ms = {"upload": [], "superpoint": [], "superedge": [], "front_end": [], "total": []}
    for r in range(reps + 1):  # the first round warms up every shape
        t_up, _ = event_ms(upload)
        t_sp, (sp, _) = event_ms(lambda: ops.sp_points(xyz, comp, n_com, labels, 1, N_LABELS))
        t_se, (se, n_cand) = event_ms(lambda: superedges(sp[:5]))
        t_fe, _ = event_ms(lambda: ops.sp_edges_count(comp, tets))
        t_tot, g = total()
        if r:
            for k, v in (("upload", t_up), ("superpoint", t_sp), ("superedge", t_se), ("front_end", t_fe),
                         ("total", t_tot)):
                ms[k].append(v)
    med = {k: float(np.median(v)) for k, v in ms.items()}
    fe_bytes = T * (16 + 4 * 8 + 4 + 8 + 4)
    res = dict(points=n, components=n_com, tetrahedra=T, d_max=d_max, candidate_pairs=n_cand,
               superedges=int(g["source"].shape[0]), largest_component=int(np.bincount(comp_np).max()),
               delaunay_ms=delaunay_ms, upload_ms=med["upload"], upload_bytes=int(simplices.nbytes),
               superpoint_ms=med["superpoint"], superedge_ms=med["superedge"], front_end_ms=med["front_end"],
               front_end_bytes=int(fe_bytes),
               front_end_fraction_of_3_35_TBps=fe_bytes / HBM_BYTES_PER_S / (med["front_end"] * 1e-3),
               total_ms=med["total"], spread_total_ms=[float(min(ms["total"])), float(max(ms["total"]))])
    if host:
        from oracle import sp_graph_ref as sref
        t0 = time.perf_counter()
        sref.compute_sp_graph(xyz_np, d_max, comp_np, labels_np, N_LABELS, simplices)
        res["host_oracle_ms"] = 1e3 * (time.perf_counter() - t0)
        res["speedup_vs_host_oracle"] = res["host_oracle_ms"] / res["total_ms"]
    else:
        res["host_oracle_ms"] = "not run: --no-host"
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--sizes", default="room,scan")
    p.add_argument("--no-host", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sp_graph.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from superpoint_graph_b200 import _lib
    from test_geometry import falloff_cloud
    from test_sp_graph import _big_cloud
    _lib.lib()
    res = {"bench": "sp_graph", "card": card(), "cpu": os.uname().machine, "nproc": os.cpu_count(), "reps": a.reps}
    sizes = a.sizes.split(",")
    if "room" in sizes:
        xyz, comp, labels = _big_cloud(1000000, 21)
        res["room"] = run_size(xyz, comp, labels, 0.5, a.reps, not a.no_host, dev)
    if "scan" in sizes:
        rng = np.random.default_rng(23)
        xyz = falloff_cloud(3000000, 22)
        xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)  # the faces are exactly planar: qhull crawls
        labels = rng.integers(0, N_LABELS + 1, xyz.shape[0]).astype(np.uint8)
        res["scan"] = run_size(xyz, voxel_partition(xyz, 2.0), labels, 0.5, a.reps, not a.no_host, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
