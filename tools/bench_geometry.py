"""k-NN graphs and geometric features of a point cloud (partition/graphs.py compute_graph_nn_2 + ply_c compute_geof);
prints one JSON line.

    python tools/bench_geometry.py [--reps 7] [--sizes room,scene] [--no-host]

Sizes (seeded clouds, the generators of tests/test_geometry.py):
  room   10^6 points on the surfaces of a room (floor, ceiling, walls, a table, a cylinder), at (k_nn1, k_nn2) =
         (10, 45) (partition/partition.py:146-152) and (5, 20) (supervized_partition/graph_processing.py:146,176)
  scene  10^7 points of a LiDAR-like scan whose density falls off as 1 / range^2, at (10, 45)
For each: `grid_wall_ms`, a host clock around the whole grid set-up ending in a synchronise (host and device time: the
bounds, up to four builds and their occupancy read-backs); `grid_build_ms`, one build at the chosen cell size (keys,
sort, cell table) timed with CUDA events; the query and compute_geof, each timed with CUDA events; and `total_ms`, a
host clock around compute_graph_nn_2 + compute_geof ending in a synchronise; medians over `reps` repetitions, the arms
alternated.  `geof` also reports its algorithmic bytes (xyz and ids read once, the features written) over 3.35 TB/s.  The host arm (room only, once): scikit-learn's
NearestNeighbors(algorithm='kd_tree') as the reference calls it, plus oracle/geometry_ref.py's compute_geof; it is
reported as not run when scikit-learn does not import.  The card's name, power limit and maximum SM clock are read
in the same run.  Without a CUDA device the script exits.
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


def run_size(xyz_np, pairs, reps, dev):
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_geometry import build_grid, compute_geof, compute_graph_nn_2
    n = xyz_np.shape[0]
    xyz = torch.from_numpy(xyz_np).to(dev)
    res = {}
    for k1, k2 in pairs:
        def phases():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            grid, ws = build_grid(xyz, k2)
            torch.cuda.synchronize()
            t_wall = 1e3 * (time.perf_counter() - t0)
            t_grid, _ = event_ms(lambda: ops.knn_grid(xyz, grid, ws))
            t_query, (_, _, _, target2) = event_ms(lambda: ops.knn_query(n, k2, k1, grid, ws, True))
            t_geof, _ = event_ms(lambda: compute_geof(xyz, target2, k2))
            return t_wall, t_grid, t_query, t_geof, grid

        def total():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, target2 = compute_graph_nn_2(xyz, k1, k2)
            compute_geof(xyz, target2, k2)
            torch.cuda.synchronize()
            return 1e3 * (time.perf_counter() - t0)

        phases()
        total()
        ms = {"grid_wall": [], "grid": [], "query": [], "geof": [], "total": []}
        for _ in range(reps):
            w, g, q, f, grid = phases()
            ms["grid_wall"].append(w)
            ms["grid"].append(g)
            ms["query"].append(q)
            ms["geof"].append(f)
            ms["total"].append(total())
        med = {k: float(np.median(v)) for k, v in ms.items()}
        geof_bytes = n * 12 + n * k2 * 8 + n * 16
        res["%d_%d" % (k1, k2)] = dict(
            grid_wall_ms=med["grid_wall"], grid_build_ms=med["grid"], query_ms=med["query"], geof_ms=med["geof"],
            total_ms=med["total"],
            points_per_s=n / (med["total"] * 1e-3), cell=grid[3], cells_per_axis=list(grid[4:]),
            geof_bytes=int(geof_bytes), geof_fraction_of_3_35_TBps=geof_bytes / HBM_BYTES_PER_S / (med["geof"] * 1e-3),
            spread_total_ms=[float(min(ms["total"])), float(max(ms["total"]))])
    res["points"] = n
    return res


def host_arm(xyz, k1, k2):
    try:
        from sklearn.neighbors import NearestNeighbors
    except ImportError:
        return "not run: scikit-learn does not import"
    from oracle import geometry_ref as gref
    t0 = time.perf_counter()
    nn = NearestNeighbors(n_neighbors=k2 + 1, algorithm="kd_tree").fit(xyz)
    distances, neighbors = nn.kneighbors(xyz)
    t1 = time.perf_counter()
    geof = gref.compute_geof(xyz, neighbors[:, 1:].reshape(-1), k2)
    t2 = time.perf_counter()
    return dict(pair="%d_%d" % (k1, k2), sklearn_knn_ms=1e3 * (t1 - t0), oracle_geof_ms=1e3 * (t2 - t1),
                total_ms=1e3 * (t2 - t0), nan_rows=int(np.isnan(geof).any(1).sum()),
                host_threads=torch.get_num_threads())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=7)
    p.add_argument("--sizes", default="room,scene")
    p.add_argument("--no-host", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_geometry.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from superpoint_graph_b200 import _lib
    from test_geometry import falloff_cloud, room_cloud
    _lib.lib()
    res = {"bench": "knn_graph_geof", "card": card(), "cpu": os.uname().machine, "nproc": os.cpu_count(),
           "reps": a.reps}
    sizes = a.sizes.split(",")
    if "room" in sizes:
        xyz = room_cloud(1000000, 11)
        res["room"] = run_size(xyz, [(10, 45), (5, 20)], a.reps, dev)
        res["room"]["host"] = "not run: --no-host" if a.no_host else host_arm(xyz, 10, 45)
        if isinstance(res["room"]["host"], dict):
            res["room"]["speedup_vs_host"] = res["room"]["host"]["total_ms"] / res["room"]["10_45"]["total_ms"]
    if "scene" in sizes:
        res["scene"] = run_size(falloff_cloud(10000000, 12), [(10, 45)], a.reps, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
