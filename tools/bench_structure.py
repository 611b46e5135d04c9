"""The learned partition's graph structure (superpoint_graph_b200/spg_structure.py); prints one JSON line.

    python tools/bench_structure.py [--reps 3] [--sizes room,scan] [--voronoi 0.01] [--no-host]

Sizes are tools/bench_delaunay.py's: `room`, 10^6 points of tests/test_sp_graph.py's room, and `scan`, 3 10^6 points
of tests/test_geometry.py's LiDAR-like scan with 1 cm of noise.  For each, medians over `reps` of the host clock
around work ending in a synchronise, with the L2 cache flushed (a 256 MiB write) before every run:
  `delaunay_ms`       spg_delaunay.delaunay(xyz)
  `vor_graph_ms`      spg_structure.compute_graph_nn_2(xyz, 5, 20, voronoi) from the precomputed device simplices
                      (the k-NN query included)
  `vor_graph_tri_ms`  the same with the triangulation included
  `knn_graph_ms`      spg_geometry.compute_graph_nn_2(xyz, 5, 20), the k-NN part alone
  `cc_ms`             spg_structure.connected_comp on the Voronoi graph, mask from a label field
  `structure_ms`      compute_structure(vkitti, voronoi, no plane, no geof) end to end, triangulation included
and, unless --no-host, once on the host from the same simplices and neighbour lists: `host_vor_ms` (numpy:
oracle/structure_ref.voronoi_graph, the reference's formula) and `host_cc_ms` (scipy's connected_components).  The
card's name, power limit and maximum SM clock are read in the same run.  Without a CUDA device the script exits.
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

_FLUSH = None


def timed(fn, reps):
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times, out = [], None
    for _ in range(reps):
        _FLUSH.fill_(1)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    return float(np.median(times)), out


def run_size(xyz_np, reps, voronoi, host, dev):
    from oracle import structure_ref
    from superpoint_graph_b200 import spg_geometry
    from superpoint_graph_b200 import spg_structure as st
    from superpoint_graph_b200.spg_delaunay import delaunay

    xyz = torch.from_numpy(xyz_np).to(dev)
    n = xyz.shape[0]
    out = {"n": int(n)}
    timed(lambda: st.compute_graph_nn_2(xyz, 5, 20, voronoi=voronoi), 1)  # warm-up of every shape
    out["delaunay_ms"], simp = timed(lambda: delaunay(xyz), reps)
    out["tetrahedra"] = int(simp.shape[0])
    out["vor_graph_ms"], (graph, target2) = timed(
        lambda: st.compute_graph_nn_2(xyz, 5, 20, voronoi=voronoi, simplices=simp), reps)
    out["vor_graph_tri_ms"], _ = timed(lambda: st.compute_graph_nn_2(xyz, 5, 20, voronoi=voronoi), reps)
    out["knn_graph_ms"], _ = timed(lambda: spg_geometry.compute_graph_nn_2(xyz, 5, 20), reps)
    out["edges"] = int(graph["source"].shape[0])
    out["kept_candidates"] = int(graph["distances"].shape[0])
    band = torch.floor(xyz[:, 2] * 2).to(torch.int64)
    active = (band[graph["source"]] == band[graph["target"]]).to(torch.uint8)
    out["cc_ms"], (comps, _) = timed(lambda: st.connected_comp(n, graph["source"], graph["target"], active, 0), reps)
    out["components"] = len(comps)
    labels = torch.nn.functional.one_hot(band.clamp(0, 12), 13).to(torch.int64)
    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=20, use_voronoi=voronoi, compute_geof=0, plane_model=0)
    out["structure_ms"], _ = timed(lambda: st.compute_structure(args, "vkitti", xyz, xyz, labels), reps)
    if host:
        simp_np = simp.cpu().numpy()
        nb = target2.cpu().numpy().reshape(n, 20)
        t = time.perf_counter()
        structure_ref.voronoi_graph(xyz_np, simp_np, nb, 5, voronoi)
        out["host_vor_ms"] = (time.perf_counter() - t) * 1e3
        s, tg, a = graph["source"].cpu().numpy(), graph["target"].cpu().numpy(), active.cpu().numpy()
        t = time.perf_counter()
        structure_ref.connected_comp(n, s, tg, a)
        out["host_cc_ms"] = (time.perf_counter() - t) * 1e3
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--sizes", default="room,scan")
    p.add_argument("--voronoi", type=float, default=0.01)
    p.add_argument("--no-host", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_structure.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from bench_sp_graph import card
    from superpoint_graph_b200 import _lib
    from test_geometry import falloff_cloud
    from test_sp_graph import _big_cloud
    _lib.lib()
    res = {"bench": "structure", "card": card(), "cpu": os.uname().machine, "nproc": os.cpu_count(), "reps": a.reps,
           "voronoi": a.voronoi}
    for size in a.sizes.split(","):
        if size.startswith("room"):
            xyz = _big_cloud(int(size[4:]) if size[4:] else 1000000, 21)[0]
        elif size == "scan":
            rng = np.random.default_rng(23)
            xyz = falloff_cloud(3000000, 22)
            xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)
        else:
            sys.exit("unknown size %r" % size)
        res[size] = run_size(np.ascontiguousarray(xyz, dtype=np.float32), a.reps, a.voronoi, not a.no_host, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
