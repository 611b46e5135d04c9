"""Times the device cut pursuit (spg_cut_pursuit.cutpursuit) and prints one JSON line.

    python tools/bench_cut_pursuit.py [--room N] [--learned N] [--host N]

room: N points (default 10^6) of a synthetic room (axis-aligned walls, floor and boxes, sampled with noise), 7
synthetic features per point in the layout of partition.py:165-166 (four geometric channels, verticality x2 and
rgb/255, each constant per surface plus noise; not compute_geof's output), k = 10 nearest-neighbour edges with edge_weight = 1 / (1 + d / mean d)
(partition.py:175), reg_strength 0.1, L2 mode.
learned: N vertices (default 10^5) with 4-D embeddings plus 0.2 xyz, k = 5, lambda = 1/20, cutoff 10,
weight_decay 0.7, SPG mode.
host: the float64 oracle (oracle/cut_pursuit_ref.py, a pure-Python max flow) on the first N vertices of each with
their own k-NN graph (default 10^4), with its time and the device-to-oracle energy ratio on the same crop.
Per-stage CUDA-event times (ms), push-relabel rounds, iterations, components and the final energy are reported,
with the card's name, power limit and maximum SM clock read in the same run.  The reference's libcp needs Boost,
which is not available here: its time is "not measured".
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superpoint_graph_b200 import spg_cut_pursuit as cp  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def room(n, rng):
    """A 6 x 5 x 3 m room: floor, ceiling, four walls and three boxes; features constant per surface plus noise."""
    surf = rng.integers(0, 9, n)
    xyz = rng.uniform(0, 1, (n, 3)) * np.array([6.0, 5.0, 3.0])
    xyz[surf == 0, 2] = 0.0
    xyz[surf == 1, 2] = 3.0
    xyz[surf == 2, 0] = 0.0
    xyz[surf == 3, 0] = 6.0
    xyz[surf == 4, 1] = 0.0
    xyz[surf == 5, 1] = 5.0
    for b in range(3):
        m = surf == 6 + b
        xyz[m] = np.array([1.0 + 1.5 * b, 1.0 + b, 0.0]) + rng.uniform(0, 0.8, (m.sum(), 3)) * np.array([1, 1, 0.8])
    geo = rng.uniform(0, 1, (9, 4))
    rgb = rng.uniform(0, 1, (9, 3))
    vert = np.where(np.isin(np.arange(9), [2, 3, 4, 5]), 1.0, 0.0)
    feat = np.concatenate([geo[surf], 2 * vert[surf][:, None], rgb[surf]], 1)
    feat += rng.normal(0, 0.03, feat.shape)
    xyz += rng.normal(0, 0.005, xyz.shape)
    return xyz.astype(np.float32), feat.astype(np.float32)


def knn_edges(xyz, k):
    d, nn = cKDTree(xyz).query(xyz, k + 1)
    src = np.repeat(np.arange(len(xyz)), k)
    return src, nn[:, 1:].ravel(), d[:, 1:].ravel()


class Timer:
    def __init__(self):
        self.ms = {}
        self.pending = []

    def __call__(self, stage):
        timer = self

        class Scope:
            def __enter__(self):
                self.s = torch.cuda.Event(enable_timing=True)
                self.e = torch.cuda.Event(enable_timing=True)
                self.s.record()

            def __exit__(self, *a):
                self.e.record()
                timer.pending.append((stage, self.s, self.e))
                return False

        return Scope()

    def collect(self):
        torch.cuda.synchronize()
        for stage, s, e in self.pending:
            self.ms[stage] = self.ms.get(stage, 0.0) + s.elapsed_time(e)
        return {k: round(v, 3) for k, v in self.ms.items()}


def device_run(obs, src, tgt, w, lam, cutoff, spatial, wd):
    args = (torch.from_numpy(obs).cuda(), torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(),
            torch.from_numpy(w).cuda())
    cp.cutpursuit(*args, lam, cutoff=cutoff, spatial=spatial, weight_decay=wd)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = cp.prepare(*args, lam, cutoff, spatial, wd)
    timer, stats = Timer(), {}
    cp.run(st, lam, cutoff, spatial, wd, 0, timer=timer, stats=stats)
    st.output()
    torch.cuda.synchronize()
    total = (time.perf_counter() - t0) * 1e3
    stats["stage_ms"] = timer.collect()
    stats["total_ms"] = round(total, 2)
    return stats


def host_arm(obs, xyz, k, weigh, lam, cutoff, spatial, wd, m):
    """The device and the oracle on the first m vertices with their own k-NN graph."""
    from oracle import cut_pursuit_ref as R
    src, tgt, d = knn_edges(xyz[:m], k)
    args = (obs[:m], src, tgt, weigh(d))
    dev = device_run(*args, lam, cutoff, spatial, wd)
    ref = {}
    t0 = time.perf_counter()
    R.cutpursuit(*args, lam, cutoff=cutoff, spatial=spatial, weight_decay=wd, stats=ref)
    return dict(n=m, oracle_s=round(time.perf_counter() - t0, 2), device_ms=dev["total_ms"],
                energy_ratio=dev["energy"] / ref["energy"], components=dev["components"],
                oracle_components=ref["components"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--room", type=int, default=1_000_000)
    ap.add_argument("--learned", type=int, default=100_000)
    ap.add_argument("--host", type=int, default=10_000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cut_pursuit needs a CUDA device")
    rng = np.random.default_rng(0)
    res = {"card": card(), "libcp": "not measured"}
    xyz, feat = room(a.room, rng)
    src, tgt, d = knn_edges(xyz, 10)
    weigh = lambda d: (1.0 / (1.0 + d / d.mean())).astype(np.float32)  # noqa: E731
    res["room"] = dict(n=a.room, n_edges=len(src), **device_run(feat, src, tgt, weigh(d), 0.1, 0, 0, 1.0))
    res["room"]["host"] = host_arm(feat, xyz, 10, weigh, 0.1, 0, 0, 1.0, a.host)
    lx = rng.uniform(0, 4, (a.learned, 3)).astype(np.float32)
    piece = (lx[:, 0] // 1 + 4 * (lx[:, 1] // 1)).astype(np.int64)
    emb = rng.normal(0, 1, (16, 4))[piece] + rng.normal(0, 0.1, (a.learned, 4))
    obs = np.concatenate([emb, 0.2 * lx], 1).astype(np.float32)
    s2, t2, _ = knn_edges(lx, 5)
    w2 = np.ones(len(s2), np.float32)
    res["learned"] = dict(n=a.learned, n_edges=len(s2), **device_run(obs, s2, t2, w2, 1 / 20, 10, 1, 0.7))
    res["learned"]["host"] = host_arm(obs, lx, 5, lambda d: np.ones(len(d), np.float32), 1 / 20, 10, 1, 0.7,
                                      a.host)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
