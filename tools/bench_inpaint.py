"""Times Semantic3D's label inpainting on the device (spg_cut_pursuit.cutpursuit2 and
spg_structure.compute_structure(..., inpaint=True)) and prints one JSON line.

    python tools/bench_inpaint.py [--sizes 1000000,5000000] [--crop 10000] [--repeats 3]

Workload: Semantic3D-shaped synthetic scans of N points (a 60 x 60 m patch of ground whose terrain class changes
every 10 m, building walls, vegetation and car-sized boxes: 8 classes), labelled on about 70 % of the points (the
rest in unlabelled blobs and scattered points, plus a few unlabelled clusters far from the scan, which stay apart as
NaN-valued components), the 5-NN graph of the device (k_nn_adj = 5), lambda 0.01 as graph_processing.py:163.
cutpursuit2: the median of `repeats` timed calls on the problem already on the device (set-up, the main loop and the
output), with its iterations, components and push-relabel rounds.  compute_structure: the
median of `repeats` calls from host arrays to the device structure.  oracle: the float64 oracle
(oracle/cut_pursuit2_ref.py cutpursuit2, a pure-Python max flow) on the inpainting problem of a `crop`-point disc of
the first scan, its time and whether the device's in_component equals it.  The card's name, power limit and maximum
SM clock are read in the same run.  libcp's cutpursuit2 needs Boost, which is not available here: "not measured".
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from superpoint_graph_b200 import spg_cut_pursuit as cp  # noqa: E402
from superpoint_graph_b200 import spg_structure as st  # noqa: E402

LAMBDA, K_ADJ, K_LOCAL = 0.01, 5, 20


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def scan(n, rng):
    """xyz float32 [n, 3], rgb uint8 [n, 3], labels int64 [n, 9] (column 0: unlabelled)."""
    kind = rng.choice(4, n, p=[0.55, 0.2, 0.15, 0.1])  # ground, walls, vegetation, boxes
    xyz = rng.uniform(0, 60, (n, 3))
    xyz[:, 2] = rng.normal(0, 0.02, n)
    cls = np.where((np.floor(xyz[:, 0] / 10) + np.floor(xyz[:, 1] / 10)) % 2 == 0, 1, 2)  # man-made / natural
    w = kind == 1  # four building walls 8 m high
    side = rng.integers(0, 4, n)
    xyz[w, 2] = rng.uniform(0, 8, w.sum())
    xyz[w & (side == 0), 0] = 5.0
    xyz[w & (side == 1), 0] = 55.0
    xyz[w & (side == 2), 1] = 5.0
    xyz[w & (side == 3), 1] = 55.0
    cls[w] = 5
    v = kind == 2  # 40 trees / bushes
    centre = rng.uniform(8, 52, (40, 2))[rng.integers(0, 40, v.sum())]
    xyz[v, :2] = centre + rng.normal(0, 1.0, (v.sum(), 2))
    xyz[v, 2] = rng.uniform(0, 6, v.sum())
    cls[v] = np.where(xyz[v, 2] > 2, 3, 4)
    b = kind == 3  # 30 boxes: cars, hardscape, artefacts
    k = rng.integers(0, 30, b.sum())
    xyz[b, :2] = rng.uniform(8, 52, (30, 2))[k] + rng.uniform(0, [4.0, 2.0], (b.sum(), 2))
    xyz[b, 2] = rng.uniform(0, 1.5, b.sum())
    cls[b] = np.array([6, 7, 8])[k % 3]
    labels = np.zeros((n, 9), np.int64)
    labels[np.arange(n), cls] = rng.integers(1, 5, n)
    unlab = rng.uniform(size=n) < 0.12
    for c in rng.uniform(0, 60, (25, 2)):  # unlabelled blobs of 3 m radius
        unlab |= ((xyz[:, :2] - c) ** 2).sum(1) < 9.0
    stray = rng.uniform(size=n) < 2e-4  # unlabelled clusters far from the scan
    xyz[stray] = np.array([200.0, 200.0, 0.0]) + rng.integers(0, 5, (stray.sum(), 1)) * 20.0 + \
        rng.normal(0, 0.3, (stray.sum(), 3))
    unlab |= stray
    labels[unlab, 1:] = 0
    labels[unlab, 0] = 1
    rgb = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    return xyz.astype(np.float32), rgb, labels


def problem(xyz, labels):
    """The inpainting problem of graph_processing.py:152-162 on the device's 5-NN graph."""
    graph, _ = st.compute_graph_nn_2(torch.from_numpy(xyz).cuda(), K_ADJ, K_LOCAL)
    hard, s, t, ew, nw = st.inpainting_problem(torch.from_numpy(labels).cuda(), graph)
    return hard.to(torch.float32).reshape(-1, 1), s, t, ew, nw


def timed_cutpursuit2(args, repeats):
    cp.cutpursuit2(*args, LAMBDA)  # warm-up
    times, stats = [], {}
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        state = cp.prepare(*args[:4], LAMBDA, 0, 1, 1.0, node_weight=args[4])
        cp.run(state, LAMBDA, 0, 1, 1.0, 0, stats=stats)
        _, inc = state.output()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return dict(ms=round(float(np.median(times)), 2), ms_all=[round(x, 2) for x in times],
                iterations=stats["iterations"], components=stats["components"],
                push_relabel_rounds=stats["push_relabel_rounds"]), inc


def timed_structure(xyz, rgb, labels, repeats):
    args = types.SimpleNamespace(k_nn_adj=K_ADJ, k_nn_local=K_LOCAL, use_voronoi=0.0, compute_geof=0, plane_model=0)
    times = []
    for i in range(repeats + 1):  # the first call warms the structure kernels up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = st.compute_structure(args, "sema3d", xyz, rgb, labels, inpaint=True)
        torch.cuda.synchronize()
        if i:
            times.append((time.perf_counter() - t0) * 1e3)
    return dict(ms=round(float(np.median(times)), 2), ms_all=[round(x, 2) for x in times],
                objects=int(out["objects"].max().item()) + 1,
                transitions=int(out["is_transition"].sum().item()))


def oracle_arm(xyz, labels, m):
    from scipy.spatial import cKDTree

    from oracle import cut_pursuit2_ref as R
    _, idx = cKDTree(xyz[:, :2]).query(np.array([30.0, 30.0]), m)
    idx = np.sort(idx)
    args = problem(np.ascontiguousarray(xyz[idx]), np.ascontiguousarray(labels[idx]))
    _, inc = cp.cutpursuit2(*args, LAMBDA)
    host = [a.cpu().numpy() for a in args]
    ref = {}
    t0 = time.perf_counter()
    _, _, comp = R.cutpursuit2(*host, LAMBDA, stats=ref)
    return dict(n=m, n_edges=int(host[1].size), oracle_s=round(time.perf_counter() - t0, 2),
                equal=bool(np.array_equal(inc.cpu().numpy(), comp)), components=ref["components"],
                iterations=ref["iterations"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,5000000")
    ap.add_argument("--crop", type=int, default=10_000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_inpaint needs a CUDA device")
    res = {"card": card(), "libcp": "not measured", "lambda": LAMBDA, "k_nn_adj": K_ADJ}
    first = None
    for n in [int(s) for s in a.sizes.split(",")]:
        xyz, rgb, labels = scan(n, np.random.default_rng(n))
        first = first or (xyz, labels)
        args = problem(xyz, labels)
        r = dict(n=n, n_edges=int(args[1].numel()), labelled=round(float((labels[:, 1:].sum(1) > 0).mean()), 3))
        r["cutpursuit2"], _ = timed_cutpursuit2(args, a.repeats)
        del args
        r["compute_structure"] = timed_structure(xyz, rgb, labels, a.repeats)
        res[str(n)] = r
    if a.crop:
        res["oracle"] = oracle_arm(*first, a.crop)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
