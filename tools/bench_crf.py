"""ECC-CRF kernel timings (ECC_CRFModule, `crf_<R>` model configs); prints one JSON line.

    python tools/bench_crf.py [--reps 50]

Two sizes, C = 13 classes (S3DIS, vKITTI), R = 3 iterations, random [E, C, C] filters (the filter
network is not part of what is timed):
  batch  configs[1]-sized: synthetic.make_batch, 1024 superpoints, ~10 in-edges per node
  sweep  100 k superpoints, ~1 M edges, L2 flushed (256 MiB memset) before every timed launch group

Timed with CUDA events, after warm-up, median over `reps` repetitions:
  fwd        crf_softmax + R x crf_fwd (the module's forward without the filter network)
  composed   the same recurrence from existing pieces: ops.ecc_fwd (the generic ECC kernel at C != 32),
             then torch's subtraction and softmax, per iteration; alternated with `fwd` in one loop
  bwd_steps  R x crf_bwd (gradient w.r.t. U)
  bwd_w      the filter gradient of all R iterations (ops.ecc_bwd_w, n_iter = R)
Algorithmic bytes of one forward iteration: filters 4*C*C*E, idxn 4*E, rowptr 4*(N+1), Q gathered (counted
once) 4*C*N, Z and Q written 8*C*N, U read 4*C*N (about 680 B per edge at C = 13).  `fwd` is reported as
GB/s and as a share of the H100 SXM's 3.35 TB/s HBM3 bandwidth: a kernel-level HBM bound, not an
end-to-end figure.  The card's name, power limit and maximum SM clock are read in the same run.

There is no CPU fallback: without a CUDA device the script exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12  # B/s, NVIDIA H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def iter_bytes(N, E, C):
    return 4 * C * C * E + 4 * E + 4 * (N + 1) + 4 * C * N + 8 * C * N + 4 * C * N


def run_size(dev, label, batch, C, R, reps, flush):
    from superpoint_graph_b200 import ops
    N, E = batch["degs"].numel(), batch["idxn"].numel()
    graph = ops.EccGraph(batch["idxn"], None, batch["degs"], n_in=N)
    graph.to(dev)
    torch.manual_seed(0)
    U = torch.randn(N, C, device=dev) * 2
    W = torch.randn(E, C, C, device=dev) * 0.3
    g = torch.randn(N, C, device=dev)
    qs = torch.empty((R, N, C), device=dev)
    out = torch.empty((N, C), device=dev)
    gps = torch.empty((R, N, C), device=dev)
    gu = torch.empty((N, C), device=dev)
    gw = torch.empty((E, C, C), device=dev)

    def fwd():
        ops.crf_softmax(U, out=qs[0])
        for r in range(1, R + 1):
            ops.crf_fwd_step(U, qs[r - 1], W, graph, out if r == R else qs[r], softmax=r < R)

    def composed():
        q = torch.softmax(U, 1)
        for r in range(1, R + 1):
            z = U - ops.ecc_fwd(q, W, graph, C)
            q = torch.softmax(z, 1) if r < R else z
        return q

    def bwd_steps():
        torch.neg(g, out=gps[R - 1])
        du_in = g
        for r in range(R, 0, -1):
            ops.crf_bwd_step(W, gps[r - 1], qs[r - 1], du_in, gu, gps[r - 2] if r > 1 else None, graph)
            du_in = gu

    def bwd_w():
        ops.ecc_bwd_w(qs, gps, graph, (E, C, C), n_iter=R, out=gw)

    fwd()
    ref = composed()
    err = float((out - ref).abs().max() / ref.abs().max())

    def timed(fn):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)

    cases = dict(fwd=fwd, composed=composed, bwd_steps=bwd_steps, bwd_w=bwd_w)
    for fn in cases.values():  # warm-up of every timed shape
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in cases}
    for _ in range(reps):  # alternated in one loop: the same clocks and neighbours for every case
        for k, fn in cases.items():
            times[k].append(timed(fn))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    nb = iter_bytes(N, E, C) * R
    res = dict(size=label, nodes=N, edges=E, C=C, R=R, l2_flushed=flush is not None,
               max_rel_diff_fused_vs_composed=err)
    for k, ms in med.items():
        res["%s_ms" % k] = round(ms, 5)
    res["fwd_algorithmic_bytes"] = nb
    res["fwd_GBps"] = round(nb / (med["fwd"] * 1e-3) / 1e9, 1)
    res["fwd_share_of_hbm_peak"] = round(nb / (med["fwd"] * 1e-3) / HBM_PEAK, 3)
    res["composed_over_fused"] = round(med["composed"] / med["fwd"], 2)
    res["bwd_w_share_of_backward"] = round(med["bwd_w"] / (med["bwd_w"] + med["bwd_steps"]), 3)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--sweep-nodes", type=int, default=100000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_crf.py measures the sm_90a kernels and needs a CUDA device")
    from superpoint_graph_b200 import _lib
    from superpoint_graph_b200.synthetic import make_batch
    _lib.lib()
    dev = torch.device("cuda:0")
    line = dict(bench="ecc_crf", card=card(), hbm_peak_Bps=HBM_PEAK, bound="kernel-level HBM bound (bytes)")
    C, R = 13, 3
    small = make_batch(n_nodes=1024, seed=1)
    big = make_batch(n_nodes=args.sweep_nodes, seed=5, npts=1, minpts=1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    line["batch"] = run_size(dev, "configs[1]-sized batch, f_13,crf_3", small, C, R, args.reps, None)
    line["sweep"] = run_size(dev, "sweep, L2 flushed", big, C, R, args.reps, flush)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
