"""Recurrent LSTM-ECC timings (`lstm_*` model configs); prints one JSON line.

    python tools/bench_lstm.py [--reps 30]

H = 32, R = 10 recurrent steps, LSTMCellEx with layer norm and input gate, random vector filters [E, H] (the
filter network is not part of what is timed).  Two sizes:
  batch  configs[1]-sized: synthetic.make_batch, 1024 superpoints
  sweep  100 k superpoints, L2 flushed (256 MiB memset) before every timed launch group

Three paths, alternated in one loop so that they see the same clocks and neighbours, each forward and
backward (the backward up to the per-row parameter-gradient factors; the weight GEMMs and the filter
gradient are the same for every path and not timed):
  lstm_fused  the persistent R x {ECC, cell} kernels (spg_rnn_vv_lstm_fwd/bwd)
  lstm_steps  the per-step kernels: R x (ecc_fwd + lstm_fwd), R x (lstm_bwd + ecc_bwd_x)
  gru_fused   the GRU's persistent kernels at the same sizes (spg_rnn_vv_fwd/bwd)
CUDA events, after warm-up, median over `reps` repetitions.  The card's name, power limit and maximum SM
clock are read in the same run.

There is no CPU fallback: without a CUDA device the script exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, R = 32, 10


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def cell_weights(G, dev):
    torch.manual_seed(0)
    s = H ** -0.5
    w = [torch.empty(G * H, H, device=dev).uniform_(-s, s), torch.empty(G * H, H, device=dev).uniform_(-s, s),
         torch.empty(G * H, device=dev).uniform_(-s, s), torch.empty(G * H, device=dev).uniform_(-s, s),
         torch.empty(H, H, device=dev).uniform_(-s, s), torch.empty(H, device=dev).uniform_(-s, s)]
    return w


def run_size(dev, batch, reps, flush):
    from superpoint_graph_b200 import ops
    N, E = batch["degs"].numel(), batch["idxn"].numel()
    graph = ops.EccGraph(batch["idxn"], None, batch["degs"], n_in=N)
    graph.to(dev)
    flags = ops.GRU_LAYERNORM | ops.GRU_INGATE | ops.GRU_BIAS
    W = torch.randn(E, H, device=dev) * 0.5
    assert ops.rnn_vv_supported(W, graph, N, H)
    lw, gw = cell_weights(4, dev), cell_weights(3, dev)
    x0 = torch.randn(N, H, device=dev)
    gtop = torch.randn(N, H, device=dev)

    def buffers(G, lstm):
        hs = torch.empty((R + 1, N, H), device=dev)
        hs[0].copy_(x0)
        cs = torch.zeros((R + 1, N, H), device=dev) if lstm else None
        return dict(hs=hs, cs=cs, inps=torch.empty((R, N, H), device=dev),
                    d_gi=torch.empty((R, N, G * H), device=dev), d_gh=torch.empty((R, N, G * H), device=dev),
                    d_q=torch.empty((R, N, H), device=dev), xp=torch.empty((R, N, H), device=dev),
                    ginp=torch.empty((R, N, H), device=dev),
                    dpre=None if lstm else torch.empty((R, N, 4 * H), device=dev))

    bl, bs, bg = buffers(4, True), buffers(4, True), buffers(3, False)
    dc = torch.empty((N, H), device=dev)

    def lstm_fused_fwd():
        ops.rnn_vv_fwd(bl["hs"], bl["inps"], W, graph, lw, flags, cs=bl["cs"])

    def lstm_fused_bwd():
        ops.rnn_vv_bwd(bl["hs"], bl["inps"], W, graph, lw, flags, gtop, None, bl["ginp"], bl["d_gi"], bl["d_gh"],
                       bl["d_q"], bl["xp"], None, cs=bl["cs"])

    def lstm_steps_fwd():
        for r in range(R):
            inp = ops.ecc_fwd(bs["hs"][r], W, graph, H, out=bs["inps"][r])
            ops.lstm_fwd(inp, bs["hs"][r], bs["cs"][r], *lw, flags, out=bs["hs"][r + 1], out_c=bs["cs"][r + 1])

    def lstm_steps_bwd():
        gh = gtop
        for r in range(R - 1, -1, -1):
            d_h = ops.lstm_bwd(bs["inps"][r], bs["hs"][r], bs["cs"][r], gh, None if r == R - 1 else dc, *lw, flags,
                               bs["d_gi"][r], bs["d_gh"][r], bs["d_q"][r], bs["xp"][r], d_x=bs["ginp"][r],
                               d_c=dc)[1]
            gh = ops.ecc_bwd_x(W, bs["ginp"][r], graph, H, add0=d_h)

    def gru_fused_fwd():
        ops.rnn_vv_fwd(bg["hs"], bg["inps"], W, graph, gw, flags)

    def gru_fused_bwd():
        ops.rnn_vv_bwd(bg["hs"], bg["inps"], W, graph, gw, flags, gtop, None, bg["ginp"], bg["d_gi"], bg["d_gh"],
                       bg["d_q"], bg["xp"], bg["dpre"])

    cases = dict(lstm_fused_fwd=lstm_fused_fwd, lstm_steps_fwd=lstm_steps_fwd, gru_fused_fwd=gru_fused_fwd,
                 lstm_fused_bwd=lstm_fused_bwd, lstm_steps_bwd=lstm_steps_bwd, gru_fused_bwd=gru_fused_bwd)
    for fn in cases.values():  # warm-up of every timed shape
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    same = bool(torch.equal(bl["hs"], bs["hs"]) and torch.equal(bl["cs"], bs["cs"])
                and torch.equal(bl["d_gi"], bs["d_gi"]) and torch.equal(bl["ginp"], bs["ginp"]))

    def timed(fn):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e)

    times = {k: [] for k in cases}
    for _ in range(reps):
        for k, fn in cases.items():
            times[k].append(timed(fn))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = dict(nodes=N, edges=E, l2_flushed=flush is not None, fused_bit_identical_to_steps=same)
    res["ms"] = {k: round(ms, 4) for k, ms in med.items()}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--sweep-nodes", type=int, default=100000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lstm.py measures the sm_90a kernels and needs a CUDA device")
    from superpoint_graph_b200 import _lib
    from superpoint_graph_b200.synthetic import make_batch
    _lib.lib()
    dev = torch.device("cuda:0")
    line = dict(bench="rnn_ecc_lstm", H=H, R=R, card=card())
    small = make_batch(n_nodes=1024, seed=1)
    big = make_batch(n_nodes=args.sweep_nodes, seed=5, npts=1, minpts=1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    line["batch"] = run_size(dev, small, args.reps, None)
    line["sweep"] = run_size(dev, big, args.reps, flush)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
