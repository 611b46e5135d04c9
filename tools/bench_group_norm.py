"""GroupNorm PointNet timings (norm='layer' | 'group'); prints one JSON line.

    python tools/bench_group_norm.py [--clouds 150000] [--reps 15]

Workload: the learned-partition LocalCloudEmbedder (supervized_partition.py defaults): external STN
[[16, 64], [32, 16]] on the first 2 of 6 features, PointNet [[32, 128], [34, 32, 32, 4]] with the 11 global
features + the flattened transform, 20 points per cloud, prelast_do 0; norm in {batch, layer, group (2)}.
  train  one training step of the embedder: forward and backward from a fixed output gradient
  eval   one eval-mode forward
Two paths per norm, alternated in one loop so that they see the same clocks and neighbours:
  ours   the modules of this package (CUDA kernels through the C-ABI)
  torch  the same nn.Sequential containers run eagerly by torch (cuDNN conv1d, F.group_norm or batch_norm,
         ReLU, max_pool1d), i.e. the reference's composition
CUDA events, after warm-up, median over `reps` repetitions.

Kernel times: one profiled training step of `ours` per GroupNorm norm in a separate pass (ops.prof_enable),
summed over the launches of gn_fwd, gn_bwd and gn_bwd_final.  Achieved bytes/s use the bytes the algorithm
has to move, computed below from the layer shapes: the forward reads y and writes the activation (2 x 4 B per
element), the backward reads G and y and writes dY (3 x 4 B); the kernels' re-reads of a segment from L1/L2
are not counted.  Against the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s.  The card's name, power limit
and maximum SM clock are read in the same run.

There is no CPU fallback: without a CUDA device the script exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

L, NFEAT, NGLOB = 20, 6, 11
STN_W = ([16, 64], [32, 16])
PTN_W = ([32, 128], [34, 32, 32, 4])
HBM_BPS = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def models(norm, dev):
    from superpoint_graph_b200.spg_pointnet import PointNet, STNkD
    torch.manual_seed(0)
    m = torch.nn.Module()
    m.stn = STNkD(2, STN_W[0], STN_W[1], norm=norm, n_group=2)
    m.ptn = PointNet(PTN_W[0], PTN_W[1], [], [], NFEAT, 0, prelast_do=0, nfeat_global=NGLOB + 4, norm=norm, n_group=2)
    with torch.no_grad():
        m.stn.proj.weight.normal_(0, 0.1)
    return m.to(dev)


def eager(m, clouds, glob):
    """LocalCloudEmbedder.run_batch on torch's own modules (learning/pointnet.py:55-61,120-133,195-207)."""
    stn, ptn = m.stn, m.ptn
    h = stn.convs(clouds[:, :2, :])
    h = stn.fcs(F.max_pool1d(h, h.size(2)).squeeze(2))
    T = stn.proj(h).view(-1, 2, 2) + torch.eye(2, device=clouds.device).unsqueeze(0)
    xy = torch.bmm(clouds[:, :2, :].transpose(1, 2), T).transpose(1, 2)
    x = ptn.convs(torch.cat([xy, clouds[:, 2:, :]], 1))
    x = torch.cat([F.max_pool1d(x, x.size(2)).squeeze(2), glob, T.view(-1, 4)], 1)
    return F.normalize(ptn.fcs(x))


def gn_bytes(B):
    """(forward, backward) bytes the GroupNorm layers of one training step have to move."""
    elems = sum(B * L * c for c in STN_W[0] + PTN_W[0]) + sum(B * c for c in STN_W[1] + PTN_W[1][:-1])
    return 2 * 4 * elems, 3 * 4 * elems


def timed(fn, reps_out, start, end):
    start.record()
    fn()
    end.record()
    end.synchronize()
    reps_out.append(start.elapsed_time(end))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=150000)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_group_norm needs a CUDA device")
    from superpoint_graph_b200 import _lib, ops
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder
    _lib.lib()
    dev = torch.device("cuda:0")
    B = args.clouds
    torch.manual_seed(1)
    clouds = torch.randn(B, NFEAT, L, device=dev) * 0.5
    glob = torch.randn(B, NGLOB, device=dev)
    gy = torch.randn(B, 4, device=dev)
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    norms = ["batch", "layer", "group"]
    ms = {n: models(n, dev) for n in norms}

    def train(path, n):
        m = ms[n]
        m.train()
        out = emb.run_batch(m, clouds, glob) if path == "ours" else eager(m, clouds, glob)
        out.backward(gy)
        m.zero_grad(set_to_none=True)

    def evaluate(path, n):
        m = ms[n]
        m.eval()
        with torch.no_grad():
            emb.run_batch(m, clouds, glob) if path == "ours" else eager(m, clouds, glob)

    cases = [(mode, path, n) for n in norms for mode in ("train", "eval") for path in ("ours", "torch")]
    fns = {"train": train, "eval": evaluate}
    for mode, path, n in cases:  # warm-up: module loads, cuDNN algorithm choice, allocator
        for _ in range(2):
            fns[mode](path, n)
    torch.cuda.synchronize()
    times = {c: [] for c in cases}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.reps):
        for c in cases:
            mode, path, n = c
            timed(lambda: fns[mode](path, n), times[c], start, end)

    def med(v):
        v = sorted(v)
        return v[len(v) // 2]

    res = {"card": card(), "clouds": B, "points": L, "reps": args.reps, "ms": {}}
    for mode, path, n in cases:
        res["ms"]["%s/%s/%s" % (n, mode, path)] = round(med(times[(mode, path, n)]), 3)
    # per-kernel times of the GroupNorm passes, profiled in a pass of their own
    fwd_b, bwd_b = gn_bytes(B)
    res["kernels"] = {}
    for n in ("layer", "group"):
        torch.cuda.synchronize()
        ops.prof_enable(1)
        ops.prof_reset()
        train("ours", n)
        torch.cuda.synchronize()
        k = ops.prof_collect()
        ops.prof_enable(0)
        f_ms = k["gn_fwd"][1]
        b_ms = k["gn_bwd"][1] + k.get("gn_bwd_final", (0, 0.0))[1]
        res["kernels"][n] = {
            "gn_fwd_ms": round(f_ms, 3), "gn_fwd_launches": k["gn_fwd"][0], "gn_fwd_bytes": fwd_b,
            "gn_fwd_GBps": round(fwd_b / f_ms / 1e6, 1), "gn_fwd_of_hbm": round(fwd_b * 1e3 / f_ms / HBM_BPS, 3),
            "gn_bwd_ms": round(b_ms, 3), "gn_bwd_launches": k["gn_bwd"][0], "gn_bwd_bytes": bwd_b,
            "gn_bwd_GBps": round(bwd_b / b_ms / 1e6, 1), "gn_bwd_of_hbm": round(bwd_b * 1e3 / b_ms / HBM_BPS, 3),
            "step_total_ms_profiled": round(sum(v[1] for v in k.values()), 3),
        }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
