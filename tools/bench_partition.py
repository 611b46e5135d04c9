"""Learned-partition objective timings (supervized_partition.py:220-230 after the embedding); prints one JSON line.

    python tools/bench_partition.py [--reps 15] [--cpu-reps 1] [--cpu-full]

Workload: embeddings [V, 4] (the --ptn_widths default), k_nn_adj 5 edges per vertex, TVH_zhang, euclidian,
crosspartition weights with transition_factor 5 (the supervized_partition.py defaults), a given predicted
partition (cut pursuit stays on the host and is not timed).  Two sizes:
  train  5 x 10^4 vertices, 2.5 x 10^5 edges (batch 5 x --max_ver_train 1e4)
  scene  10^6 vertices, 5 x 10^6 edges (one full-scene evaluation)
Arms, each one objective: distances, weights, loss, backward to the embeddings:
  device  superpoint_graph_b200.spg_partition (csrc/partition.cu), inputs on the device
  torch   the reference's distance and loss in eager torch on the GPU, with the weights from the ported host
          code (oracle/partition_ref.py's loop-free restatement, computed once and not timed; `host_weights_ms` is
          its time, `weights_equal` says whether the device weights are bit-identical to them)
  host    the oracle's port of the reference path on the host cores (torch CPU distance/loss/backward, the
          reference's per-pair crosspartition loop); `--cpu-reps` runs at the train size, at the scene size
          only with --cpu-full (the loop is O(component pairs x transition edges))
Device arms: CUDA events around the whole objective after warm-up, median of `reps` alternated runs.  The card's
name, power limit and maximum SM clock are read in the same run.  Without a CUDA device the script exits.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARGS = SimpleNamespace(loss_weight="crosspartition", loss="TVH_zhang", dist_type="euclidian", transition_factor=5.0,
                       k_nn_adj=5, edge_weight_threshold=-0.5, spatial_emb=0, cuda=1)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def make_batch(V, k, seed):
    """k neighbours per vertex within a window of the vertex order (spatially coherent ids, as a kNN graph of a
    sorted cloud); objects as runs of ~800 vertices with 2 % label noise; predicted components as runs of ~37."""
    g = torch.Generator().manual_seed(seed)
    src = torch.arange(V).repeat_interleave(k)
    tgt = (src + torch.randint(1, 40, (V * k,), generator=g)) % V
    obj = torch.div(torch.arange(V), 800, rounding_mode="floor")
    obj = obj ^ (torch.rand(V, generator=g) < 0.02).long()
    pic = torch.div(torch.arange(V) + torch.randint(0, 3, (V,), generator=g), 37, rounding_mode="floor")
    is_tr = (obj[src] != obj[tgt]).to(torch.uint8)
    emb = torch.nn.functional.normalize(torch.randn(V, 4, generator=g))
    return dict(src=src, tgt=tgt, obj=obj, pic=pic, is_tr=is_tr, emb=emb)


def device_step(b):
    from superpoint_graph_b200 import spg_partition as sp
    emb = b["emb_d"].detach().requires_grad_(True)
    diff = sp.compute_dist(emb, b["src_d"], b["tgt_d"], ARGS.dist_type)
    w = sp.compute_weight_loss(ARGS, emb, b["obj_d"], b["src_d"], b["tgt_d"], b["is_tr_d"], diff, False,
                               partition=(None, b["pic_d"]))
    l1, l2 = sp.compute_loss(ARGS, diff, b["is_tr_d"], w)
    ((l1 + l2) / w.shape[0] * 1000).backward()
    return emb.grad


def torch_step(b, ref, emb0, src, tgt, is_tr, w):
    emb = emb0.detach().requires_grad_(True)
    l1, l2 = ref.compute_loss(ARGS, ref.compute_dist(emb, src, tgt, ARGS.dist_type), is_tr, w)
    ((l1 + l2) / w.shape[0] * 1000).backward()
    return emb.grad


def host_step(b, ref):
    emb = b["emb"].clone().requires_grad_(True)
    s, t = b["src"].numpy(), b["tgt"].numpy()
    diff = ref.compute_dist(emb, s, t, ARGS.dist_type)
    w = ref.compute_weights_XPART(None, b["pic"].numpy(), None, s, t, b["is_tr"].numpy(),
                                  ARGS.transition_factor * 2 * ARGS.k_nn_adj)
    l1, l2 = ref.compute_loss(ARGS, diff, b["is_tr"], torch.from_numpy(w))
    ((l1 + l2) / len(w) * 1000).backward()
    return w


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def run_size(name, V, k, reps, cpu_reps, dev):
    from oracle import partition_ref as ref
    b = make_batch(V, k, seed=V)
    for key in ("src", "tgt", "obj", "pic", "is_tr", "emb"):
        b[key + "_d"] = b[key].to(dev)
    ref.xpart_components(b["pic"].numpy()[:100], b["src"].numpy()[:0], b["tgt"].numpy()[:0], b["is_tr"].numpy()[:0])
    t0 = time.perf_counter()
    w_host = ref.compute_weights_XPART_sorted(b["pic"].numpy(), b["src"].numpy(), b["tgt"].numpy(),
                                              b["is_tr"].numpy(), ARGS.transition_factor * 2 * ARGS.k_nn_adj)
    host_weights_ms = 1e3 * (time.perf_counter() - t0)
    w_d = torch.from_numpy(w_host).to(dev)
    targs = (b, ref, b["emb_d"], b["src_d"], b["tgt_d"], b["is_tr_d"], w_d)
    from superpoint_graph_b200 import spg_partition as sp
    w_dev = sp.compute_weights_XPART(None, b["pic_d"], None, b["src_d"], b["tgt_d"], b["is_tr_d"],
                                     ARGS.transition_factor * 2 * ARGS.k_nn_adj)
    weights_equal = bool(np.array_equal(w_dev.cpu().numpy(), w_host))
    g1 = device_step(b)
    g2 = device_step(b)
    gt = torch_step(*targs)
    torch.cuda.synchronize()
    for _ in range(3):
        device_step(b)
        torch_step(*targs)
    ms = {"device": [], "torch": []}
    for _ in range(reps):
        ms["device"].append(timed(lambda: device_step(b), reps))
        ms["torch"].append(timed(lambda: torch_step(*targs), reps))
    out = dict(vertices=V, edges=int(b["src"].numel()), transitions=int(b["is_tr"].sum()),
               device_ms=float(np.median(ms["device"])), torch_gpu_ms=float(np.median(ms["torch"])),
               host_weights_ms=host_weights_ms, weights_equal=weights_equal, bit_identical_repeat=bool(torch.equal(g1, g2)),
               grad_rel_err_vs_torch=float((g1 - gt).abs().max() / gt.abs().max()))
    if cpu_reps > 0:
        times = []
        for _ in range(cpu_reps):
            t0 = time.perf_counter()
            w_loop = host_step(b, ref)
            times.append(1e3 * (time.perf_counter() - t0))
        out["weights_equal"] = out["weights_equal"] and bool(np.array_equal(w_loop, w_host))
        out["host_ms"] = float(np.median(times))
        out["host_threads"] = torch.get_num_threads()
        out["speedup_vs_host"] = out["host_ms"] / out["device_ms"]
    else:
        out["host_ms"] = "not run"
    out["speedup_vs_torch_gpu"] = out["torch_gpu_ms"] / out["device_ms"]
    return name, out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=15)
    p.add_argument("--cpu-reps", type=int, default=1)
    p.add_argument("--cpu-full", action="store_true", help="also run the host arm at the scene size")
    p.add_argument("--sizes", default="train,scene")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_partition.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from superpoint_graph_b200 import _lib
    _lib.lib()
    sizes = {"train": (50000, 5), "scene": (1000000, 5)}
    res = {"bench": "learned_partition_objective", "card": card(), "loss": ARGS.loss, "dist_type": ARGS.dist_type,
           "loss_weight": ARGS.loss_weight, "cpu": os.uname().machine, "nproc": os.cpu_count()}
    for name in a.sizes.split(","):
        V, k = sizes[name]
        cpu_reps = a.cpu_reps if (name == "train" or a.cpu_full) else 0
        res[name] = run_size(name, V, k, a.reps, cpu_reps, dev)[1]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
