"""Times the superpoint graph's batch builder (spg_loader.load_batch) and prints one JSON line.

    python tools/bench_spg_batch.py [--reps 15] [--workloads s3dis_train,sema3d_eval]

Workloads:
  s3dis_train    synthetic rooms of 2 000 - 5 000 superpoints at ~10 edges per node, batch 2, nneigh 100, order 3,
                 hardcutoff 512, minpts 40, 14 point attributes, ptn_npts 128 (main.py's S3DIS defaults)
  sema3d_eval    one whole graph of 10^5 superpoints / 10^6 edges, train=False

For each: `load_batch` end to end (host draws and read-backs included, host clock around a synchronised call),
median of --reps runs after 3 warm-up runs; then, in a separate profiled run of --reps calls, the device part alone:
the mean per call of the GPU time of every kernel and copy torch.profiler records (CUDA activities), split into the
graph builder's own kernels (sb_select / sb_edges and the CUB scans and sorts they launch) and the rest (the clouds'
cloud_build, uploads, read-backs, collation copies).  With
SPG_REFERENCE set to a reference checkout, the reference's `loader` + `eccpc_collate` run on the host cores over
the compat igraph stand-in (compat/igraph.py: real igraph is not required) on the same graphs; without it that arm
is reported as "not measured".

Each workload also runs the `device_rng=True` arm (`seed` = the run's index), alternated run by run with the host
arm in the same timed loop.  Per arm: the end-to-end median, the profiled device time, the synchronising operations
torch reports under `torch.cuda.set_sync_debug_mode("warn")` in one call, and the time the arm spends formatting
`clouds_meta` from the kept ids (timed apart on the ids of one batch).  The host arm keeps the keys above; the
device arm's are under "device_rng".
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
import types
import warnings
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from superpoint_graph_b200 import spg_loader  # noqa: E402

ARGS = dict(spg_augm_nneigh=100, spg_augm_order=3, spg_augm_hardcutoff=512, ptn_minpts=40, ptn_npts=128,
            pc_attribs="xyzrgbelpsvXYZ", pc_xyznormalize=1, pc_augm_scale=0, pc_augm_rot=1, pc_augm_mirror_prob=0,
            pc_augm_jitter=1)


def make_graph(rng, n, deg):
    """Random geometric-ish graph: each vertex linked to `deg` / 2 random near ids, both directions."""
    half = max(deg // 2, 1)
    src = np.repeat(np.arange(n), half)
    dst = (src + rng.integers(1, 50, size=src.size)) % n
    edges = np.concatenate([np.stack([src, dst], 1), np.stack([dst, src], 1)])
    counts = np.clip(rng.lognormal(np.log(120.0), 1.0, size=n), 5, 2000).astype(np.int64)
    node_gt_size = np.zeros((n, 14), np.int64)
    node_gt_size[np.arange(n), 1 + rng.integers(0, 13, size=n)] = counts
    node_gt = np.argmax(node_gt_size[:, 1:], 1)[:, None]
    feats = rng.standard_normal((edges.shape[0], 13)).astype(np.float32)
    return node_gt, node_gt_size, edges, feats, counts


def clouds_for(rng, counts, cap):
    return {i: rng.standard_normal((int(min(c, cap)), 14)).astype(np.float32) for i, c in enumerate(counts)}


def call(gs, cs, names, train, args, r, device_rng):
    if device_rng:
        return spg_loader.load_batch(gs, cs, names, train, args, device_rng=True, seed=r)
    random.seed(r)
    np.random.seed(r)
    return spg_loader.load_batch(gs, cs, names, train, args)


def time_product(gs, cs, names, train, args, reps):
    """End-to-end medians (host arm, device_rng arm), the arms alternated run by run."""
    ends = {False: [], True: []}
    for r in range(reps + 3):
        for device_rng in (False, True):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call(gs, cs, names, train, args, r, device_rng)
            torch.cuda.synchronize()
            if r >= 3:
                ends[device_rng].append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ends[False])), float(np.median(ends[True]))


def sync_count(gs, cs, names, train, args, device_rng):
    """Synchronising operations torch reports in one call (after one unreported call)."""
    call(gs, cs, names, train, args, 0, device_rng)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            call(gs, cs, names, train, args, 1, device_rng)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchronizing" in str(w.message) for w in caught)


def meta_time(gs, cs, names, train, args, device_rng, reps=5):
    """ms to format one batch's clouds_meta from its kept ids, as the arm's load_batch does."""
    meta = call(gs, cs, names, train, args, 0, device_rng)[2][0]
    ids = {}
    for m in meta:
        nm, v = m.rsplit(".", 1)
        ids.setdefault(nm, []).append(int(v))
    kept = [(nm, np.array(v, np.int32) if device_rng else v) for nm, v in ids.items()]
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        if device_rng:
            [nm + "." + str(v) for nm, vv in kept for v in vv.tolist()]
        else:
            ["{}.{:d}".format(nm, v) for nm, vv in kept for v in vv]
        out.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(out))


def device_time(gs, cs, names, train, args, reps, device_rng=False):
    """(all device ms, graph-builder kernel ms) per call, means over `reps` profiled calls."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(reps):
            call(gs, cs, names, train, args, r, device_rng)
        torch.cuda.synchronize()
    total = graph = 0.0
    for ev in prof.key_averages():
        us = ev.self_device_time_total
        total += us
        if "sb_" in ev.key or "cub" in ev.key.lower():
            graph += us
    return total / 1e3 / reps, graph / 1e3 / reps


def time_reference(graphs, clouds, names, train, args, reps):
    ref = os.environ.get("SPG_REFERENCE")
    if not ref:
        return "not measured"
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden_spg_batch as mg  # the reference's source text on the compat stand-ins

    ns = mg.reference_namespace()

    class _File(object):  # parsed clouds served from memory (no file reads timed)
        def __init__(self, path, mode="r"):
            self._c = clouds_by_path[path]

        def __getitem__(self, key):
            return self._c[int(key)]

    clouds_by_path = {"/db/parsed/%s.h5" % nm: clouds[nm] for nm in names}
    ns["h5py"] = types.SimpleNamespace(File=_File)
    a = SimpleNamespace(**args.__dict__)
    out = []
    for r in range(reps + 1):
        random.seed(r)
        np.random.seed(r)
        entries = [ns["spg_to_igraph"](*graphs[nm], nm) for nm in names]
        t0 = time.perf_counter()
        ns["eccpc_collate"]([ns["loader"](e, train, a, "/db", 0) for e in entries])
        if r >= 1:
            out.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(out))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--workloads", default="s3dis_train,sema3d_eval")
    opt = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spg_batch needs a CUDA device")
    rng = np.random.default_rng(0)
    result = {"gpu": gpu_info(), "reps": opt.reps}
    workloads = [("s3dis_train", [int(rng.integers(2000, 5001)) for _ in range(2)], 10, True, 256),
                 ("sema3d_eval", [100_000], 10, False, 48)]
    for tag, sizes, deg, train, cap in workloads:
        if tag not in opt.workloads.split(","):
            result[tag] = "not measured"
            continue
        args = SimpleNamespace(**ARGS)
        gs, cs = spg_loader.GraphStore(), spg_loader.SuperpointStore()
        graphs, clouds, names = {}, {}, []
        for b, n in enumerate(sizes):
            nm = "%s_%d" % (tag, b)
            node_gt, node_gt_size, edges, feats, counts = make_graph(rng, n, deg)
            graphs[nm] = (node_gt, node_gt_size, edges, feats)
            clouds[nm] = clouds_for(rng, counts, cap)
            gs.add(node_gt, node_gt_size, edges, feats, nm)
            cs.add(nm, clouds[nm])
            names.append(nm)
        gs.finalize("cuda")
        cs.finalize("cuda")
        end, end_rng = time_product(gs, cs, names, train, args, opt.reps)
        dev_all, dev_graph = device_time(gs, cs, names, train, args, opt.reps)
        rng_all, rng_graph = device_time(gs, cs, names, train, args, opt.reps, device_rng=True)
        result[tag] = {"vertices": sizes, "edges": [int(graphs[nm][2].shape[0]) for nm in names],
                       "load_batch_ms": round(end, 3), "device_ms": round(dev_all, 4),
                       "device_graph_kernels_ms": round(dev_graph, 4),
                       "reference_host_compat_igraph_ms": time_reference(graphs, clouds, names, train, args,
                                                                          opt.reps),
                       "syncs": sync_count(gs, cs, names, train, args, False),
                       "clouds_meta_ms": round(meta_time(gs, cs, names, train, args, False), 3),
                       "device_rng": {"load_batch_ms": round(end_rng, 3), "device_ms": round(rng_all, 4),
                                      "device_graph_kernels_ms": round(rng_graph, 4),
                                      "syncs": sync_count(gs, cs, names, train, args, True),
                                      "clouds_meta_ms": round(meta_time(gs, cs, names, train, args, True), 3)}}
        print(json.dumps({tag: result[tag]}), file=sys.stderr, flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
