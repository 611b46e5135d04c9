"""Learned-partition batch builder timings (graph_loader + graph_collate of supervized_partition); prints one JSON line.

    python tools/bench_partition_loader.py [--reps 15] [--sizes train,scene]

Synthetic files with spatially coherent vertex ids (points sorted along x, neighbour ids and 5 edges per vertex
within a window of the vertex order, as a kNN of a sorted cloud), 30-wide local_geometry, 14 label columns.
Two sizes:
  train  5 files of 10^5 vertices, max_ver_train 10^4 (a window of the vertex order as the sub-graph mask),
         k_nn_local 20, global_feat eXYrgb, use_rgb 1, rotation and jitter on
  scene  1 file of 10^6 vertices, evaluation (nothing augmented or sub-sampled), same features
Arms, the same masks given to both:
  host        oracle/partition_loader_ref.py (the reference's numpy loader and collate) on the host cores, then a
              pinned upload of the collated outputs; `host_ms` and `copy_ms` are reported separately
  device      superpoint_graph_b200.spg_partition_loader.load_batch from the resident store, host noise
  device_rng  the same with device_rng=True (the jitter normals drawn on the device)
Host clock around every arm, ending in a device synchronise; medians of `reps` alternated runs after warm-up.
`lp_local_clouds` is also timed alone (CUDA events, median of `reps`), with its algorithmic bytes over 3.35 TB/s.
`outputs_agree`: every output bit-identical for eval; for train, integer outputs identical and float outputs within
1 ulp (the rotation is BLAS's float32 matmul on the host).  The card's name, power limit and maximum SM clock are
read in the same run.  Without a CUDA device the script exits.
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

HBM_BYTES_PER_S = 3.35e12
K_GEOMETRY, N_LABELS = 30, 14


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def make_file(n, seed):
    """read_structure's tuple for a synthetic file of n vertices."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, [50, 10, 4], size=(n, 3)).astype(np.float32)
    xyz = xyz[np.argsort(xyz[:, 0], kind="stable")]
    v = np.arange(n)
    off = rng.integers(-40, 41, size=(n, K_GEOMETRY - 1))
    lg = np.concatenate([v[:, None], np.clip(v[:, None] + off, 0, n - 1)], 1).astype(np.uint32)
    src = np.repeat(v, 5)
    tgt = np.clip(src + rng.integers(1, 40, size=5 * n), 0, n - 1)
    obj = v // 800
    labels = np.zeros((n, N_LABELS), np.uint32)
    labels[v, 1 + obj % 13] = 1
    return (xyz, rng.integers(0, 256, size=(n, 3)).astype(np.float32), src, tgt,
            (obj[src] != obj[tgt]).astype(np.uint8), lg, labels, obj,
            ((xyz[:, 2] - 2) / 4).astype(np.float32), (xyz[:, :2] / 50).astype(np.float32))


def window_mask(n, m, seed):
    start = int(np.random.default_rng(seed).integers(0, n - m))
    mask = np.zeros(n, bool)
    mask[start:start + m] = True
    return mask


def sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def local_clouds_bytes(n_sel, k, use_rgb, G, C, subsampled):
    F = 3 + 3 * use_rgb
    read = n_sel * (k * 4 + k * 12 * (1 + use_rgb) + 12 + 12 * use_rgb + 4 + 8 + 4 * C + 4 + (4 if subsampled else 0))
    write = n_sel * (F * k * 4 + G * 4 + 12 + 8 * C + 8)
    return read + write


def ulps(a, b):
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def flat(batch):
    _, src, tgt, tr, labels, objects, (clouds, cglob, _), xyz = batch
    return [np.asarray(x.cpu().numpy() if torch.is_tensor(x) else x)
            for x in (src, tgt, tr, labels, objects, clouds, cglob, xyz)]


def run_size(name, n_files, n_ver, max_ver, train, reps, dev):
    from oracle import partition_loader_ref as lref
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_partition_loader import PartitionStore, global_columns, host_draws, load_batch
    args = SimpleNamespace(ver_value="ptn", k_nn_local=20, use_rgb=1, global_feat="eXYrgb", pc_augm_rot=int(train),
                           pc_augm_jitter=int(train), max_ver_train=max_ver)
    names = ["bench/f%d.h5" % i for i in range(n_files)]
    files = {nm: make_file(n_ver, i) for i, nm in enumerate(names)}
    masks = [window_mask(n_ver, max_ver, 100 + i) for i in range(n_files)] if (train and 0 < max_ver < n_ver) else None
    store = PartitionStore()
    for nm in names:
        store.add(nm, *files[nm])
    store.finalize(dev)
    seed = 7

    def host_arm():
        t0 = time.perf_counter()
        np.random.seed(seed)
        draws = [host_draws(n_ver, args, True) for _ in names] if train else None
        out = lref.load_batch(files, names, train, args, draws, masks)
        host_ms = 1e3 * (time.perf_counter() - t0)
        arrs = flat(out)
        pinned = [torch.from_numpy(np.ascontiguousarray(a.astype(np.int64) if a.dtype == np.uint32 else a)).pin_memory()
                  for a in arrs]
        copy_ms, dev_out = sync_ms(lambda: [p.to(dev, non_blocking=True) for p in pinned])
        return host_ms, copy_ms, arrs, sum(p.numel() * p.element_size() for p in pinned)

    def device_arm(rng_on):
        np.random.seed(seed)
        return sync_ms(lambda: load_batch(store, names, train, args, selected=masks, device_rng=rng_on, seed=seed))

    # warm-up, outputs
    h_ms, c_ms, host_out, host_bytes = host_arm()
    _, dev_batch = device_arm(False)
    device_arm(True)
    dev_out = flat(dev_batch)
    if train:
        ints_equal = all(np.array_equal(a.astype(np.int64), b.astype(np.int64)) for a, b in zip(host_out[:5], dev_out[:5]))
        max_ulp = int(max(ulps(a, b).max() for a, b in zip(host_out[5:], dev_out[5:])))
        agree = ints_equal and max_ulp <= 1
    else:
        agree = all(np.array_equal(a.view(np.uint8), b.astype(a.dtype).view(np.uint8))
                    for a, b in zip(host_out, dev_out))
        max_ulp = 0
    ms = {"host": [], "copy": [], "device": [], "device_rng": []}
    for _ in range(reps):
        h, c, _, _ = host_arm()
        ms["host"].append(h)
        ms["copy"].append(c)
        ms["device"].append(device_arm(False)[0])
        ms["device_rng"].append(device_arm(True)[0])
    N = dev_out[7].shape[0]
    n_tot = n_files * n_ver
    mask_bytes = n_tot if masks else 0
    dev_h2d = mask_bytes + (n_files * 9 * 4 if train else 0) + n_files * 8
    # lp_local_clouds alone, on the first file's kept vertices of the last batch layout
    f = store.file(names[0])
    gflags, G = global_columns(args.global_feat)
    n_sel = int(masks[0].sum()) if masks else n_ver
    sel = torch.from_numpy(np.nonzero(masks[0])[0].astype(np.int32)).to(dev) if masks else None
    out = [torch.empty((n_sel, 6, 20), dtype=torch.float32, device=dev),
           torch.empty((n_sel, G), dtype=torch.float32, device=dev), torch.empty((n_sel, 3), dtype=torch.float32, device=dev),
           torch.empty((n_sel, N_LABELS), dtype=torch.int64, device=dev), torch.empty(n_sel, dtype=torch.int64, device=dev)]
    off = torch.zeros(1, dtype=torch.int64, device=dev)

    def clouds_once():
        ops.lp_local_clouds(f["xyz"], f["rgb"], True, f["geometry"], 20, sel, n_sel, f["elevation"], f["xyn"],
                            f["labels"], f["objects"], off, True, gflags, *out)

    for _ in range(3):
        clouds_once()
    kt = []
    for _ in range(max(reps, 15)):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        clouds_once()
        e.record()
        e.synchronize()
        kt.append(s.elapsed_time(e))
    kb = local_clouds_bytes(n_sel, 20, 1, G, N_LABELS, masks is not None)
    k_ms = float(np.median(kt))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return dict(files=n_files, vertices_per_file=n_ver, max_ver_train=max_ver if train else None, train=train,
                batch_vertices=int(N), batch_edges=int(dev_out[0].shape[0]),
                host_ms=med["host"], copy_ms=med["copy"], host_total_ms=med["host"] + med["copy"],
                device_ms=med["device"], device_rng_ms=med["device_rng"],
                speedup_vs_host=(med["host"] + med["copy"]) / med["device"],
                h2d_bytes=dict(host=int(host_bytes), device=int(dev_h2d + (n_tot * 24 if train else 0)),
                               device_rng=int(dev_h2d)),
                lp_local_clouds=dict(rows=n_sel, ms=k_ms, bytes=int(kb),
                                     fraction_of_3_35_TBps=kb / HBM_BYTES_PER_S / (k_ms * 1e-3)),
                outputs_agree=bool(agree), max_float_ulp=max_ulp, host_threads=torch.get_num_threads())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=15)
    p.add_argument("--sizes", default="train,scene")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_partition_loader.py needs a CUDA device")
    dev = torch.device("cuda:0")
    from superpoint_graph_b200 import _lib
    _lib.lib()
    sizes = {"train": (5, 100000, 10000, True), "scene": (1, 1000000, 0, False)}
    res = {"bench": "learned_partition_batch_loader", "card": card(), "cpu": os.uname().machine,
           "nproc": os.cpu_count(), "reps": a.reps}
    for name in a.sizes.split(","):
        res[name] = run_size(name, *sizes[name], a.reps, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
