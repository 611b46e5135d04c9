"""Weight-gradient GEMM timings (`ops.tc_dw`: tc_dw_kernel + split-K reduce) per layer shape; prints one JSON line.

    python tools/bench_tc_dw.py [--reps 25] [--save DIR | --compare DIR] [--lib PATH]

Shapes (CO, CI): the eight point-wise layers of the flagship batch (main 32->64->64->128->128->256, STN
32->64->64->128) and the vKITTI widths ptn_widths=[[64,64,128],[64,32,32]] that the wgmma kernel takes.  Two
row counts: M = 120 576 (942 clouds of 128 points, the flagship batch) and M = 1 280 000 (sweep-sized).  P goes
through the fused affine + ReLU prologue, as in the training step.

Every timed launch follows a 256 MiB memset that flushes L2; CUDA events, median over `reps` after warm-up.
Reported per shape: ms, algorithmic bytes 4*M*(CO+CI), GB/s and the fraction of the H100 SXM data-sheet
3.35 TB/s.  The card's name, power limit and maximum SM clock are read in the same run.

--save DIR writes each shape's dW for seeded inputs, --compare DIR checks a later build against them with
torch.equal (the kernel's results must not depend on how it moves its bytes).  --lib PATH times another
build of libspg_b200.so.

There is no CPU fallback: without a CUDA device the script exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FLAGSHIP = [(64, 32), (64, 64), (128, 64), (128, 128), (256, 128), (64, 32), (64, 64), (128, 64)]
VKITTI = [(64, 32), (64, 64), (128, 64)]  # [64,64,128] and the STN's 32->64 on a 32-padded input
ROWS = (120576, 1280000)
HBM_BYTES_PER_S = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def inputs(M, co, ci, dev):
    g = torch.Generator(device=dev).manual_seed(1000003 * co + 1009 * ci + M % 997)
    dY = torch.randn(M, co, device=dev, generator=g)
    P = torch.randn(M, ci, device=dev, generator=g) * 1.3 + 0.2
    scale = torch.rand(ci, device=dev, generator=g) + 0.5
    shift = torch.randn(ci, device=dev, generator=g)
    return dY, P, (scale, shift, True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--save", metavar="DIR")
    ap.add_argument("--compare", metavar="DIR")
    ap.add_argument("--lib", metavar="PATH")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tc_dw.py measures the sm_90a kernels and needs a CUDA device")
    from superpoint_graph_b200 import _lib, ops
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    _lib.lib()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    if args.save:
        os.makedirs(args.save, exist_ok=True)
    line = dict(bench="tc_dw", lib=_lib.LIB_PATH, card=card(), reps=args.reps, l2_flushed=True, rows={})
    mismatches = []
    for M in ROWS:
        shapes, total = {}, 0.0
        for co, ci in sorted(set(FLAGSHIP + VKITTI)):
            dY, P, aff = inputs(M, co, ci, dev)
            assert ops.tc_dw_supported(M, co, ci, co, ci)

            def run():
                return ops.tc_dw(dY, co, P, ci, M, co, ci, p_aff=aff)

            for _ in range(3):
                dW = run()
            torch.cuda.synchronize()
            name = "dw_M%d_CO%d_CI%d.pt" % (M, co, ci)
            if args.save:
                torch.save(dW.cpu(), os.path.join(args.save, name))
            if args.compare and not torch.equal(dW.cpu(), torch.load(os.path.join(args.compare, name))):
                mismatches.append(name)
            times = []
            for _ in range(args.reps):
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                run()
                e.record()
                e.synchronize()
                times.append(s.elapsed_time(e))
            ms = sorted(times)[len(times) // 2]
            nbytes = 4 * M * (co + ci)
            shapes["%dx%d" % (co, ci)] = dict(ms=round(ms, 4), bytes=nbytes, gb_per_s=round(nbytes / ms / 1e6, 1),
                                              frac_of_3350_gb_per_s=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
            total += ms * FLAGSHIP.count((co, ci))
        line["rows"][str(M)] = dict(shapes=shapes, flagship_eight_layers_ms=round(total, 4))
    if args.compare:
        line["bit_identical_to_saved"] = not mismatches
    print(json.dumps(line))
    if mismatches:
        sys.exit("dW differs from the saved outputs: " + ", ".join(mismatches))


if __name__ == "__main__":
    main()
