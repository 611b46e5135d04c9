"""Point-wise GEMM timings (`ops.tc_gemm`: tc_gemm2_kernel + tc_merge_kernel) for the 14 launches of the flagship
training step, each with the prologue and epilogue the step gives it; prints one JSON line.

    python tools/bench_tc_gemm.py [--reps 25] [--save DIR | --compare DIR] [--lib PATH]

Cases, as chain_forward / chain_backward issue them (tc_gemm's (K, N): K = reduction, N = outputs):
  forward, AFFINE prologue (BatchNorm apply + ReLU of the layer below; none on a first layer), STATS epilogue with
      the BatchNorm fold: main PointNet (32,64) (64,64) (64,128) (128,128) (128,256), STN (32,64) (64,64) (64,128);
  data gradient, BNRED epilogue (the layer below has BatchNorm), and either the BNBWD prologue with the dY side
      store (the step's lazy path) or a plain A (the last conv layer, whose dY the max-pool backward produced):
      main 256->128 (plain), 128->128, 128->64, 64->64, STN 128->64 (plain), 64->64.
Two row counts: M = 120 576 (the flagship batch) and M = 1 280 000.  Inputs are seeded; BatchNorm inputs follow
tests/test_tc_gemm.py::bn_inputs, built on the device.

Every timed launch follows a 256 MiB memset that flushes L2; CUDA events around kernel + merge, median over
`reps` after warm-up.  Reported per case: ms, algorithmic bytes (A [+ A2, dY store] + C [+ e_y]), their fraction
of the H100 SXM data-sheet 3.35 TB/s, the 3xTF32 FLOP time at the data-sheet 495 TFLOP/s (3 MMAs per product),
the selection (NS, A-ring stages, N-slices), and a twin of the same launch with no fused reduction (EPI_NONE):
the gap between the two is what the fused reductions cost.  The card's name, power limit and maximum SM clock
are read in the same run.

--save DIR writes every output of every case (C, mean, var, scale, shift, running mean/var, num_batches_tracked,
dY, s12), --compare DIR checks a later build against them with torch.equal.  --lib PATH times another build of
libspg_b200.so.

There is no CPU fallback: without a CUDA device the script exits with an error.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_tc_gemm import ref_bn_sums, selection  # noqa: E402

# (name, K, N, prologue, epilogue): prologue "none" | "affine" (BN apply + ReLU) | "bnbwd" (with dY) | "plain"
FWD = [("fwd_main_%dx%d" % kn, kn[0], kn[1], "none" if kn[0] == 32 else "affine", "stats")
       for kn in [(32, 64), (64, 64), (64, 128), (128, 128), (128, 256)]] + \
      [("fwd_stn_%dx%d" % kn, kn[0], kn[1], "none" if kn[0] == 32 else "affine", "stats")
       for kn in [(32, 64), (64, 64), (64, 128)]]
BWD = [("dx_main_256to128", 256, 128, "plain", "bnred"), ("dx_main_128to128", 128, 128, "bnbwd", "bnred"),
       ("dx_main_128to64", 128, 64, "bnbwd", "bnred"), ("dx_main_64to64", 64, 64, "bnbwd", "bnred"),
       ("dx_stn_128to64", 128, 64, "plain", "bnred"), ("dx_stn_64to64", 64, 64, "bnbwd", "bnred")]
CASES = FWD + BWD
ROWS = (120576, 1280000)
HBM_BYTES_PER_S = 3.35e12
TF32_FLOP_PER_S = 495e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def bn_inputs(g, M, C, dev, relu=True):
    """tests/test_tc_gemm.py::bn_inputs on the device: a BatchNorm+ReLU layer's raw output Y with its batch
    statistics and fold, no |Y*scale + shift| within 1e-3 of zero."""
    eps = 1e-5
    Y = torch.randn(M, C, device=dev, generator=g) * 1.5 + 0.7
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    gamma[::3] *= -1
    beta = torch.randn(C, device=dev, generator=g) * 0.5
    mean, var = Y.double().mean(0).float(), Y.double().var(0, unbiased=False).float()
    scale = (gamma.double() / torch.sqrt(var.double() + eps)).float()
    shift = (beta.double() - mean.double() * scale.double()).float()
    z = Y.double() * scale.double() + shift.double()
    znew = torch.where(z >= 0, 4e-3, -4e-3).double()
    Y = torch.where(z.abs() < 2e-3, ((znew - shift.double()) / scale.double()).float(), Y)
    del z, znew
    return dict(Y=Y, scale=scale, shift=shift, mean=mean, var=var, eps=eps, relu=relu)


def case_inputs(M, name, K, N, pro, epi, dev):
    """Seeded inputs of one case -> (A, W, call kwargs, fresh-state function for the fold's running stats)."""
    g = torch.Generator(device=dev).manual_seed(1000003 * N + 1009 * K + M % 997 + (7 if epi == "bnred" else 0))
    kw, state = {}, None
    if epi == "stats":
        W = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
        kw["bias"] = torch.randn(N, device=dev, generator=g)
        if pro == "affine":
            lo = bn_inputs(g, M, K, dev)
            A = lo["Y"]
            kw["a_aff"] = (lo["scale"], lo["shift"], True)
        else:
            A = torch.randn(M, K, device=dev, generator=g)
        gamma = torch.rand(N, device=dev, generator=g) + 0.5
        beta = torch.randn(N, device=dev, generator=g)
        rm0, rv0 = torch.randn(N, device=dev, generator=g), torch.rand(N, device=dev, generator=g) + 0.5

        def state():
            rm, rv, nbt = rm0.clone(), rv0.clone(), torch.full((), 5, dtype=torch.long, device=dev)
            kw["stats"] = True
            kw["fold"] = (gamma, beta, 1e-5, rm, rv, nbt, 0.1)
            return rm, rv, nbt
        return A, W, kw, state, True
    # data gradient of a layer W [K, N] (K = its outputs): B = W^T
    W = torch.randn(K, N, device=dev, generator=g) / K ** 0.5
    G = torch.randn(M, K, device=dev, generator=g)
    if pro == "bnbwd":
        top = bn_inputs(g, M, K, dev)
        s12 = ref_bn_sums(G.double(), *(top[k].double() for k in ("Y", "scale", "shift", "mean", "var")),
                          top["eps"], True).float()
        kw["bnbwd"] = (top["Y"], K, top["scale"], top["shift"], True, top["mean"], top["var"], s12, top["eps"],
                       True)
    low = bn_inputs(g, M, N, dev)
    kw["bnred"] = (low["Y"], N, low["scale"], low["shift"], low["mean"], low["var"], low["eps"], True)
    return G, W, kw, None, False


def algorithmic_bytes(M, K, N, pro, epi):
    n = M * (K + N)  # A, C
    if pro == "bnbwd":
        n += 2 * M * K  # A2 (the layer's raw output), dY side store
    if epi == "bnred":
        n += M * N  # e_y (the layer below's raw output)
    return 4 * n


def output_names(epi, pro):
    if epi == "stats":
        return ["C", "mean", "var", "scale", "shift", "running_mean", "running_var", "num_batches_tracked"]
    return ["C"] + (["dY"] if pro == "bnbwd" else []) + ["s12"]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--save", metavar="DIR")
    ap.add_argument("--compare", metavar="DIR")
    ap.add_argument("--lib", metavar="PATH")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tc_gemm.py measures the sm_90a kernels and needs a CUDA device")
    from superpoint_graph_b200 import _lib, ops
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    _lib.lib()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    if args.save:
        os.makedirs(args.save, exist_ok=True)
    line = dict(bench="tc_gemm", lib=_lib.LIB_PATH, card=card(), reps=args.reps, l2_flushed=True, rows={})
    mismatches = []

    def timed(run):
        for _ in range(3):
            run()
        times = []
        for _ in range(args.reps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run()
            e.record()
            e.synchronize()
            times.append(s.elapsed_time(e))
        return sorted(times)[len(times) // 2]

    for M in ROWS:
        cases, total, total_none = {}, 0.0, 0.0
        for name, K, N, pro, epi in CASES:
            ops.PACK_CACHE.clear()
            A, W, kw, state, fwd = case_inputs(M, name, K, N, pro, epi, dev)
            assert ops.tc_supported(M, N, K, K, N)
            ldw, tr = (K, False) if fwd else (N, True)
            extra = state() if state else ()

            def run(kw=kw):
                return ops.tc_gemm(A, K, W, ldw, tr, M, N, K, **kw)

            outs = run()
            outs = (list(outs) if isinstance(outs, tuple) else [outs]) + list(extra)
            torch.cuda.synchronize()
            for oname, t in zip(output_names(epi, pro), outs):
                fname = "M%d_%s_%s.pt" % (M, name, oname)
                if args.save:
                    torch.save(t.cpu(), os.path.join(args.save, fname))
                if args.compare and not torch.equal(t.cpu(), torch.load(os.path.join(args.compare, fname))):
                    mismatches.append(fname)
            del outs
            ms = timed(run)
            # diagnostic twin: the same launch without the fused column reduction (EPI_NONE)
            kw_none = {k: v for k, v in kw.items() if k not in ("stats", "fold", "bnred")}
            ms_none = timed(lambda: ops.tc_gemm(A, K, W, ldw, tr, M, N, K, **kw_none))
            nbytes = algorithmic_bytes(M, K, N, pro, epi)
            flop_ms = 3 * 2 * M * N * K / TF32_FLOP_PER_S * 1e3
            cases[name] = dict(K=K, N=N, prologue=pro, epilogue=epi, ms=round(ms, 4), bytes=nbytes,
                               frac_of_3350_gb_per_s=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3),
                               byte_floor_ms=round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
                               tf32x3_flop_ms=round(flop_ms, 4), selection=list(selection(N, K)),
                               ms_epi_none=round(ms_none, 4))
            total += ms
            total_none += ms_none
            del A, W, kw, kw_none
            torch.cuda.empty_cache()
        line["rows"][str(M)] = dict(cases=cases, fourteen_launches_ms=round(total, 4),
                                    fourteen_launches_epi_none_ms=round(total_none, 4))
    if args.compare:
        line["bit_identical_to_saved"] = not mismatches
    print(json.dumps(line))
    if mismatches:
        sys.exit("outputs differ from the saved ones: " + ", ".join(mismatches))


if __name__ == "__main__":
    main()
