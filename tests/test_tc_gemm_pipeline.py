"""What the ping-pong pipeline of tc_gemm2.cu can get wrong and the float64 tests of test_tc_gemm.py do not
show: results that depend on timing, and the tile a warpgroup runs with no valid row.

Each consumer warpgroup has its own A ring, filled by its own producer warpgroup, and the two take turns on
the tensor cores.  LONG = 128*132*12 + 45 rows give every CTA 12 tiles or more, so at the deepest ring (4
stages) both mbarrier phases of every stage of both rings are waited on several times.  TAIL = 128*301 + 40
ends the last tile inside warpgroup 0's half: warpgroup 1 has no valid row there and must still take its
turn and release its stages.  Every slice width NS the kernel has (32, 64, 128) runs with both prologues,
AFFINE with the STATS epilogue and BNBWD with BNRED."""
import pytest
import torch

from test_tc_gemm import (SENTINEL, _fresh_weight_images, _image, bn_inputs, check, d64, dev, gen,  # noqa: F401
                          randn, ref_bn_backward, ref_bn_sums, selection)

LONG = 128 * 132 * 12 + 45
TAIL = 128 * 301 + 40
# (N, K) of a forward layer (AFFINE + STATS) and of a data gradient (BNBWD + BNRED) per slice width
FWD = {32: (32, 32), 64: (64, 64), 128: (128, 128)}
BWD = {32: (64, 320), 64: (64, 128), 128: (128, 128)}


def _forward(gen, dev, M, N, K):
    """Seeded forward layer: A is a BatchNorm+ReLU layer's raw output, applied by the prologue."""
    low, low_h = bn_inputs(gen, M, K, dev, True)
    W = randn(gen, N, K) / K ** 0.5
    bias = 100 + randn(gen, N)
    gamma, beta = torch.rand(N, generator=gen) + 0.5, randn(gen, N)
    ref = torch.relu(d64(low_h["Y"]) * d64(low_h["scale"]) + d64(low_h["shift"])) @ W.double().t() + bias.double()
    return low, W.to(dev), bias.to(dev), gamma.to(dev), beta.to(dev), ref


def _backward(gen, dev, M, N, K):
    """Seeded data gradient of a layer W [K, N] with BatchNorm+ReLU on both sides (see test_tc_gemm_bn_backward)."""
    G = randn(gen, M, K)
    top, top_h = bn_inputs(gen, M, K, dev, True)
    hk = [d64(top_h[k]) for k in ("Y", "scale", "shift", "mean", "var")]
    s12 = ref_bn_sums(G.double(), *hk, top_h["eps"], True).float()
    low, low_h = bn_inputs(gen, M, N, dev, True)
    W = randn(gen, K, N) / K ** 0.5
    dY_ref = ref_bn_backward(G.double(), *hk, s12.double(), top_h["eps"], True)
    bnbwd = (top["Y"], K, top["scale"], top["shift"], True, top["mean"], top["var"], s12.to(dev), top["eps"], True)
    bnred = (low["Y"], N, low["scale"], low["shift"], low["mean"], low["var"], low["eps"], True)
    return G.to(dev), W, W.to(dev), bnbwd, bnred, low_h, dY_ref


def _check_stats(res, ref):
    C, mean, var = res[0], res[1], res[2]
    check("pipe_forward", C, ref, 1e-5)
    C64 = C.double().cpu()
    check("pipe_mean", mean, C64.mean(0), 1e-6)
    check("pipe_var", var, C64.var(0, unbiased=False), 1e-5)


def _check_backward(res, W, dY_ref, low_h):
    C, dY, s12 = res
    check("pipe_dY", dY, dY_ref, 1e-5)
    check("pipe_dx", C, dY_ref @ W.double(), 1e-5)
    C64 = C.double().cpu()
    Y2, sc2, sh2, mu2, var2 = (d64(low_h[k]) for k in ("Y", "scale", "shift", "mean", "var"))
    gz = C64 * ((Y2 * sc2 + sh2) > 0)
    xhat = (Y2 - mu2) / torch.sqrt(var2 + low_h["eps"])
    scale = max(float(gz.abs().sum(0).max()), float((gz * xhat).abs().sum(0).max()))
    check("pipe_s12", s12, ref_bn_sums(C64, Y2, sc2, sh2, mu2, var2, low_h["eps"], True), 1e-5, scale=scale)


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [32, 64, 128])
def test_forward_stats_long_runs(dev, gen, ns):
    """AFFINE + STATS with the BatchNorm fold over many tiles per CTA: two calls agree bitwise (every output,
    running statistics included) and match float64."""
    from superpoint_graph_b200 import ops
    M, (N, K) = LONG, FWD[ns]
    assert selection(N, K)[0] == ns
    low, W, bias, gamma, beta, ref = _forward(gen, dev, M, N, K)

    def run():
        rm, rv = torch.zeros(N, device=dev), torch.ones(N, device=dev)
        nbt = torch.zeros((), dtype=torch.long, device=dev)
        return ops.tc_gemm(low["Y"], K, W, K, False, M, N, K, bias=bias,
                           a_aff=(low["scale"], low["shift"], True), stats=True,
                           fold=(gamma, beta, 1e-5, rm, rv, nbt, 0.1)) + (rm, rv, nbt)

    first, second = run(), run()
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    _check_stats(first, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [32, 64, 128])
def test_backward_bnred_long_runs(dev, gen, ns):
    """BNBWD (with the dY side store) + BNRED over many tiles per CTA: two calls agree bitwise and match
    float64."""
    from superpoint_graph_b200 import ops
    M, (N, K) = LONG, BWD[ns]
    assert selection(N, K)[0] == ns
    G, W, Wd, bnbwd, bnred, low_h, dY_ref = _backward(gen, dev, M, N, K)

    def run():
        return ops.tc_gemm(G, K, Wd, N, True, M, N, K, bnbwd=bnbwd, bnred=bnred)

    first, second = run(), run()
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    _check_backward(first, W, dY_ref, low_h)


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [32, 64, 128])
def test_tail_in_first_half(dev, gen, ns):
    """M = 128*301 + 40: through the C-ABI with C [M+3, N+4] and dY [M+3, K+4] filled with a sentinel, the
    data gradient writes exactly the [M, N] and [M, K] blocks, with the values (and sums) of the dense call,
    which match float64; then the same for the forward with STATS."""
    from superpoint_graph_b200 import _lib, ops
    M, (N, K) = TAIL, BWD[ns]
    G, W, Wd, bnbwd, bnred, low_h, dY_ref = _backward(gen, dev, M, N, K)
    want = ops.tc_gemm(G, K, Wd, N, True, M, N, K, bnbwd=bnbwd, bnred=bnred)
    _check_backward(want, W, dY_ref, low_h)
    Y, _, sc, sh, _, mu, var, s12, eps, _ = bnbwd
    Y2, _, sc2, sh2, mu2, var2, eps2, _ = bnred
    ldc, lddy = N + 4, K + 4
    C = torch.full((M + 3, ldc), SENTINEL, device=dev)
    dY = torch.full((M + 3, lddy), SENTINEL, device=dev)
    e_s12 = torch.empty(2 * N, device=dev)
    ws = torch.empty(_lib.lib().spg_tc_gemm_max_partials() * max(N, 128) * 3, device=dev)
    _lib.call("spg_tc_gemm_ex", G, K, _image(Wd, N, True, N, K, K, dev), None, C, ldc, M, N, K, sc, sh, 1,
              Y, K, mu, var, s12, float(eps), dY, lddy, 2, ws,
              None, None, None, None, 0.0, None, None, None, None, None, 0.0,
              Y2, N, sc2, sh2, mu2, var2, float(eps2), 1, e_s12, _lib.current_stream())
    for got, ref, cols in ((C, want[0], N), (dY, want[1], K)):
        assert torch.equal(got[:M, :cols], ref)
        assert bool((got[:M, cols:] == SENTINEL).all()) and bool((got[M:] == SENTINEL).all())
    assert torch.equal(e_s12, want[2])

    N, K = FWD[ns]
    low, Wf, bias, _, _, ref = _forward(gen, dev, M, N, K)
    aff = (low["scale"], low["shift"], True)
    want = ops.tc_gemm(low["Y"], K, Wf, K, False, M, N, K, bias=bias, a_aff=aff, stats=True)
    _check_stats(want, ref)
    ldc = N + 4
    C = torch.full((M + 3, ldc), SENTINEL, device=dev)
    mean, var = torch.empty(N, device=dev), torch.empty(N, device=dev)
    _lib.call("spg_tc_gemm_ex", low["Y"], K, _image(Wf, K, False, N, K, K, dev), bias, C, ldc, M, N, K,
              aff[0], aff[1], 1, None, 0, None, None, None, 0.0, None, 0, 1, ws,
              mean, var, None, None, 0.0, None, None, None, None, None, 0.0,
              None, 0, None, None, None, None, 0.0, 0, None, _lib.current_stream())
    assert torch.equal(C[:M, :N], want[0])
    assert bool((C[:M, N:] == SENTINEL).all()) and bool((C[M:] == SENTINEL).all())
    assert torch.equal(mean, want[1]) and torch.equal(var, want[2])
