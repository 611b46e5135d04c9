"""The tensor-core GEMMs, their fused BatchNorm stages and the SIMT GEMM's fused statistics, called
kernel by kernel and compared with float64 references computed on the CPU from the same fp32 inputs:

  * tc_gemm2.cu: the forward / data-gradient GEMM at every (slice width NS, A-ring stages, N-slices)
    selection pick_ns can make, with its AFFINE and BNBWD prologues and its STATS and BNRED epilogues;
  * tc_dw.cu: the weight-gradient GEMM at all nine (CO, CI) instantiations;
  * tc_pack.cu: the batched weight packer against the single one;
  * dense.cu: spg_gemm with fused batch statistics, including a problem taller than one launch.

Every product is 3xTF32 or fp32, i.e. fp32-equivalent (DESIGN §3: ~1e-6 relative).  The bounds are
1e-5 of the tensor maximum; means 1e-6 and variances 1e-5.  The
data are mean-zero, so a skipped or duplicated 32-row chunk or 128-row tile moves a result by ~1e-2
relative, far above the bounds.  Every case draws from its own seed.

Row counts: 512 is the smallest M the wgmma path takes; 512 + 7 leaves a last warp with fewer than 8
valid rows; 128*5 + 72 ends the tail tile inside the second warpgroup; MULTI gives every CTA several
tiles plus a tail (301 tiles > 2 * 132 CTAs for one slice)."""
import zlib

import pytest
import torch

from test_gpu_parity import close

# --------------------------------------------------------------------------------------------------
# Python copy of the tile selection of tc_gemm2.cu (fixed_smem / stages_for / pick_ns)
T2_KC, T2_EPI_WARPS, STAGE_BYTES, MAX_STAGES, NUM_SMS = 32, 8, 2 * 128 * 32 * 4, 4, 132


def _fixed_smem(ns, k):
    return (k // T2_KC) * 2 * ns * T2_KC * 4 + (4 * k + ns + 4 * ns + T2_EPI_WARPS * ns * 4) * 4


def _stages_for(ns, k):
    return min((232448 - 1024 - _fixed_smem(ns, k)) // STAGE_BYTES, MAX_STAGES)


def _pick_ns(n, k):
    if n % 128 == 0 and _stages_for(128, k) >= 2:
        return 128
    if n % 64 == 0 and _stages_for(64, k) >= 2:
        return 64
    if n % 32 == 0 and n <= 64 and _stages_for(32, k) >= 2:
        return 32
    return 0


def selection(n, k):
    """(NS, A-ring stages, N-slices) the kernel runs (N, K) with, or None if it does not take it."""
    if n > 256 or k % T2_KC:
        return None
    ns = _pick_ns(n, k)
    return (ns, _stages_for(ns, k), n // ns) if ns else None


# (N, K) -> (NS, stages, slices): one shape for every selection there is (test_shape_table_is_complete)
SHAPES = {
    (32, 32): (32, 4, 1), (32, 384): (32, 3, 1), (32, 512): (32, 2, 1),
    (64, 320): (32, 4, 2), (64, 384): (32, 3, 2), (64, 512): (32, 2, 2),
    (64, 64): (64, 4, 1), (64, 192): (64, 3, 1), (64, 256): (64, 2, 1),
    (128, 160): (64, 4, 2), (128, 192): (64, 3, 2), (128, 256): (64, 2, 2),
    (192, 96): (64, 4, 3), (192, 192): (64, 3, 3), (192, 256): (64, 2, 3),
    (256, 160): (64, 4, 4), (256, 192): (64, 3, 4), (256, 256): (64, 2, 4),
    (128, 64): (128, 4, 1), (128, 96): (128, 3, 1), (128, 128): (128, 2, 1),
    (256, 64): (128, 4, 2), (256, 96): (128, 3, 2), (256, 128): (128, 2, 2),
}
MULTI = 128 * 301 + 45
GEMM_ROWS = (512, 512 + 7, 128 * 5 + 72, MULTI)
PROLOGUES = ("none", "scale", "shift", "scale_shift_relu")
DW_SHAPES = [(co, ci) for co in (64, 128, 256) for ci in (32, 64, 128)]
DW_ROWS = (2048, 2048 + 5, 32 * 132 + 31, 5000, 100003)
P_AFFS = ("none", "scale_shift", "scale_shift_relu", "shift")


# --------------------------------------------------------------------------------------------------
# float64 references
def ref_affine(x, scale, shift, relu):
    y = x
    if scale is not None:
        y = y * scale
    if shift is not None:
        y = y + shift
    return torch.relu(y) if relu else y


def ref_bn_backward(G, Y, scale, shift, mean, var, s12, eps, relu):
    """dL/dY of a = relu?(Y*scale + shift), the training-mode BatchNorm (batch mean/var) folded into
    scale/shift, from G = dL/da and the layer's sums s12 = sum gz | sum gz*xhat (gz = dL/d(BN out))."""
    M, K = Y.shape
    gz = G * ((Y * scale + shift) > 0) if relu else G
    xhat = (Y - mean) / torch.sqrt(var + eps)
    return scale * (gz - s12[:K] / M - xhat * s12[K:] / M)


def ref_bn_sums(G, Y, scale, shift, mean, var, eps, relu):
    """BatchNorm-backward sums s1 | s2 = sum_m gz | sum_m gz*xhat of the same layer (= d/dbeta, d/dgamma)."""
    gz = G * ((Y * scale + shift) > 0) if relu else G
    xhat = (Y - mean) / torch.sqrt(var + eps)
    return torch.cat([gz.sum(0), (gz * xhat).sum(0)])


def _bn_fold64(Y, gamma, beta, eps):
    mean, var = Y.mean(0), Y.var(0, unbiased=False)
    scale = gamma / torch.sqrt(var + eps)
    return mean, var, scale, beta - mean * scale


@pytest.mark.parametrize("relu", [True, False])
def test_reference_bn_backward_matches_autograd(relu):
    """The two BatchNorm-backward references above against torch.autograd through
    BatchNorm1d(track_running_stats=False) [+ ReLU] in float64."""
    g = torch.Generator().manual_seed(11 + relu)
    M, K, eps = 300, 24, 1e-5
    Y = (torch.randn(M, K, generator=g, dtype=torch.float64) * 2 + 0.5).requires_grad_(True)
    G = torch.randn(M, K, generator=g, dtype=torch.float64)
    bn = torch.nn.BatchNorm1d(K, eps=eps, track_running_stats=False).double()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(K, generator=g, dtype=torch.float64) + 0.5)
        bn.weight[::3] *= -1
        bn.bias.copy_(torch.randn(K, generator=g, dtype=torch.float64))
    a = bn(Y)
    (torch.relu(a) if relu else a).backward(G)
    Yd = Y.detach()
    mean, var, scale, shift = _bn_fold64(Yd, bn.weight.detach(), bn.bias.detach(), eps)
    s12 = ref_bn_sums(G, Yd, scale, shift, mean, var, eps, relu)
    torch.testing.assert_close(s12[:K], bn.bias.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(s12[K:], bn.weight.grad, rtol=1e-12, atol=1e-12)
    dY = ref_bn_backward(G, Yd, scale, shift, mean, var, s12, eps, relu)
    torch.testing.assert_close(dY, Y.grad, rtol=1e-10, atol=1e-12)


def test_shape_table_is_complete():
    """SHAPES names the selection it means, and between them they cover every selection pick_ns can
    make for any supported (N, K)."""
    for (n, k), want in SHAPES.items():
        assert selection(n, k) == want, (n, k)
    every = {selection(n, k) for n in range(32, 257, 32) for k in range(32, 4097, 32)} - {None}
    assert every == set(SHAPES.values())


# --------------------------------------------------------------------------------------------------
# GPU helpers
MEASURED = {}  # test group -> largest error / bound scale seen (printed at the end of the module)


def check(group, got, want, rtol, scale=None):
    """close(got, want, rtol) against max |want| (or against `scale`), recording the error."""
    got = torch.as_tensor(got).detach().double().cpu()
    want = torch.as_tensor(want).detach().double().cpu()
    assert got.shape == want.shape, (got.shape, want.shape)
    s = float(want.abs().max()) if scale is None else float(scale)
    err = float((got - want).abs().max())
    MEASURED[group] = max(MEASURED.get(group, 0.0), err / max(s, 1e-30))
    if scale is None:
        close(got, want, rtol)
    else:
        assert torch.isfinite(got).all(), "non-finite values"
        assert err <= rtol * s, "max err %g vs scale %g (rel %g)" % (err, s, err / max(s, 1e-30))


@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    yield torch.device("cuda:0")
    if MEASURED:
        print("\n[test_tc_gemm] largest error / scale per group:")
        for k in sorted(MEASURED):
            print("  %-12s %.3e" % (k, MEASURED[k]))


@pytest.fixture(autouse=True)
def _fresh_weight_images():
    # ops caches weight images by the weight's address: a tensor of an earlier case may have lived there
    from superpoint_graph_b200 import ops
    ops.PACK_CACHE.clear()
    yield
    ops.PACK_CACHE.clear()


@pytest.fixture
def gen(request):
    return torch.Generator().manual_seed(zlib.crc32(request.node.nodeid.encode()))


def randn(g, *shape):
    return torch.randn(*shape, generator=g)


def padded(x, ld, fill=float("nan")):
    """x [M, C] stored with leading dimension ld; the padding holds `fill` (NaN: any read shows)."""
    out = torch.full((x.shape[0], ld), fill, dtype=x.dtype)
    out[:, :x.shape[1]] = x
    return out


def d64(x):
    return None if x is None else x.double().cpu()


def bn_inputs(g, M, C, dev, relu):
    """A BatchNorm+ReLU layer's raw output Y [M, C] with its batch statistics and fold, as the
    forward leaves them (fp32), with no |Y*scale + shift| within 1e-3 of zero: there the ReLU mask
    could legitimately differ between the kernel's fmaf and float64."""
    eps = 1e-5
    Y = randn(g, M, C) * 1.5 + 0.7
    gamma = torch.rand(C, generator=g) + 0.5
    gamma[::3] *= -1
    beta = randn(g, C) * 0.5
    mean, var = Y.double().mean(0).float(), Y.double().var(0, unbiased=False).float()
    scale = (gamma.double() / torch.sqrt(var.double() + eps)).float()
    shift = (beta.double() - mean.double() * scale.double()).float()
    z = Y.double() * scale.double() + shift.double()
    near = z.abs() < 2e-3
    znew = torch.where(z >= 0, 4e-3, -4e-3).double()
    Y = torch.where(near, ((znew - shift.double()) / scale.double()).float(), Y)
    assert float((Y.double() * scale.double() + shift.double()).abs().min()) > 1e-3
    t = dict(Y=Y, scale=scale, shift=shift, mean=mean, var=var, eps=eps, relu=relu)
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in t.items()}, t


# --------------------------------------------------------------------------------------------------
# A. tc_gemm forward (PRO_AFFINE)
def _forward_cases():
    cases = []
    for i, (N, K) in enumerate(SHAPES):
        for j, M in enumerate(GEMM_ROWS):
            pro = PROLOGUES[(i + j) % 4]
            bias, transpose, lda = i % 2 == 0, i % 3 == 1, K + 4 * (j % 2)
            cases.append(pytest.param(N, K, M, pro, bias, transpose, lda, id="N%d-K%d-M%d-%s-%s-%s-lda%d" % (
                N, K, M, pro, "bias" if bias else "nobias", "WT" if transpose else "W", lda)))
    return cases


@pytest.mark.gpu
def test_selection_matches_library(dev):
    """The Python copy of the selection accepts exactly the shapes spg_tc_gemm_supported accepts."""
    from superpoint_graph_b200 import _lib
    for n in range(8, 300, 8):
        for k in range(8, 1100, 8):
            assert bool(_lib.lib().spg_tc_gemm_supported(4096, n, k)) == (selection(n, k) is not None), (n, k)


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,M,pro,has_bias,transpose,lda", _forward_cases())
def test_tc_gemm_forward(dev, gen, N, K, M, pro, has_bias, transpose, lda):
    from superpoint_graph_b200 import ops
    assert ops.tc_supported(M, N, K, lda, N) and selection(N, K) == SHAPES[(N, K)]
    A = randn(gen, M, K)
    W = randn(gen, N, K) / K ** 0.5
    bias = randn(gen, N) if has_bias else None
    scale = torch.rand(K, generator=gen) + 0.5 if pro in ("scale", "scale_shift_relu") else None
    if scale is not None:
        scale[::4] *= -1
    shift = randn(gen, K) if pro in ("shift", "scale_shift_relu") else None
    relu = pro == "scale_shift_relu"
    Wd = (W.t().contiguous() if transpose else W).to(dev)
    aff = None if pro == "none" else tuple(x.to(dev) if x is not None else None for x in (scale, shift)) + (relu,)
    C = ops.tc_gemm(padded(A, lda).to(dev), lda, Wd, K if not transpose else N, transpose, M, N, K,
                    bias=None if bias is None else bias.to(dev), a_aff=aff)
    ref = ref_affine(A.double(), d64(scale), d64(shift), relu) @ W.double().t()
    if bias is not None:
        ref += bias.double()
    check("forward", C, ref, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,kv", [(64, 32, 13), (128, 64, 40), (256, 32, 14)])
def test_tc_gemm_k_valid(dev, gen, N, K, kv):
    """K zero-padded to a multiple of 32 as chain_forward does: A's columns kv..K hold large finite
    values that the zero rows of the weight image must cancel."""
    from superpoint_graph_b200 import ops
    M = MULTI
    A = randn(gen, M, K)
    A[:, kv:] = 1e30
    W = randn(gen, N, kv) / kv ** 0.5
    bias = randn(gen, N)
    C = ops.tc_gemm(A.to(dev), K, W.to(dev), kv, False, M, N, K, bias=bias.to(dev), k_valid=kv)
    check("forward", C, A[:, :kv].double() @ W.double().t() + bias.double(), 1e-5)


# --------------------------------------------------------------------------------------------------
# B. EPI_STATS, with and without the BatchNorm fold
@pytest.mark.gpu
@pytest.mark.parametrize("fold", [False, True])
@pytest.mark.parametrize("M", [MULTI, 128 * 7 + 40])
@pytest.mark.parametrize("N,K", [(64, 64), (256, 64), (192, 96), (32, 512), (256, 192)])
def test_tc_gemm_stats(dev, gen, N, K, M, fold):
    """Statistics checked against the float64 statistics of the C the kernel returned (so that the
    reduction is judged apart from the GEMM's rounding); bias ~100 makes cancellation show.  M = 128*7 +
    40 leaves warps 3-7 of the last tile without a valid row."""
    from superpoint_graph_b200 import ops
    A = randn(gen, M, K)
    W = randn(gen, N, K) / K ** 0.5
    bias = 100 + randn(gen, N)
    args = dict(bias=bias.to(dev), stats=True)
    mom, eps = 0.1, 1e-5
    if fold:
        gamma = torch.rand(N, generator=gen) + 0.5
        gamma[::4] *= -1
        beta = randn(gen, N)
        rm0, rv0 = randn(gen, N), torch.rand(N, generator=gen) + 0.5
        rm, rv = rm0.to(dev), rv0.to(dev)
        nbt = torch.full((), 5, dtype=torch.long, device=dev)
        args["fold"] = (gamma.to(dev), beta.to(dev), eps, rm, rv, nbt, mom)
    res = ops.tc_gemm(A.to(dev), K, W.to(dev), K, False, M, N, K, **args)
    C = res[0]
    check("forward", C, A.double() @ W.double().t() + bias.double(), 1e-5)
    C64 = C.double().cpu()
    check("stats_mean", res[1], C64.mean(0), 1e-6)
    check("stats_var", res[2], C64.var(0, unbiased=False), 1e-5)
    if not fold:
        assert len(res) == 3
        return
    scale = gamma.double() / torch.sqrt(C64.var(0, unbiased=False) + eps)
    check("stats_fold", res[3], scale, 1e-5)
    check("stats_fold", res[4], beta.double() - C64.mean(0) * scale, 1e-5)
    bn = torch.nn.BatchNorm1d(N, eps=eps, momentum=mom).double()
    with torch.no_grad():
        bn.running_mean.copy_(rm0.double())
        bn.running_var.copy_(rv0.double())
        bn.num_batches_tracked.fill_(5)
    bn.train()
    bn(C64)
    check("stats_fold", rm, bn.running_mean, 1e-6)
    check("stats_fold", rv, bn.running_var, 1e-5)
    assert int(nbt) == int(bn.num_batches_tracked) == 6


# --------------------------------------------------------------------------------------------------
# C. PRO_BNBWD [+ EPI_BNRED], called the way chain_backward calls it
@pytest.mark.gpu
@pytest.mark.parametrize("relu,relu_below", [(True, True), (True, False), (False, True), (False, False),
                                             (True, None)])
@pytest.mark.parametrize("N,K,M", [(64, 128, 512 + 7), (256, 64, MULTI), (192, 96, 128 * 5 + 72),
                                   (64, 320, MULTI)])
def test_tc_gemm_bn_backward(dev, gen, N, K, M, relu, relu_below):
    """Data gradient of a layer W [K, N] (K = this layer's outputs, N = its inputs) whose output went
    through BatchNorm [+ ReLU]: the prologue turns G = dL/d(activation) into dL/dY (also stored), the
    product gives the layer below's dL/d(activation), and the epilogue reduces that layer's sums
    (relu_below None: no layer below with BatchNorm).  N = 256, 192 and 64 at K = 320 run 2 or 3
    N-slices, of which only slice 0 stores dY."""
    from superpoint_graph_b200 import ops
    assert selection(N, K) is not None
    G = randn(gen, M, K)
    top, top_h = bn_inputs(gen, M, K, dev, relu)
    s12 = ref_bn_sums(G.double(), *(d64(top_h[k]) for k in ("Y", "scale", "shift", "mean", "var")),
                      top_h["eps"], relu).float()
    W = randn(gen, K, N) / K ** 0.5
    bnbwd = (top["Y"], K, top["scale"], top["shift"], relu, top["mean"], top["var"], s12.to(dev), top["eps"], True)
    bnred = None
    if relu_below is not None:
        low, low_h = bn_inputs(gen, M, N, dev, relu_below)
        bnred = (low["Y"], N, low["scale"], low["shift"], low["mean"], low["var"], low["eps"], relu_below)
    res = ops.tc_gemm(G.to(dev), K, W.to(dev), N, True, M, N, K, bnbwd=bnbwd, bnred=bnred)
    assert len(res) == (3 if bnred is not None else 2)
    C, dY = res[0], res[1]
    dY_ref = ref_bn_backward(G.double(), *(d64(top_h[k]) for k in ("Y", "scale", "shift", "mean", "var")),
                             s12.double(), top_h["eps"], relu)
    check("bnbwd_dY", dY, dY_ref, 1e-5)
    check("bnbwd_C", C, dY_ref @ W.double(), 1e-5)
    if bnred is None:
        return
    # the layer below's sums come from the kernel's own C
    C64 = C.double().cpu()
    Y2, sc2, sh2, mu2, var2 = (d64(low_h[k]) for k in ("Y", "scale", "shift", "mean", "var"))
    gz = C64 * ((Y2 * sc2 + sh2) > 0) if relu_below else C64
    xhat = (Y2 - mu2) / torch.sqrt(var2 + low_h["eps"])
    scale = max(float(gz.abs().sum(0).max()), float((gz * xhat).abs().sum(0).max()))
    ref = ref_bn_sums(C64, Y2, sc2, sh2, mu2, var2, low_h["eps"], relu_below)
    check("bnred_s12", res[2], ref, 1e-5, scale=scale)


# --------------------------------------------------------------------------------------------------
# D. tc_dw at every instantiation
def _dw_cases():
    cases = []
    for i, (co, ci) in enumerate(DW_SHAPES):
        for j, M in enumerate(DW_ROWS):
            aff = P_AFFS[(i + j) % 4]
            lddy, ldp = co + 4 * ((i + j) % 2), ci + 8 * (j % 2)
            cases.append(pytest.param(co, ci, M, aff, lddy, ldp,
                                      id="CO%d-CI%d-M%d-%s-lddy%d-ldp%d" % (co, ci, M, aff, lddy, ldp)))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("co,ci,M,aff,lddy,ldp", _dw_cases())
def test_tc_dw(dev, gen, co, ci, M, aff, lddy, ldp):
    """dW = dY^T f(P).  M = 2048 is the smallest M the wgmma path takes; 32*132 + 31 gives one chunk
    more than there are CTAs; at M = 5000 every CTA takes 64 points and CTAs 79..131 get none (their
    partials must be zero); 100003 accumulates ~760 points per CTA.  The bound is the module's 1e-5 of the
    maximum: at 760 fp32 accumulations per CTA and 132 partials the expected error is ~1e-6 of it."""
    from superpoint_graph_b200 import ops
    assert ops.tc_dw_supported(M, co, ci, lddy, ldp)
    dY = randn(gen, M, co)
    P = randn(gen, M, ci) * 1.3 + 0.2
    scale = shift = None
    if aff in ("scale_shift", "scale_shift_relu"):
        scale = torch.rand(ci, generator=gen) + 0.5
        scale[::4] *= -1
    if aff != "none":
        shift = randn(gen, ci)
    relu = aff == "scale_shift_relu"
    p_aff = None if aff == "none" else (None if scale is None else scale.to(dev), shift.to(dev), relu)
    dW = ops.tc_dw(padded(dY, lddy).to(dev), lddy, padded(P, ldp).to(dev), ldp, M, co, ci, p_aff=p_aff)
    ref = dY.double().t() @ ref_affine(P.double(), d64(scale), d64(shift), relu)
    check("dw", dW, ref, 1e-5)


# --------------------------------------------------------------------------------------------------
# E. write set and determinism
def _image(W, ldw, transpose, N, K, kv, dev):
    from superpoint_graph_b200 import _lib
    img = torch.empty(2 * N * K, dtype=torch.float32, device=dev)
    _lib.call("spg_tc_pack_weights", W, ldw, int(transpose), N, K, kv, img, _lib.current_stream())
    return img


SENTINEL = -1.2345e37


@pytest.mark.gpu
@pytest.mark.parametrize("M", [512 + 7, 128 * 301 + 72])
def test_tc_gemm_write_set(dev, gen, M):
    """Through the C-ABI with C [M+3, ldc = N+4] and dY [M+3, K+4] filled with a sentinel: the kernel
    writes exactly the [M, N] (and [M, K]) block, with the same values as with dense outputs."""
    from superpoint_graph_b200 import _lib, ops
    N, K = 256, 64  # two N-slices
    G = randn(gen, M, K)
    top, top_h = bn_inputs(gen, M, K, dev, True)
    low, _ = bn_inputs(gen, M, N, dev, True)
    s12 = ref_bn_sums(G.double(), *(d64(top_h[k]) for k in ("Y", "scale", "shift", "mean", "var")),
                      top_h["eps"], True).float().to(dev)
    W = (randn(gen, K, N) / K ** 0.5).to(dev)
    Gd = G.to(dev)
    want = ops.tc_gemm(Gd, K, W, N, True, M, N, K,
                       bnbwd=(top["Y"], K, top["scale"], top["shift"], True, top["mean"], top["var"], s12,
                              top["eps"], True),
                       bnred=(low["Y"], N, low["scale"], low["shift"], low["mean"], low["var"], low["eps"], True))
    ldc, lddy = N + 4, K + 4
    C = torch.full((M + 3, ldc), SENTINEL, device=dev)
    dY = torch.full((M + 3, lddy), SENTINEL, device=dev)
    e_s12 = torch.empty(2 * N, device=dev)
    ws = torch.empty(_lib.lib().spg_tc_gemm_max_partials() * N * 3, device=dev)
    img = _image(W, N, True, N, K, K, dev)
    _lib.call("spg_tc_gemm_ex", Gd, K, img, None, C, ldc, M, N, K, top["scale"], top["shift"], 1,
              top["Y"], K, top["mean"], top["var"], s12, float(top["eps"]), dY, lddy, 2, ws,
              None, None, None, None, 0.0, None, None, None, None, None, 0.0,
              low["Y"], N, low["scale"], low["shift"], low["mean"], low["var"], float(low["eps"]), 1, e_s12,
              _lib.current_stream())
    for got, ref, cols in ((C, want[0], N), (dY, want[1], K)):
        assert torch.equal(got[:M, :cols], ref)
        assert bool((got[:M, cols:] == SENTINEL).all()) and bool((got[M:] == SENTINEL).all())
    assert torch.equal(e_s12, want[2])
    # forward with the statistics epilogue
    A = randn(gen, M, K).to(dev)
    Wf = (randn(gen, N, K) / K ** 0.5).to(dev)
    bias = (100 + randn(gen, N)).to(dev)
    want = ops.tc_gemm(A, K, Wf, K, False, M, N, K, bias=bias, stats=True)
    C.fill_(SENTINEL)
    mean, var = torch.empty(N, device=dev), torch.empty(N, device=dev)
    _lib.call("spg_tc_gemm_ex", A, K, _image(Wf, K, False, N, K, K, dev), bias, C, ldc, M, N, K, None, None, 0,
              None, 0, None, None, None, 0.0, None, 0, 1, ws,
              mean, var, None, None, 0.0, None, None, None, None, None, 0.0,
              None, 0, None, None, None, None, 0.0, 0, None, _lib.current_stream())
    assert torch.equal(C[:M, :N], want[0])
    assert bool((C[:M, N:] == SENTINEL).all()) and bool((C[M:] == SENTINEL).all())
    assert torch.equal(mean, want[1]) and torch.equal(var, want[2])


@pytest.mark.gpu
def test_fused_reductions_are_deterministic(dev, gen):
    """STATS (with the fold), BNRED and tc_dw merge their per-CTA partials in a fixed order: the same
    inputs give bitwise the same outputs (CUDA graph replay relies on it)."""
    from superpoint_graph_b200 import ops
    M, N, K = 128 * 301 + 72, 256, 64  # a layer K -> N: forward over two N-slices, data gradient N -> K
    A = randn(gen, M, K).to(dev)
    W = (randn(gen, N, K) / K ** 0.5).to(dev)
    bias = (100 + randn(gen, N)).to(dev)
    gamma, beta = (torch.rand(N, generator=gen) + 0.5).to(dev), randn(gen, N).to(dev)

    def stats():
        rm, rv = torch.zeros(N, device=dev), torch.ones(N, device=dev)
        nbt = torch.zeros((), dtype=torch.long, device=dev)
        return ops.tc_gemm(A, K, W, K, False, M, N, K, bias=bias, stats=True,
                           fold=(gamma, beta, 1e-5, rm, rv, nbt, 0.1)) + (rm, rv)

    G = randn(gen, M, N)
    top, top_h = bn_inputs(gen, M, N, dev, True)
    low, _ = bn_inputs(gen, M, K, dev, True)
    s12 = ref_bn_sums(G.double(), *(d64(top_h[k]) for k in ("Y", "scale", "shift", "mean", "var")),
                      top_h["eps"], True).float().to(dev)
    G = G.to(dev)

    def bnred():
        return ops.tc_gemm(G, N, W, K, True, M, K, N,
                           bnbwd=(top["Y"], N, top["scale"], top["shift"], True, top["mean"], top["var"], s12,
                                  top["eps"], True),
                           bnred=(low["Y"], K, low["scale"], low["shift"], low["mean"], low["var"], low["eps"], True))

    sc, sh = (torch.rand(K, generator=gen) + 0.5).to(dev), randn(gen, K).to(dev)

    def dw():
        return (ops.tc_dw(G, N, A, K, M, N, K, p_aff=(sc, sh, True)),)

    for run in (stats, bnred, dw):
        first, second = run(), run()
        for a, b in zip(first, second):
            assert torch.equal(a, b), run.__name__


# --------------------------------------------------------------------------------------------------
# F. weight images: batched packer == single packer
@pytest.mark.gpu
def test_prepack_matches_single_pack(dev, gen):
    from superpoint_graph_b200 import ops
    Ws = [randn(gen, 64, 13), randn(gen, 20, 64), randn(gen, 128, 64), randn(gen, 256, 40), randn(gen, 50, 192)]
    Ws = [w.to(dev) for w in Ws]
    jobs = [(Ws[0], 13, False, 64, 32, 13),     # forward, K padded 13 -> 32
            (Ws[1], 64, True, 64, 32, 20),      # transposed, K padded 20 -> 32
            (Ws[2], 64, False, 128, 64, 64),
            (Ws[2], 64, True, 64, 128, 128),
            (Ws[3], 40, False, 256, 64, 40),
            (Ws[4], 192, True, 192, 64, 50)]
    ops.prepack(jobs)
    for W, ldw, tr, N, K, kv in jobs:
        got = ops.PACK_CACHE[(W.data_ptr(), ldw, int(tr), N, K, kv)]
        assert torch.equal(got.view(torch.int32), _image(W, ldw, tr, N, K, kv, dev).view(torch.int32)), \
            (tuple(W.shape), tr, N, K, kv)


# --------------------------------------------------------------------------------------------------
# G. SIMT gemm with fused statistics
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(10037, 70, 13), (3001, 32, 13), (1000, 130, 45)])
def test_gemm_stats_fold(dev, gen, M, N, K):
    """The filter network's first layer (K = 13) and FC-like shapes: M not a multiple of 128, N not a
    multiple of 64."""
    from superpoint_graph_b200 import ops
    A = randn(gen, M, K)
    B = randn(gen, N, K) / K ** 0.5
    bias = 100 + randn(gen, N)
    gamma, beta = torch.rand(N, generator=gen) + 0.5, randn(gen, N)
    gamma[::4] *= -1
    rm0, rv0 = randn(gen, N), torch.rand(N, generator=gen) + 0.5
    rm, rv = rm0.to(dev), rv0.to(dev)
    nbt = torch.full((), 2, dtype=torch.long, device=dev)
    eps, mom = 1e-5, 0.1
    out, mean, var, scale, shift = ops.gemm(A.to(dev), K, True, B.to(dev), K, True, M, N, K, bias=bias.to(dev),
                                            stats=True, fold=(gamma.to(dev), beta.to(dev), eps, rm, rv, nbt, mom))
    check("simt_C", out, A.double() @ B.double().t() + bias.double(), 1e-5)
    C64 = out.double().cpu()
    check("simt_mean", mean, C64.mean(0), 1e-6)
    check("simt_var", var, C64.var(0, unbiased=False), 1e-5)
    sc = gamma.double() / torch.sqrt(C64.var(0, unbiased=False) + eps)
    check("simt_fold", scale, sc, 1e-5)
    check("simt_fold", shift, beta.double() - C64.mean(0) * sc, 1e-5)
    bn = torch.nn.BatchNorm1d(N, eps=eps, momentum=mom).double()
    with torch.no_grad():
        bn.running_mean.copy_(rm0.double())
        bn.running_var.copy_(rv0.double())
    bn.train()
    bn(C64)
    check("simt_fold", rm, bn.running_mean, 1e-6)
    check("simt_fold", rv, bn.running_var, 1e-5)
    assert int(nbt) == 3


@pytest.mark.gpu
def test_gemm_stats_taller_than_one_launch(dev):
    """M = 65535*128 + 200 rows: spg_gemm runs two row slabs (blockIdx.y <= 65535) that write their tile
    statistics at stats_tile0, and the 65537 tile partials need three merge levels.  ~1.5 GB of device
    memory; the float64 statistics are computed on the device, in row blocks."""
    from superpoint_graph_b200 import ops
    M, N, K = 65535 * 128 + 200, 32, 13
    g = torch.Generator(device=dev).manual_seed(20261016)
    A = torch.randn(M, K, device=dev, generator=g)
    B = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    bias = 100 + torch.randn(N, device=dev, generator=g)
    gamma, beta = torch.rand(N, device=dev, generator=g) + 0.5, torch.randn(N, device=dev, generator=g)
    rm0, rv0 = torch.randn(N, device=dev, generator=g), torch.rand(N, device=dev, generator=g) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros((), dtype=torch.long, device=dev)
    eps, mom = 1e-5, 0.1
    out, mean, var, scale, shift = ops.gemm(A, K, True, B, K, True, M, N, K, bias=bias, stats=True,
                                            fold=(gamma, beta, eps, rm, rv, nbt, mom))
    # C at the first rows and from 300 rows before the slab boundary to the end, in float64 on the CPU
    rows = torch.cat([torch.arange(0, 300), torch.arange(65535 * 128 - 300, M)])
    assert int(rows.max()) == M - 1
    rows = rows.to(dev)
    ref = A[rows].double().cpu() @ B.double().cpu().t() + bias.double().cpu()
    check("simt_C", out[rows], ref, 1e-5)
    step = 1 << 20
    s = torch.zeros(N, dtype=torch.float64, device=dev)
    for r in range(0, M, step):
        s += out[r:r + step].sum(0, dtype=torch.float64)
    mu = s / M
    q = torch.zeros(N, dtype=torch.float64, device=dev)
    for r in range(0, M, step):
        q += ((out[r:r + step].double() - mu) ** 2).sum(0)
    v = q / M
    check("simt_mean", mean, mu, 1e-6)
    check("simt_var", var, v, 1e-5)
    sc = gamma.double() / torch.sqrt(v + eps)
    check("simt_fold", scale, sc, 1e-5)
    check("simt_fold", shift, beta.double() - mu * sc, 1e-5)
    check("simt_fold", rm, (1 - mom) * rm0.double() + mom * mu, 1e-6)
    check("simt_fold", rv, (1 - mom) * rv0.double() + mom * v * M / (M - 1), 1e-5)
    assert int(nbt) == 1
