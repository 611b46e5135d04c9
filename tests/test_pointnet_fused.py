"""The fused eval-mode PointNet trunk (csrc/pointnet_fused.cu), called kernel by kernel and compared with
float64 references computed on the CPU from the same fp32 inputs:

  * its host entry points (spg_pointnet_fused_supported and the two image-row counts) against Python
    copies of them, and the chain table CHAINS, which between its rows reaches every first-layer width,
    every inner transition, every (previous, last) width pair, 1-layer and 6-layer chains and the
    production chains;
  * the fp32 (3xTF32) kernel on every CHAINS row against an unfused float64 reference: xy transform
    (row vector times T + I), conv, BatchNorm with running statistics, ReLU, max over the points.  The
    bound is 1e-5 of the pooled tensor's maximum, as for the tc_gemm tests: 3xTF32 is fp32-equivalent and
    the only other difference is the fp32 fold of BatchNorm into the weights and bias;
  * the bf16 kernel on every CHAINS row against a float64 emulation of its own rounding: the transformed
    inputs rounded to bf16 (round to nearest even), the weights as bf16(fp32(W * scale)), the fp32 folded
    bias the kernel was given, exact accumulation, every non-last layer's ReLU output rounded to bf16 and
    the last layer max-pooled unrounded.  What is left is fp32 accumulation order and the rare activation
    whose bf16 rounding flips by one ulp because of it: unbiased, but a flip at a large activation of an
    inner layer reaches the pooled output, so the error grows with depth.  Bound BF16_TOL = 3e-3 of the tensor
    maximum; the largest error measured over the whole module (H100 SXM, 700 W) is 1.3e-3, on the 6-layer
    chain; rounding toward zero instead is 8e-3 or more away on every chain.  The fp32 path's largest
    measured error is 3.4e-6 (bound 1e-5).  Both maxima are printed at the end of a run (pytest -s);
  * the bf16 weight packer, bit for bit, and the folded biases;
  * F from 1 to 16 with and without T, batch sizes around the 132-CTA grid and far beyond it (many
    superpoints per CTA: the mbarrier phases of both weight rings wrap many times), a planted argmax at every
    row / warp / warpgroup position, channels that are dead at every point, the write set of `pooled`,
    determinism, kernel identity and the argument checks of both entry points.

Both bounds are shown to be able to fail (test_reference_bounds_can_fail): on the tests' own data, a bf16
emulation that rounds toward zero, and an fp32 emulation with one TF32 product (the lo terms dropped), are
each further from their reference than the bound.

NaN inputs are outside what this module pins: the fused epilogue's ReLU and max use fmaxf, which drops a
NaN where torch would propagate it, and the layer-by-layer path does the same (fmaxf in its ReLU prologues
and epilogues, pointnet.cu, tc_gemm2.cu, bn_act.cu).

The folded weight image is cached by ops.pointnet_fused_image.  The last group of tests checks that the
cache never serves an image older than the weights and statistics it was folded from: after a training
step (the optimizer writes the parameters through raw pointers), after a training-mode forward (the
running statistics are written inside the fold kernels), through a captured eval graph, and for a new
model whose tensors land at a freed model's addresses.

Every case draws from its own seed."""
import gc
import zlib

import numpy as np
import pytest
import torch
import torch.nn as nn

from test_gpu_parity import close

# --------------------------------------------------------------------------------------------------
# Python copies of the host entry points (pointnet_fused.cu)
PF_ROWS, PF_MAXF, PF_MAX_LAYERS, PF_MAXK, PF_MAX_BIAS = 128, 16, 6, 128, 1024
WIDTHS = (32, 64, 128, 256)
SPG_OK, SPG_E_BADARG, SPG_E_UNSUPPORTED, SPG_E_ALIGN = 0, -1, -2, -3


def supported(F, n_points, widths):
    if n_points != PF_ROWS or not 1 <= F <= PF_MAXF or not 1 <= len(widths) <= PF_MAX_LAYERS:
        return False
    for i, n in enumerate(widths):
        if n not in WIDTHS or (i + 1 < len(widths) and n > PF_MAXK):
            return False
    return sum(widths) <= PF_MAX_BIAS


def image_rows(widths):
    rows, k = 0, 32
    for n in widths:
        rows += (k // 32) * 2 * n
        k = n
    return rows


def bf16_image_rows(widths):
    rows, k = 0, 64
    for n in widths:
        rows += (k // 64) * n
        k = max(n, 64)
    return rows


# Chains the GPU tests run (test_chain_table_is_complete says what they cover between them).  PRODUCTION: the
# chains of the benchmarked models (S3DIS / Semantic3D main and STN chains, vKITTI main and STN chains).
CHAINS = [
    (256,), (32,), (64,), (128,),
    (64, 64, 128, 128, 256), (64, 64, 128), (32, 64),
    (32, 32, 128, 32, 64, 32), (128, 64, 32, 128, 64, 256),
    (32, 32), (64, 32, 128), (128, 32, 256), (64, 64), (128, 32), (64, 128, 64), (32, 128, 128),
]
PRODUCTION = [(64, 64, 128, 128, 256), (64, 64, 128), (32, 64)]
CHAIN_F = (14, 9, 11, 16, 3, 2, 15)


def chain_id(w):
    return "-".join(str(n) for n in w)


def _chain_case(i, widths):
    """(F, conv bias) of CHAINS row i: the features cycle through CHAIN_F, every other row has no bias."""
    return CHAIN_F[i % len(CHAIN_F)], i % 2 == 0


def test_python_copies_match_library():
    """supported / image_rows / bf16_image_rows equal the library's host functions over a grid of F, n_points,
    layer counts and widths (valid and invalid)."""
    from superpoint_graph_b200 import _lib
    L = _lib.lib()
    rng = np.random.default_rng(7)
    pool = (16, 31, 32, 48, 64, 96, 128, 192, 256, 512)
    n_checked = 0
    for nl in range(0, 8):
        draws = [tuple(rng.choice(pool, nl).tolist()) for _ in range(40)]
        draws += [tuple(rng.choice(WIDTHS, nl).tolist()) for _ in range(40)]
        if nl <= 2:
            draws += [tuple(w) for w in np.array(np.meshgrid(*[pool] * nl)).reshape(nl, -1).T.tolist()] if nl else [()]
        for w in set(draws):
            arr = torch.tensor(list(w) or [0], dtype=torch.int32)
            assert L.spg_pointnet_fused_image_rows(9, nl, arr.data_ptr()) == image_rows(w), w
            assert L.spg_pointnet_fused_bf16_image_rows(9, nl, arr.data_ptr()) == bf16_image_rows(w), w
            for F in range(0, 18):
                for npts in (127, 128, 129):
                    got = bool(L.spg_pointnet_fused_supported(F, npts, nl, arr.data_ptr()))
                    assert got == supported(F, npts, w), (F, npts, w)
                    n_checked += 1
    assert n_checked > 10000


def test_chain_table_is_complete():
    """CHAINS holds every first-layer width, all 9 inner transitions, all 12 (previous, last) width pairs,
    1-layer chains including [256], two 6-layer chains and the production chains; every row is supported."""
    for i, w in enumerate(CHAINS):
        F, _ = _chain_case(i, w)
        assert supported(F, 128, w), w
    inner = (32, 64, 128)
    assert {w[0] for w in CHAINS} == set(WIDTHS)
    middle = {(w[i], w[i + 1]) for w in CHAINS for i in range(len(w) - 2)}
    assert middle == {(a, b) for a in inner for b in inner}
    last = {(w[-2], w[-1]) for w in CHAINS if len(w) > 1}
    assert last == {(a, b) for a in inner for b in WIDTHS}
    assert (256,) in CHAINS and sum(len(w) == 1 for w in CHAINS) >= 2
    assert sum(len(w) == 6 for w in CHAINS) >= 2
    assert all(p in CHAINS for p in PRODUCTION)
    assert len(set(CHAINS)) == len(CHAINS)


# --------------------------------------------------------------------------------------------------
# synthetic layers and float64 references
FP32_TOL = 1e-5
BF16_TOL = 3e-3
EPS = 1e-3


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def make_chain(g, F, widths, bias=True, dead=()):
    """nn.Sequential of Conv1d(k=1) + BatchNorm1d + ReLU layers with W ~ N(0, 1/K), an optional conv bias
    and non-trivial running statistics, gamma, beta and eps.  dead = [(layer, channel)]: that channel is
    zero-weighted with a negative folded bias, so its ReLU output is 0 at every point."""
    mods, k = [], F
    for li, n in enumerate(widths):
        conv = nn.Conv1d(k, n, 1, bias=bias)
        bn = nn.BatchNorm1d(n, eps=EPS)
        with torch.no_grad():
            conv.weight.copy_(torch.randn(n, k, 1, generator=g) / k ** 0.5)
            if bias:
                conv.bias.copy_(torch.randn(n, generator=g) * 0.1)
            bn.running_mean.copy_(torch.randn(n, generator=g) * 0.2)
            bn.running_var.copy_(torch.rand(n, generator=g) * 1.5 + 0.5)
            bn.weight.copy_(torch.rand(n, generator=g) + 0.5)
            bn.weight[::5] *= -1
            bn.bias.copy_(torch.randn(n, generator=g) * 0.2 + 0.1)
            for dl, dc in dead:
                if dl == li:
                    conv.weight[dc] = 0
                    if bias:
                        conv.bias[dc] = 0
                    bn.running_mean[dc] = 0
                    bn.bias[dc] = -0.5
                    bn.weight[dc] = abs(float(bn.weight[dc]))
        mods += [conv, bn, nn.ReLU()]
        k = n
    return nn.Sequential(*mods).eval()


def chain_layers(seq):
    """[(W [N, K], b | None, rm, rv, gamma, beta, eps)] as float64 CPU tensors."""
    out = []
    mods = list(seq.children())
    for i in range(0, len(mods), 3):
        conv, bn = mods[i], mods[i + 1]
        d = lambda t: None if t is None else t.detach().double().cpu()  # noqa: E731
        out.append((d(conv.weight)[:, :, 0], d(conv.bias), d(bn.running_mean), d(bn.running_var),
                    d(bn.weight), d(bn.bias), bn.eps))
    return out


def xy_transform(x, T, add_eye):
    """x [B, F, L] float64; (x0, x1) <- (x0, x1) (T + add_eye * I), T [B, 4] row-major 2x2."""
    if T is None:
        return x
    t = T.double().view(-1, 2, 2) + (torch.eye(2, dtype=torch.float64) if add_eye else 0)
    x = x.clone()
    x0, x1 = x[:, 0].clone(), x[:, 1].clone()
    x[:, 0] = x0 * t[:, 0, 0, None] + x1 * t[:, 1, 0, None]
    x[:, 1] = x0 * t[:, 0, 1, None] + x1 * t[:, 1, 1, None]
    return x


def ref_fp32(clouds, T, add_eye, layers):
    """Unfused float64 reference: transform, conv, BatchNorm (running statistics), ReLU, max over points."""
    a = xy_transform(clouds.double().cpu(), None if T is None else T.cpu(), add_eye).transpose(1, 2)
    for W, b, rm, rv, gm, bt, eps in layers:
        z = a @ W.t() + (0 if b is None else b)
        a = torch.relu((z - rm) / torch.sqrt(rv + eps) * gm + bt)
    return a.max(1).values


def round_bf16(x, mode="rne"):
    """float64 -> fp32 (nearest) -> bf16, to nearest even ("rne") or toward zero ("rtz"); back as float64."""
    f = x.float()
    if mode == "rne":
        return f.to(torch.bfloat16).double()
    bits = f.view(torch.int32) & ~0xFFFF
    return bits.view(torch.float32).double()


def tf32(x):
    """The kernel's tf32 split (to_tf32: round half away on the 13 dropped bits) of fp32 values."""
    bits = (x.float().view(torch.int32) + 0x1000) & ~0x1FFF
    return bits.view(torch.float32).double()


def folded(layers):
    """fp32 scale = gamma / sqrt(rv + eps) and the float64 folded bias b*s + beta - rm*s of each layer."""
    out = []
    for W, b, rm, rv, gm, bt, eps in layers:
        s32 = (gm.float() / torch.sqrt(rv.float() + eps)).double()
        s = gm / torch.sqrt(rv + eps)
        out.append((s32, (0 if b is None else b * s) + bt - rm * s))
    return out


def xy_transform_fp32(x, T, add_eye):
    """The kernel's fp32 transform: t = T + I in fp32, x0' = fmaf(x0, t00, fp32(x1 * t10)), likewise x1'.
    With few features one input whose bf16 rounding flips moves the output by ~2^-9, so the bf16 emulation
    rounds exactly where the kernel does (the fma as one rounding of the float64 sum)."""
    x = x.float().cpu()
    if T is None:
        return x.double()
    t = T.float().cpu().view(-1, 2, 2) + (torch.eye(2) if add_eye else 0)
    x0, x1 = x[:, 0].clone(), x[:, 1].clone()
    x = x.clone()
    for j in (0, 1):
        p = x1 * t[:, 1, j, None]
        x[:, j] = (x0.double() * t[:, 0, j, None].double() + p.double()).float()
    return x.double()


def emu_bf16(clouds, T, add_eye, layers, scales, biases, mode="rne"):
    """float64 emulation of the bf16 kernel's rounding (module docstring); scales / biases as the kernel
    got them (fp32)."""
    x = xy_transform_fp32(clouds, T, add_eye)
    a = round_bf16(x, mode).transpose(1, 2)
    for li, ((W, *_), s, bias) in enumerate(zip(layers, scales, biases)):
        Wb = round_bf16((W.float() * s.float()[:, None]).double(), mode)
        z = torch.relu(a @ Wb.t() + bias.double())
        a = z if li + 1 == len(layers) else round_bf16(z, mode)
    return a.max(1).values


def emu_1xtf32(clouds, T, add_eye, layers, scales, biases):
    """fp32 kernel with the lo terms dropped: one TF32 product per term, activations kept in fp32."""
    x = xy_transform(clouds.double().cpu(), None if T is None else T.cpu(), add_eye).float().double()
    a = x.transpose(1, 2)
    for (W, *_), s, bias in zip(layers, scales, biases):
        Wt = tf32((W.float() * s.float()[:, None]).double())
        a = torch.relu(tf32(a) @ Wt.t() + bias.double()).float().double()
    return a.max(1).values


def make_inputs(g, B, F, planted=False):
    """clouds [B, F, 128] and a per-superpoint T [B, 4].  planted: point b % 128 of cloud b is scaled up so
    that it holds the maximum of most channels."""
    x = torch.randn(B, F, 128, generator=g) * 0.5
    if planted:
        b = torch.arange(B)
        x[b, :, b % 128] = x[b, :, b % 128].abs() * 6 + 0.5
    T = torch.randn(B, 4, generator=g) * 0.3
    return x, T


def test_reference_bounds_can_fail():
    """The emulation-based bounds can fail: on the tests' own data, rounding toward zero instead of to
    nearest moves the bf16 emulation by more than BF16_TOL, and dropping the lo terms of 3xTF32 moves the
    fp32 result by more than FP32_TOL."""
    for i, w in enumerate(CHAINS):
        F, has_bias = _chain_case(i, w)
        g = _gen("chain", w)
        seq = make_chain(g, F, w, has_bias)
        clouds, T = make_inputs(g, 200, F)
        layers = chain_layers(seq)
        fl = folded(layers)
        scales = [s for s, _ in fl]
        biases = [bb.float() for _, bb in fl]
        want = ref_fp32(clouds, T, True, layers)
        scale = float(want.abs().max())
        rne = emu_bf16(clouds, T, True, layers, scales, biases)
        rtz = emu_bf16(clouds, T, True, layers, scales, biases, mode="rtz")
        assert float((rne - rtz).abs().max()) > 2 * BF16_TOL * float(rne.abs().max()), w
        one = emu_1xtf32(clouds, T, True, layers, scales, biases)
        assert float((one - want).abs().max()) > 5 * FP32_TOL * scale, w
        # and the rounding-to-nearest emulation of the kernel's own arithmetic is within bf16's reach of fp32
        assert float((rne - want).abs().max()) < 3e-2 * scale, w


# --------------------------------------------------------------------------------------------------
# GPU helpers
MEASURED = {}  # group -> largest error / tensor maximum seen (printed at the end of the module)


def check(group, got, want, rtol):
    got = torch.as_tensor(got).detach().double().cpu()
    want = torch.as_tensor(want).detach().double().cpu()
    assert got.shape == want.shape, (got.shape, want.shape)
    assert torch.isfinite(got).all(), "non-finite values"
    s = float(want.abs().max())
    err = float((got - want).abs().max())
    MEASURED[group] = max(MEASURED.get(group, 0.0), err / max(s, 1e-30))
    assert err <= rtol * s, "max err %g vs scale %g (rel %g)" % (err, s, err / max(s, 1e-30))


@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    yield torch.device("cuda:0")
    if MEASURED:
        print("\n[test_pointnet_fused] largest error / tensor maximum per group:")
        for k in sorted(MEASURED):
            print("  %-10s %.3e" % (k, MEASURED[k]))


def _prod_layers(seq):
    """The chain in the form the PointNet module hands to ops.pointnet_fused_image."""
    from superpoint_graph_b200.dense import parse_sequential
    from superpoint_graph_b200.spg_pointnet import _conv_layers
    specs, params = parse_sequential(seq, False)
    return _conv_layers(specs, params), specs, params


def fused(seq, clouds, T, bf16, add_eye=1, pooled=None, ldp=None):
    """Runs the chain through ops.pointnet_fused_image and the kernel; returns (pooled [B, N], image, bias)."""
    from superpoint_graph_b200 import _lib, ops
    layers, _, _ = _prod_layers(seq)
    F = clouds.shape[1]
    image, bias, widths = ops.pointnet_fused_image(layers, F, bf16=bf16)
    B, N = clouds.shape[0], int(widths[-1])
    if pooled is None:
        pooled = torch.empty((B, N), dtype=torch.float32, device=clouds.device)
        ldp = N
    if add_eye == 1:
        ops.pointnet_fused_eval(clouds, T, image, bias, widths, pooled, ldp)
    else:
        name = "spg_pointnet_fused_eval_bf16" if bf16 else "spg_pointnet_fused_eval"
        _lib.call(name, clouds, B, F, 128, T, add_eye, image, bias, int(widths.numel()), widths.data_ptr(),
                  pooled, ldp, _lib.current_stream())
    return pooled, image, bias


def _scales(seq, dev):
    """fp32 BatchNorm scales as the library's fold computes them (the scale the packers multiply by)."""
    from superpoint_graph_b200 import ops
    out = []
    mods = list(seq.children())
    for i in range(0, len(mods), 3):
        bn = mods[i + 1]
        s, _ = ops.bn_fold(bn.running_mean, bn.running_var, bn.weight, bn.bias, bn.eps)
        out.append(s.double().cpu())
    return out


def run_case(dev, group, seq, clouds, T, bf16, add_eye=1):
    """Kernel vs its reference (fp32: float64 unfused; bf16: float64 emulation); returns the kernel's result."""
    layers = chain_layers(seq)
    got, _, bias = fused(seq, clouds.to(dev), None if T is None else T.to(dev), bf16, add_eye)
    if bf16:
        widths = [l[0].shape[0] for l in layers]
        biases = list(bias.cpu().split(widths))
        want = emu_bf16(clouds, T, add_eye, layers, _scales(seq, dev), biases)
        check(group, got, want, BF16_TOL)
    else:
        want = ref_fp32(clouds, T, add_eye, layers)
        check(group, got, want, FP32_TOL)
    return got, want


# --------------------------------------------------------------------------------------------------
# every CHAINS row
@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("widths", CHAINS, ids=[chain_id(w) for w in CHAINS])
def test_chain(dev, widths, bf16):
    F, has_bias = _chain_case(CHAINS.index(widths), widths)
    g = _gen("chain", widths)
    seq = make_chain(g, F, widths, has_bias)
    clouds, T = make_inputs(g, 200, F)
    run_case(dev, "bf16" if bf16 else "fp32", seq.to(dev), clouds, T, bf16)


@pytest.mark.gpu
@pytest.mark.parametrize("widths", CHAINS, ids=[chain_id(w) for w in CHAINS])
def test_chain_matches_layered_path(dev, widths, monkeypatch):
    """The fused kernel and the layer-by-layer eval path (GEMMs, deferred BatchNorm/ReLU, segmented max-pool)
    on the same chain and clouds agree to 2e-5; the fused kernel ran exactly once, the layered path never."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_pointnet import _Clouds, _pool
    F, has_bias = _chain_case(CHAINS.index(widths), widths)
    g = _gen("layered", widths)
    seq = make_chain(g, F, widths, has_bias).to(dev)
    clouds, T = make_inputs(g, 150, F)
    clouds, T = clouds.to(dev), T.to(dev)
    _, specs, params = _prod_layers(seq)
    out = {}
    for fz in (True, False):
        pooled = torch.empty((150, widths[-1]), dtype=torch.float32, device=dev)
        ops.prof_reset()
        _pool(_Clouds(clouds), T, specs, params, False, fz, pooled)
        assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == int(fz)
        out[fz] = pooled
    close(out[True], out[False], 2e-5)


# --------------------------------------------------------------------------------------------------
# packers and the folded bias
def _unswizzle_bf16(img, N, K):
    """[K/64][N][64] SWIZZLE_128B bf16 image (int16 bits) -> [N, K] (a Python copy of sw128_off)."""
    n = torch.arange(N)[:, None]
    k = torch.arange(K)[None, :]
    kc, kk = k // 64, k % 64
    c16 = kk >> 3
    off = (n >> 3) * 1024 + (n & 7) * 128 + ((c16 ^ (n & 7)) << 4)
    idx = kc * N * 64 + (off >> 1) + (kk & 7)
    return img.view(torch.int16).cpu()[idx]


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,kv,ldw,scaled", [
    (64, 64, 64, 64, False), (128, 64, 9, 9, True), (32, 64, 14, 17, True), (256, 128, 128, 131, False),
    (128, 128, 100, 128, True), (64, 64, 32, 32, True), (8, 192, 150, 160, True)])
def test_pack_weights_bf16(dev, N, K, kv, ldw, scaled):
    """spg_tc_pack_weights_bf16 unswizzled equals bf16(fp32(W * scale)) bit for bit; K padding is +0."""
    from superpoint_graph_b200 import _lib
    g = _gen("pack", N, K, kv, ldw, scaled)
    W = torch.randn(N, ldw, generator=g)
    W[:, kv:] = float("nan")  # never read
    s = (torch.rand(N, generator=g) * 3 - 1.5) if scaled else None
    img = torch.full((N * K,), float("nan"), dtype=torch.bfloat16, device=dev)
    _lib.call("spg_tc_pack_weights_bf16", W.to(dev), ldw, None if s is None else s.to(dev), N, K, kv, img,
              _lib.current_stream())
    want = torch.zeros(N, K, dtype=torch.float32)
    want[:, :kv] = W[:, :kv] * (s[:, None] if scaled else 1.0)
    assert torch.equal(_unswizzle_bf16(img, N, K), want.to(torch.bfloat16).view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("has_bias", [True, False], ids=["bias", "nobias"])
def test_fused_image_bias_and_bf16_image(dev, has_bias):
    """pointnet_fused_image's folded bias is b*s + beta - rm*s (float64, to fp32 rounding); its bf16 image
    holds every layer's bf16(fp32(W * s)) bit for bit, including the 64-wide K chunk after a 32-wide layer,
    whose upper half must be zeros."""
    from superpoint_graph_b200 import ops
    widths = (32, 128, 32, 64)
    F = 11
    seq = make_chain(_gen("image", has_bias), F, widths, has_bias).to(dev)
    layers, _, _ = _prod_layers(seq)
    ref = chain_layers(seq)
    want_bias = torch.cat([bb for _, bb in folded(ref)])
    for bf16 in (False, True):
        image, bias, _ = ops.pointnet_fused_image(layers, F, bf16=bf16)
        close(bias, want_bias, 1e-6)
    scales = _scales(seq, dev)
    row, K = 0, 64
    for (W, *_), s in zip(ref, scales):
        N, kv = W.shape
        blk = image[row * 64:(row + (K // 64) * N) * 64]
        want = torch.zeros(N, K, dtype=torch.float32)
        want[:, :kv] = W.float() * s.float()[:, None]
        assert torch.equal(_unswizzle_bf16(blk, N, K), want.to(torch.bfloat16).view(torch.int16)), (N, K, kv)
        row += (K // 64) * N
        K = max(N, 64)
    assert row == bf16_image_rows(widths)


# --------------------------------------------------------------------------------------------------
# features, transform, batch sizes, argmax positions, write set
@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("tmode", ["noT", "eye1", "eye0"])
@pytest.mark.parametrize("F", [1, 2, 3, 9, 11, 14, 15, 16])
def test_features_and_transform(dev, F, tmode, bf16):
    """Every feature count with T = None, T + I and T alone; each superpoint has its own T, so a wrong cloud
    index for T fails."""
    if F == 1 and tmode != "noT":
        pytest.skip("T needs two features (test_abi_errors checks that it is refused)")
    g = _gen("features", F, tmode)
    seq = make_chain(g, F, (64, 128), True).to(dev)
    clouds, T = make_inputs(g, 140, F)
    T = None if tmode == "noT" else T * 3
    run_case(dev, "bf16" if bf16 else "fp32", seq, clouds, T, bf16, add_eye=0 if tmode == "eye0" else 1)


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("widths", [(64, 32, 128), (32, 64)], ids=chain_id)
@pytest.mark.parametrize("B", [1, 2, 131, 132, 133, 265, 5000])
def test_batch_sizes(dev, B, widths, bf16):
    """Up to 38 superpoints per CTA: both weight rings (2 fp32 stages, 8 bf16 stages) and the input double
    buffer wrap their mbarrier phases many times."""
    g = _gen("batch", B, widths)
    seq = make_chain(g, 9, widths, True).to(dev)
    clouds, T = make_inputs(g, B, 9)
    run_case(dev, "bf16" if bf16 else "fp32", seq, clouds, T, bf16)


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("widths,dead", [
    ((64, 64, 128, 128, 256), [(4, 3), (4, 200), (4, 255)]),
    ((32, 64), [(0, 5), (1, 0), (1, 63)]),
    ((128, 32), [(1, 31)]),
], ids=["s3dis", "stn-vkitti-inner-dead", "last32"])
def test_argmax_positions_and_dead_channels(dev, widths, dead, bf16):
    """The maximum of cloud b sits at point b % 128 for many channels, so across 256 clouds every row, warp
    and warpgroup of the CTA wins the cross-warp max-pool; channels dead at every point pool to exactly 0."""
    g = _gen("argmax", widths)
    seq = make_chain(g, 14, widths, True, dead=dead).to(dev)
    clouds, T = make_inputs(g, 256, 14, planted=True)
    got, _ = run_case(dev, "bf16" if bf16 else "fp32", seq, clouds, T, bf16)
    layers = chain_layers(seq)
    a = xy_transform(clouds.double(), T, True).transpose(1, 2)
    for W, b, rm, rv, gm, bt, eps in layers:
        a = torch.relu((a @ W.t() + (0 if b is None else b) - rm) / torch.sqrt(rv + eps) * gm + bt)
    arg = a.argmax(1)  # [B, N]
    won = arg == (torch.arange(256) % 128)[:, None]
    assert won.any(1).all(), "a planted point holds no channel's maximum"
    assert won.double().mean() > 0.1, float(won.double().mean())
    for dl, dc in dead:
        if dl == len(widths) - 1:
            assert torch.equal(got[:, dc].cpu(), torch.zeros(256)), dc


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("extra", [4, 5])
def test_write_set(dev, extra, bf16):
    """pooled as the column slice [:, :N] of a NaN-filled buffer with ldp = N + extra, as the PointNet does
    when global features follow: columns from N on and a sentinel row after the last cloud stay NaN."""
    widths, B, F = (64, 128), 133, 14
    g = _gen("writeset", extra)
    seq = make_chain(g, F, widths, True).to(dev)
    clouds, T = make_inputs(g, B, F)
    N, ldp = widths[-1], widths[-1] + extra
    buf = torch.full(((B + 1) * ldp,), float("nan"), dtype=torch.float32, device=dev)
    pooled = buf[:B * ldp].view(B, ldp)[:, :N]
    fused(seq, clouds.to(dev), T.to(dev), bf16, pooled=pooled, ldp=ldp)
    full = buf.cpu()[:B * ldp].view(B, ldp)
    assert torch.isnan(full[:, N:]).all() and torch.isnan(buf.cpu()[B * ldp:]).all()
    want = ref_fp32(clouds, T, True, chain_layers(seq))
    close(full[:, :N], want, 3e-2 if bf16 else FP32_TOL)


# --------------------------------------------------------------------------------------------------
# determinism, kernel identity, argument checks
@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_deterministic_and_counted(dev, bf16):
    """Two launches give bit-identical results; the profiler counts exactly the launches made."""
    from superpoint_graph_b200 import ops
    g = _gen("determinism")
    seq = make_chain(g, 14, (64, 64, 128, 128, 256), True).to(dev)
    clouds, T = make_inputs(g, 1000, 14)
    clouds, T = clouds.to(dev), T.to(dev)
    fused(seq, clouds, T, bf16)  # folds the image
    ops.prof_reset()
    a, _, _ = fused(seq, clouds, T, bf16)
    b, _, _ = fused(seq, clouds, T, bf16)
    c, _, _ = fused(seq, clouds, T, bf16)
    torch.cuda.synchronize()
    assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 3
    assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_abi_errors(dev, bf16):
    """Return codes of both entry points; none of the refused calls and no n_clouds = 0 call launches."""
    from superpoint_graph_b200 import _lib, ops
    L = _lib.lib()
    fn = L.spg_pointnet_fused_eval_bf16 if bf16 else L.spg_pointnet_fused_eval
    F, B = 9, 4
    seq = make_chain(_gen("abi"), F, (64, 128), True).to(dev)
    layers, _, _ = _prod_layers(seq)
    image, bias, widths = ops.pointnet_fused_image(layers, F, bf16=bf16)
    clouds = torch.zeros(B * 17 * 128 + 4, dtype=torch.float32, device=dev)
    T = torch.zeros(B, 4, dtype=torch.float32, device=dev)
    pooled = torch.empty(B, 256, dtype=torch.float32, device=dev)
    st = _lib.current_stream()

    def call(n_clouds=B, F=F, npts=128, T=None, w=(64, 128), ldp=128, cl=None):
        wt = torch.tensor(list(w), dtype=torch.int32)
        return fn(clouds.data_ptr() if cl is None else cl, n_clouds, F, npts, None if T is None else T.data_ptr(),
                  1, image.data_ptr(), bias.data_ptr(), len(w), wt.data_ptr(), pooled.data_ptr(), ldp, st)

    ops.prof_reset()
    assert call(w=(256, 128)) == SPG_E_UNSUPPORTED
    assert call(w=(64,) * 7) == SPG_E_UNSUPPORTED
    assert call(F=17) == SPG_E_UNSUPPORTED
    assert call(npts=127) == SPG_E_UNSUPPORTED
    assert call(npts=129) == SPG_E_UNSUPPORTED
    assert call(ldp=127) == SPG_E_BADARG
    assert call(n_clouds=-1) == SPG_E_BADARG
    assert call(F=1, T=T) == SPG_E_BADARG
    assert call(cl=clouds.data_ptr() + 4) == SPG_E_ALIGN
    assert call(n_clouds=0) == SPG_OK
    torch.cuda.synchronize()
    assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 0
    assert call(F=1) == SPG_OK and call(F=2, T=T) == SPG_OK
    torch.cuda.synchronize()
    assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 2


# --------------------------------------------------------------------------------------------------
# the folded-image cache never serves weights or statistics older than the model's
def _trainer(dev, seed=5):
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    w = workloads.get("vkitti_eval", nodes=400)
    torch.manual_seed(seed)
    model = create_model(w["margs"])
    with torch.no_grad():
        model.ptn.stn.proj.weight.normal_(0, 0.05)
    model.to(dev)
    tr = Trainer(model, w["margs"])
    db = HostBatch(workloads.batch(w, seed)).to_device(dev)
    return tr, db


def _eval(tr, db, bf16):
    from superpoint_graph_b200 import ops
    tr.dtype = "bf16" if bf16 else "f32"
    try:
        ops.prof_reset()
        out = tr.eval_step(db).clone()
        torch.cuda.synchronize()
        assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 2  # STN chain + main chain, fused
        return out
    finally:
        tr.dtype = "f32"


def _changed(a, b):
    return float((a - b).abs().max()) > 1e-3 * float(b.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_eval_after_training_step(dev, bf16, monkeypatch):
    """eval_step -> train_step -> eval_step: the second eval uses the updated weights and running statistics:
    it equals an eval from a freshly folded image (bit for bit) and, in fp32, the layered path to 2e-5."""
    from superpoint_graph_b200 import ops
    tr, db = _trainer(dev)
    before = _eval(tr, db, bf16)
    tr.train_step(db)
    after = _eval(tr, db, bf16)
    assert _changed(after, before)
    ops._FUSED_IMAGES.clear()
    refolded = _eval(tr, db, bf16)
    assert torch.equal(after, refolded)
    if not bf16:
        monkeypatch.setattr(ops, "USE_FUSED_EVAL", [False])
        close(after, tr.eval_step(db), 2e-5)


@pytest.mark.gpu
def test_eval_after_training_forward_updates_statistics(dev):
    """net.eval() forward, one net.train() forward on other clouds (updates only the running statistics), then
    net.eval() again: the result follows the updated statistics (oracle with the module's new state)."""
    from oracle import nets_ref
    from superpoint_graph_b200 import ops, spg_pointnet
    F = 9
    net = spg_pointnet.PointNet([64, 64, 128], [64, 32, 32], [32, 64], [32, 16], F, F, prelast_do=0)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
    net.to(dev)
    g = _gen("running-stats")
    x, xg = torch.randn(300, F, 128, generator=g) * 0.4, torch.rand(300, generator=g) * 3
    x2 = torch.randn(300, F, 128, generator=g) * 0.8 + 0.3
    pcfg = dict(n_conv=3, n_fc=3, n_conv_stn=2, n_fc_stn=2, nfeat_stn=F)
    net.eval()
    with torch.no_grad():
        before = net(x.to(dev), xg.to(dev)).clone()
        net.train()
        net(x2.to(dev), xg.to(dev))
        net.eval()
        ops.prof_reset()
        after = net(x.to(dev), xg.to(dev))
        assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 2
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    want = nets_ref.pointnet_forward(x, xg, sd, pcfg, False)
    assert _changed(after.cpu(), before.cpu())
    close(after, want, 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_captured_eval_graph_after_training_step(dev, bf16):
    """capture_eval -> train_step -> replay_eval: the replay gives what a fresh eager eval gives, never the
    pre-step logits (or it raises)."""
    tr, db = _trainer(dev, seed=8)
    tr.dtype = "bf16" if bf16 else "f32"
    try:
        key = tr.capture_eval(db, warmup=1)
        pre = tr.replay_eval(key).clone()
    finally:
        tr.dtype = "f32"
    tr.train_step(db)
    tr.dtype = "bf16" if bf16 else "f32"
    try:
        replayed = tr.replay_eval(key).clone()
    finally:
        tr.dtype = "f32"
    from superpoint_graph_b200 import ops
    ops._FUSED_IMAGES.clear()  # the eager reference folds its own image from the current weights
    fresh = _eval(tr, db, bf16)
    assert _changed(fresh, pre)
    close(replayed, fresh, 1e-6)


@pytest.mark.gpu
def test_new_model_at_freed_addresses(dev):
    """Model A is evaluated and freed; model B (same architecture, other weights) is built in the same order in
    the same private memory pool, so its tensors land at A's addresses.  B's eval must follow B's weights."""
    from oracle import nets_ref
    from superpoint_graph_b200 import spg_pointnet
    F = 9
    pcfg = dict(n_conv=3, n_fc=3, n_conv_stn=2, n_fc_stn=2, nfeat_stn=F)
    g = _gen("address-reuse")
    x, xg = torch.randn(200, F, 128, generator=g) * 0.4, torch.rand(200, generator=g) * 3
    xd, xgd = x.to(dev), xg.to(dev)
    pool = torch.cuda.MemPool()

    def build(seed):
        net = spg_pointnet.PointNet([64, 64, 128], [64, 32, 32], [32, 64], [32, 16], F, F, prelast_do=0)
        torch.manual_seed(seed)
        with torch.no_grad():
            net.stn.proj.weight.normal_(0, 0.05)
            for m in net.modules():
                if isinstance(m, nn.Conv1d):
                    m.weight.normal_(0, 0.3)
                if isinstance(m, nn.BatchNorm1d):
                    m.running_mean.normal_(0, 0.3)
                    m.running_var.uniform_(0.5, 1.5)
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        with torch.cuda.use_mem_pool(pool):
            net.to(dev)
        return net.eval(), sd

    def ptrs(net):
        return [t.data_ptr() for t in list(net.parameters()) + list(net.buffers())]

    a, sd_a = build(1)
    with torch.no_grad():
        out_a = a(xd, xgd).cpu()
    close(out_a, nets_ref.pointnet_forward(x, xg, sd_a, pcfg, False), 1e-4)
    where = ptrs(a)
    del a
    gc.collect()
    b, sd_b = build(2)
    if ptrs(b) != where:
        pytest.skip("the allocator placed model B elsewhere: the address-reuse case did not arise")
    with torch.no_grad():
        out_b = b(xd, xgd).cpu()
    del b
    gc.collect()
    assert _changed(out_b, out_a)
    close(out_b, nets_ref.pointnet_forward(x, xg, sd_b, pcfg, False), 1e-4)
