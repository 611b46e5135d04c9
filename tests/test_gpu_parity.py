"""GPU parity: every kernel, called through the C-ABI, against the reference's golden vectors and
the pinned oracle.  Tolerances: index/segment outputs bit-exact; fp32 within 1e-4 relative (the
bound BASELINE.json's north_star states), fp64 within 1e-10."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ecc_ref, nets_ref  # noqa: E402  (checker only)

RTOL = 1e-4


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


def t(a, dev=None):
    x = torch.from_numpy(np.asarray(a))
    return x.to(dev) if dev is not None else x


def sub(d, prefix):
    return {k[len(prefix):]: t(v).clone() for k, v in d.items() if k.startswith(prefix)}


def close(a, b, rtol=RTOL, atol=0.0):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all(), "non-finite values"
    err = (a - b).abs().max().item()
    scale = b.abs().max().item()
    assert err <= atol + rtol * scale, "max err %g vs scale %g (rel %g)" % (err, scale, err / max(scale, 1e-30))


def close_grads(got, want, rtol=RTOL):
    floor = 1e-5 * max(float(torch.as_tensor(v).abs().max()) for v in want.values())
    for k, v in want.items():
        assert got[k] is not None, "missing gradient for %s" % k
        close(got[k], v, rtol, floor)


@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()  # fail loudly if the extension is missing
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------ ECC
def test_ecc_unit_fixture_fp64(golden_dir, dev):
    """The reference's unit-test scenario (strided output, zero-degree node, idxe) in double."""
    from superpoint_graph_b200.spg_ecc import GraphConvFunction
    g = load(golden_dir, "ecc_unit.npz")
    x, w, idxn, degs = t(g["x"], dev), t(g["w"], dev), t(g["idxn"]), t(g["degs"])
    for lim in (30, 1, 1e10):
        out = GraphConvFunction.apply(x, w, 10, 15, idxn.to(dev), None, degs, degs.to(dev), lim)
        close(out, g["out"], 1e-10)
    assert torch.all(out[1] == 0)
    oute = GraphConvFunction.apply(x, t(g["w30"], dev), 10, 15, idxn.to(dev), t(g["idxe"], dev), degs, degs.to(dev), 30)
    close(oute, g["out_idxe"], 1e-10)
    xv, wv = t(g["xv"], dev).requires_grad_(True), t(g["wv"], dev).requires_grad_(True)
    outv = GraphConvFunction.apply(xv, wv, 10, 10, idxn.to(dev), None, degs, degs.to(dev), 30)
    close(outv, g["outv"], 1e-10)
    outv.backward(t(g["gv"], dev))
    close(xv.grad, g["gxv"], 1e-10)
    close(wv.grad, g["gwv"], 1e-10)


def test_ecc_gradcheck_fp64(dev):
    from superpoint_graph_b200.spg_ecc import GraphConvFunction
    torch.manual_seed(0)
    n, e, cin, cout = 20, 50, 10, 15
    degs = torch.LongTensor([5, 0, 15, 20, 10])
    idxn = torch.randint(0, n, (e,))
    x = torch.randn(n, cin, dtype=torch.float64, device=dev, requires_grad=True)
    w = torch.randn(e, cin, cout, dtype=torch.float64, device=dev, requires_grad=True)
    f = lambda a, b: GraphConvFunction.apply(a, b, cin, cout, idxn.to(dev), None, degs, degs.to(dev), 30)
    assert torch.autograd.gradcheck(f, (x, w))
    idxe = torch.randint(0, 30, (e,))
    w30 = torch.randn(30, cin, cout, dtype=torch.float64, device=dev, requires_grad=True)
    f = lambda a, b: GraphConvFunction.apply(a, b, cin, cout, idxn.to(dev), idxe.to(dev), degs, degs.to(dev), 30)
    # with idxe the filter gradient is accumulated with atomics (order-dependent rounding)
    assert torch.autograd.gradcheck(f, (x, w30), nondet_tol=1e-10)
    wv = torch.randn(e, cin, dtype=torch.float64, device=dev, requires_grad=True)
    f = lambda a, b: GraphConvFunction.apply(a, b, cin, cin, idxn.to(dev), None, degs, degs.to(dev), 30)
    assert torch.autograd.gradcheck(f, (x, wv))


def test_ecc_fast_paths_golden(golden_dir, dev):
    from superpoint_graph_b200.spg_ecc import GraphConvFunction
    g = load(golden_dir, "ecc_spg.npz")
    idxn, degs = t(g["idxn"]), t(g["degs"])
    x = t(g["x"], dev).requires_grad_(True)
    wv = t(g["wv"], dev).requires_grad_(True)
    out = GraphConvFunction.apply(x, wv, 32, 32, idxn.to(dev), None, degs, degs.to(dev))
    close(out, g["out"])
    out.backward(t(g["g"], dev))
    close(x.grad, g["gx"])
    close(wv.grad, g["gw"])
    outm = GraphConvFunction.apply(x.detach(), t(g["wm"], dev), 32, 32, idxn.to(dev), None, degs, degs.to(dev))
    close(outm, g["outm"])
    for i in (3, 17, 90):
        assert torch.all(out[i] == 0) and torch.all(outm[i] == 0)


@pytest.mark.parametrize("mat", [False, True])
@pytest.mark.parametrize("n_iter", [1, 3])
def test_ecc_fast_vs_oracle(dev, mat, n_iter):
    """Random graph with heavy-tailed degrees: forward, grad_x (+ fused addends) and the batched
    filter gradient against the oracle."""
    from superpoint_graph_b200 import ops
    rng = np.random.default_rng(3)
    N, H = 700, 32
    degs_np = np.minimum(rng.geometric(0.12, size=N) - 1, 200)
    degs_np[:5] = 0
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn = torch.from_numpy(rng.integers(0, N, size=E).astype(np.int64))
    graph = ops.EccGraph(idxn, None, degs, n_in=N)
    torch.manual_seed(1)
    xs = torch.randn(n_iter, N, H)
    gs = torch.randn(n_iter, N, H)
    w = torch.randn(E, H, H) * 0.2 if mat else torch.randn(E, H)
    out = ops.ecc_fwd(xs[0].to(dev), w.to(dev), graph, H)
    close(out, ecc_ref.graph_conv_forward(xs[0], w, idxn, None, degs))
    a0, a1 = torch.randn(N, H), torch.randn(N, H)
    gx = ops.ecc_bwd_x(w.to(dev), gs[0].to(dev), graph, H, add0=a0.to(dev), add1=a1.to(dev))
    rgx, _ = ecc_ref.graph_conv_backward(xs[0], w, idxn, None, degs, gs[0])
    close(gx, rgx + a0 + a1)
    gw = ops.ecc_bwd_w(xs.to(dev), gs.to(dev), graph, tuple(w.shape), n_iter=n_iter)
    rgw = sum(ecc_ref.graph_conv_backward(xs[r], w, idxn, None, degs, gs[r])[1] for r in range(n_iter))
    close(gw, rgw)
    gw2 = ops.ecc_bwd_w(xs.to(dev), gs.to(dev), graph, tuple(w.shape), n_iter=n_iter, out=gw.clone(), accumulate=True)
    close(gw2, 2 * rgw)


def test_ecc_full_size_properties(dev):
    """Config-5 scale (100k superpoints, ~1M edges): size-independent properties — linearity in x,
    zero rows for zero-degree nodes, agreement with a torch index_add_ formulation on the device,
    <grad_x, x> == <g, out> (adjointness)."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    b = make_batch(n_nodes=100000, k=7, seed=2)
    N, E, H = b["degs"].numel(), b["idxn"].numel(), 32
    graph = ops.EccGraph(b["idxn"], None, b["degs"], n_in=N)
    torch.manual_seed(0)
    x1, x2 = torch.randn(N, H, device=dev), torch.randn(N, H, device=dev)
    w = torch.randn(E, H, device=dev)
    o1, o2, o12 = (ops.ecc_fwd(v, w, graph, H) for v in (x1, x2, x1 + x2))
    close(o12, o1 + o2, 1e-5)
    zero = (b["degs"] == 0).to(dev)
    assert zero.any() and torch.all(o1[zero] == 0)
    idxn, degs = b["idxn"].to(dev), b["degs"].to(dev)
    tgt = torch.repeat_interleave(torch.arange(N, device=dev), degs)
    ref = torch.zeros(N, H, device=dev).index_add_(0, tgt, x1[idxn] * w) / degs.clamp(min=1).unsqueeze(1)
    close(o1, ref, 1e-5)
    g = torch.randn(N, H, device=dev)
    gx = ops.ecc_bwd_x(w, g, graph, H)
    lhs, rhs = (gx.double() * x1.double()).sum(), (g.double() * o1.double()).sum()
    assert abs(lhs - rhs) <= 1e-6 * abs(rhs) + 1e-3
    gw = ops.ecc_bwd_w(x1, g, graph, (E, H))
    close(gw, x1[idxn] * (g / degs.clamp(min=1).unsqueeze(1))[tgt], 1e-5)


# ------------------------------------------------------------------------------------ GRU
@pytest.mark.parametrize("name,ln,ig", [("gru.npz", True, True), ("gru_plain.npz", False, False)])
def test_gru_cell_golden(golden_dir, dev, name, ln, ig):
    from superpoint_graph_b200.spg_modules import GRUCellEx
    g = load(golden_dir, name)
    cell = GRUCellEx(32, 32, bias=True, layernorm=ln, ingate=ig)
    cell.load_state_dict(sub(g, "sd."))
    cell.to(dev)
    x, h = t(g["x"], dev).requires_grad_(True), t(g["h"], dev).requires_grad_(True)
    hy = cell(x, h)
    close(hy, g["hy"])
    hy.backward(t(g["g"], dev))
    close(x.grad, g["gx"])
    close(h.grad, g["gh"])
    close_grads({k: p.grad for k, p in cell.named_parameters()}, sub(g, "grad."))


# ---------------------------------------------------------------------------------- dense
@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (257, 70, 13), (1000, 64, 14), (300, 257, 260), (4096, 32, 64)])
def test_gemm_layouts(dev, M, N, K):
    from superpoint_graph_b200 import ops
    torch.manual_seed(M + N + K)
    A = torch.randn(M, K, dtype=torch.float64)
    B = torch.randn(N, K, dtype=torch.float64)
    bias = torch.randn(N, dtype=torch.float64)
    ref = A @ B.t() + bias
    Af, Bf, bf = A.float().to(dev), B.float().to(dev), bias.float().to(dev)
    close(ops.gemm(Af, K, True, Bf, K, True, M, N, K, bias=bf), ref, 1e-5)
    close(ops.gemm(Af.t().contiguous(), M, False, Bf, K, True, M, N, K, bias=bf), ref, 1e-5)
    close(ops.gemm(Af, K, True, Bf.t().contiguous(), N, False, M, N, K, bias=bf), ref, 1e-5)
    close(ops.gemm(Af.t().contiguous(), M, False, Bf.t().contiguous(), N, False, M, N, K, bias=bf), ref, 1e-5)
    for split in (2, 5):
        close(ops.gemm(Af, K, True, Bf, K, True, M, N, K, bias=bf, split_k=split), ref, 1e-5)


def test_gemm_prologues_and_reduction(dev):
    from superpoint_graph_b200 import ops
    torch.manual_seed(9)
    M, N, K = 3000, 48, 100
    A = torch.randn(M, K, dtype=torch.float64)
    B = torch.randn(N, K, dtype=torch.float64)
    sc, sh = torch.rand(K, dtype=torch.float64) + 0.5, torch.randn(K, dtype=torch.float64)
    ref = torch.relu(A * sc + sh) @ B.t()
    out = ops.gemm(A.float().to(dev), K, True, B.float().to(dev), K, True, M, N, K,
                   a_aff=(sc.float().to(dev), sh.float().to(dev), True))
    close(out, ref, 1e-5)
    # weight-gradient shape: dW[N_out, K_out] = dY^T [N_out, M] * relu(aff(P))[M, K_out]
    dY, P = torch.randn(M, N, dtype=torch.float64), torch.randn(M, K, dtype=torch.float64)
    ref = dY.t() @ torch.relu(P * sc + sh)
    out = ops.gemm(dY.float().to(dev), N, False, P.float().to(dev), K, False, N, K, M,
                   b_aff=(sc.float().to(dev), sh.float().to(dev), True))
    close(out, ref, 1e-5)


@pytest.mark.parametrize("M,C", [(5000, 70), (4999, 64), (1031, 32), (777, 16), (3000, 96), (2500, 256)])
def test_colsum_bn_fold_and_bn_backward(dev, M, C):
    """Column sums, the BatchNorm fold and running statistics, the BatchNorm/ReLU forward and backward
    against nn.BatchNorm1d, from batch statistics computed in float64.  C = 70: one float per lane
    (V = 1); C % 4 == 0: V = 4, with the warp folded over several rows for the narrow power-of-two
    widths (64, 32, 16) and spanning 128 columns otherwise."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(2)
    Y = (torch.randn(M, C, dtype=torch.float64) * 3 + 100)  # large mean: cancellation-prone
    Yf = Y.float().to(dev)
    mean, var = Yf.double().mean(0).float(), Yf.double().var(0, unbiased=False).float()
    close(ops.colsum(Yf, C, M, C), Yf.double().sum(0), 1e-6)
    gamma, beta = torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev)
    gamma[::4] *= -1
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    nbt = torch.zeros((), dtype=torch.long, device=dev)
    scale, shift = ops.bn_fold(mean, var, gamma, beta, 1e-5, rm, rv, 0.1, M, nbt)
    bn = torch.nn.BatchNorm1d(C).to(dev)
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
    Yr = Yf.clone().requires_grad_(True)
    a = torch.relu(bn(Yr))
    close(ops.affine_act(Yf, C, M, C, scale, shift, True), a, 1e-5, 1e-6)
    close(rm, bn.running_mean, 1e-5)
    close(rv, bn.running_var, 1e-5)
    assert int(nbt) == 1
    G = torch.randn(M, C, device=dev)
    a.backward(G)
    s12 = ops.act_bwd_reduce(G, C, Yf, C, scale, shift, mean, var, 1e-5, True, M, C)
    s1, s2 = s12[:C], s12[C:]
    close(s1, bn.bias.grad, 1e-4, 1e-5)
    close(s2, bn.weight.grad, 1e-4, 1e-4)
    dY = ops.act_bwd_apply(G, C, Yf, C, scale, shift, mean, var, 1e-5, True, True, s1, s2, M, C)
    close(dY, Yr.grad, 1e-4, 1e-6)


@pytest.mark.parametrize("C", [16, 64])
@pytest.mark.parametrize("p", [None, 0.3])
@pytest.mark.parametrize("force", ["ld", "offset"])
def test_bn_act_one_float_per_lane_at_widths_divisible_by_4(dev, C, p, force):
    """A leading dimension of C + 1 or a pointer one float off 16 bytes runs the V = 1 kernels at
    C % 4 == 0.  affine_act and act_bwd_apply give the bits of the V = 4 kernels on the same data;
    act_bwd_reduce and colsum match float64."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(5)
    M, eps = 3001, 1e-5

    def v1(X):  # the values of X in a layout that only V = 1 accepts: (tensor, leading dimension)
        if force == "ld":
            P = torch.full((M, C + 1), float("nan"), device=dev)
            P[:, :C] = X
            return P, C + 1
        return torch.empty(M * C + 1, device=dev)[1:].view(M, C).copy_(X), C

    Y = torch.randn(M, C, device=dev) * 2 + 0.5
    G = torch.randn(M, C, device=dev)
    (Y1, ld1), (G1, _) = v1(Y), v1(G)
    scale, shift = torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev)
    mean, var = Y.double().mean(0).float(), Y.double().var(0, unbiased=False).float()
    drop = None if p is None else (p, torch.tensor([0x5EED, 17], dtype=torch.int64, device=dev))

    a4 = ops.affine_act(Y, C, M, C, scale, shift, True, drop=drop)
    assert torch.equal(ops.affine_act(Y1, ld1, M, C, scale, shift, True, drop=drop), a4)
    close(ops.colsum(Y1, ld1, M, C), Y.double().sum(0), 1e-6)

    s12 = ops.act_bwd_reduce(G1, ld1, Y1, ld1, scale, shift, mean, var, eps, True, M, C, drop=drop)
    g = G.double()
    if drop is not None:
        g = g * ops.dropout_mask(drop[1], p, M, C).double() / (1 - np.float32(p))
    Yd = Y.double()
    g = g * (Yd * scale.double() + shift.double() > 0)
    xhat = (Yd - mean.double()) / torch.sqrt(var.double() + np.float32(eps))
    close(s12[:C], g.sum(0), 1e-4, 1e-5)
    close(s12[C:], (g * xhat).sum(0), 1e-4, 1e-4)

    s1, s2 = s12[:C], s12[C:]
    d4 = ops.act_bwd_apply(G, C, Y, C, scale, shift, mean, var, eps, True, True, s1, s2, M, C, drop=drop)
    d1 = ops.act_bwd_apply(G1, ld1, Y1, ld1, scale, shift, mean, var, eps, True, True, s1, s2, M, C,
                           drop=drop)
    assert torch.equal(d1, d4)


def csr_seg(lens, dev):
    """Segment description (B, L, offsets, row_seg) of CSR segments of the given lengths."""
    lens = torch.as_tensor(lens, dtype=torch.int64)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)])
    row_seg = torch.repeat_interleave(torch.arange(len(lens), dtype=torch.int32), lens)
    return len(lens), 0, offsets.to(dev), row_seg.to(dev)


@pytest.mark.parametrize("L,C,layout", [
    pytest.param(L, C, layout, id="%d-%d%s" % (L, C, "-csr" if layout == "csr" else ""))
    for layout in ("fixed", "csr") for L, C in [(128, 70), (128, 64), (128, 256), (20, 132), (7, 8)]])
def test_segmax_and_cloud_rows(dev, L, C, layout):
    """C = 70: scalar pooling kernel; C % 4 == 0: the 128-bit one (incl. L < 8 row lanes).  layout "csr":
    the same equal-length segments given as CSR offsets, bit-identical to the fixed layout."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(5)
    B, F = 37, 14
    fixed = (B, L, None, None)
    seg = fixed if layout == "fixed" else csr_seg([L] * B, dev)
    clouds = torch.randn(B, F, L, device=dev)
    T = torch.randn(B, 2, 2, device=dev)
    rows = ops.cloud_rows(clouds, T.reshape(B, 4), 16, add_eye=True)
    Te = T + torch.eye(2, device=dev)
    xy = torch.bmm(clouds[:, :2].transpose(1, 2), Te).transpose(1, 2)
    ref = torch.cat([xy, clouds[:, 2:]], 1).permute(0, 2, 1).reshape(B * L, F)
    close(rows[:, :F], ref, 1e-6)
    assert torch.all(rows[:, F:] == 0)
    Y = torch.randn(B * L, C, device=dev)
    sc, sh = torch.randn(C, device=dev), torch.randn(C, device=dev)
    pooled = torch.empty(B, C + 2, device=dev)
    am = ops.segmax_fwd(Y, C, seg, C, sc, sh, True, pooled, C + 2)
    a = torch.relu(Y * sc + sh).view(B, L, C)
    mx, idx = a.max(1)
    close(pooled[:, :C], mx, 1e-6)
    close(a.gather(1, am.long().unsqueeze(1)).squeeze(1), mx, 1e-6)  # argmax attains the max
    if layout == "csr":
        pooled_f = torch.empty(B, C + 2, device=dev)
        assert torch.equal(am, ops.segmax_fwd(Y, C, fixed, C, sc, sh, True, pooled_f, C + 2))
        assert torch.equal(pooled[:, :C], pooled_f[:, :C])
    # without the affine the arithmetic is exact: index output must be bit-exact, first maximiser
    Yq = torch.round(Y * 4) / 4  # many ties
    am = ops.segmax_fwd(Yq, C, seg, C, None, None, False, pooled, C + 2)
    a = Yq.view(B, L, C)
    mx, _ = a.max(1)
    assert torch.equal(pooled[:, :C], mx)
    first = (a == mx.unsqueeze(1)).float().argmax(1)
    assert torch.equal(am.long(), first)
    gp = torch.randn(B, C, device=dev)
    G = ops.segmax_bwd(gp, C, am, seg, C)
    ref = torch.zeros(B, L, C, device=dev).scatter_(1, am.long().unsqueeze(1), gp.unsqueeze(1))
    assert torch.equal(G.view(B, L, C), ref)
    if layout == "csr":
        assert torch.equal(G, ops.segmax_bwd(gp, C, am, fixed, C))
    dX = torch.randn(B * L, 16, device=dev)
    dT = ops.stn_apply_bwd(clouds, dX, 16)
    ref = torch.bmm(clouds[:, :2], dX.view(B, L, 16)[:, :, :2])
    close(dT.view(B, 2, 2), ref, 1e-5)


def check_pool_vs_torch(ops, Y, seg, C, dev):
    """segmax_fwd / segmax_bwd over the CSR segments `seg` of Y [P, C] against torch: the exact max (0 for
    an empty segment), the FIRST maximiser within the segment (-1 for an empty one), the scattered gradient."""
    B, _, offsets, row_seg = seg
    P = Y.shape[0]
    pooled = torch.empty(B, C, device=dev)
    am = ops.segmax_fwd(Y, C, seg, C, None, None, False, pooled, C)
    rs = row_seg.long()
    lens = offsets[1:] - offsets[:-1]
    mx = torch.full((B, C), -float("inf"), device=dev).scatter_reduce_(0, rs[:, None].expand(P, C), Y, "amax")
    mx[lens == 0] = 0
    assert torch.equal(pooled, mx)
    assert torch.equal(am[lens == 0], torch.full_like(am[lens == 0], -1))
    full = lens > 0
    assert bool((am[full] >= 0).all()) and bool((am[full] < lens[full, None]).all())
    rows = offsets[:-1, None] + am.long()
    assert torch.equal(Y.gather(0, rows[full]), mx[full])  # the argmax attains the max ...
    l_of_row = torch.arange(P, device=dev) - offsets[rs]
    at_max = Y == mx[rs]
    assert bool((l_of_row[:, None] >= am[rs])[at_max].all())  # ... and no earlier row of its segment does
    gp = torch.randn(B, C, device=dev)
    G = ops.segmax_bwd(gp, C, am, seg, C)
    ref = torch.zeros(P, C, device=dev).scatter_(0, rows[full], gp[full])
    assert torch.equal(G, ref)
    return am


@pytest.mark.parametrize("C", [70, 64])
def test_segmax_unequal_segments(dev, C):
    """CSR segments of unequal lengths, with empty and one-row segments, on an input with many ties."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(11)
    lens = torch.randint(0, 40, (41,))
    lens[[0, 7, 40]] = 0
    lens[[1, 2, 20]] = 1
    seg = csr_seg(lens, dev)
    Y = torch.round(torch.randn(int(lens.sum()), C, device=dev) * 4) / 4
    check_pool_vs_torch(ops, Y, seg, C, dev)


def check_segmax_bn_bwd(ops, Y, seg, C, dev):
    """The fused max-pool + BatchNorm/ReLU backward against its unfused composition (segmax_bwd ->
    act_bwd_reduce -> act_bwd_apply) over the same argmax."""
    M = Y.shape[0]
    eps = 1e-5
    mean, var = Y.mean(0), Y.var(0, unbiased=False)
    scale, shift = ops.bn_fold(mean, var, torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev), eps)
    pooled = torch.empty(seg[0], C, device=dev)
    am = ops.segmax_fwd(Y, C, seg, C, scale, shift, True, pooled, C)
    gp = torch.randn(seg[0], C + 3, device=dev)  # unaligned pooled-gradient rows, as PointNet's
    s1, s2, dY = ops.segmax_bn_bwd(gp, C + 3, am, Y, C, scale, shift, mean, var, eps, True, seg, C)
    G = ops.segmax_bwd(gp, C + 3, am, seg, C)
    s12 = ops.act_bwd_reduce(G, C, Y, C, scale, shift, mean, var, eps, True, M, C)
    close(s1, s12[:C], 1e-5)
    close(s2, s12[C:], 1e-5)
    dY_ref = ops.act_bwd_apply(G, C, Y, C, scale, shift, mean, var, eps, True, True, s12[:C], s12[C:], M, C)
    close(dY, dY_ref, 1e-5)


@pytest.mark.parametrize("layout", ["fixed", "csr"])
def test_segmax_bn_bwd(dev, layout):
    from superpoint_graph_b200 import ops
    torch.manual_seed(12)
    B, L, C = 300, 24, 132
    if layout == "fixed":
        seg = (B, L, None, None)
    else:
        lens = torch.randint(0, 2 * L, (B,))
        lens[[3, 150]] = 0
        lens[[4, 151]] = 1
        seg = csr_seg(lens, dev)
    M = B * L if layout == "fixed" else int(seg[3].numel())
    check_segmax_bn_bwd(ops, torch.randn(M, C, device=dev), seg, C, dev)


def test_segmax_more_than_65535_segments(dev):
    """Ragged pooling over more segments than one launch's grid.y holds, forward and backward."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(13)
    lens = torch.randint(0, 5, (70000,))
    seg = csr_seg(lens, dev)
    C = 64
    Y = torch.round(torch.randn(int(lens.sum()), C, device=dev) * 4) / 4
    check_pool_vs_torch(ops, Y, seg, C, dev)
    check_segmax_bn_bwd(ops, torch.randn(int(lens.sum()), C, device=dev), seg, C, dev)


def test_ce_loss_and_adam(dev):
    from superpoint_graph_b200 import ops
    torch.manual_seed(6)
    n, C = 1000, 13
    logits = (torch.randn(n, C, device=dev) * 3).requires_grad_(True)
    target = torch.randint(0, C, (n,), device=dev)
    target[::17] = -100
    cw = torch.rand(C, device=dev) + 0.5
    for weight in (None, cw):
        ref = torch.nn.functional.cross_entropy(logits, target, weight=weight)
        (gref,) = torch.autograd.grad(ref, logits)
        loss, dl = ops.ce_loss(logits.detach(), target, weight)
        close(loss[0], ref, 1e-5)
        close(dl, gref, 1e-4, 1e-9)
    p = torch.randn(10001, device=dev)
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([pr], lr=1e-2)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 4):
        g = torch.randn_like(p) * 3
        pr.grad = g.clamp(-1, 1)
        opt.step()
        ops.clamp_adam_(p, g, m, v, step, lr=1e-2, grad_clip=1.0)
        close(p, pr, 1e-5, 1e-6)


# ------------------------------------------------------------------------------- networks
def _pcfg(cfg):
    return dict(n_conv=len(cfg["nf_conv"]), n_fc=len(cfg["nf_fc"]), n_conv_stn=len(cfg["nf_conv_stn"]),
                n_fc_stn=len(cfg["nf_fc_stn"]), nfeat_stn=cfg["nfeat_stn"])


def test_pointnet_small_golden(golden_dir, dev):
    from superpoint_graph_b200.spg_pointnet import PointNet
    g = load(golden_dir, "pointnet_small.npz")
    cfg = json.loads(str(g["cfg"]))
    net = PointNet(cfg["nf_conv"], cfg["nf_fc"], cfg["nf_conv_stn"], cfg["nf_fc_stn"], cfg["nfeat"],
                   cfg["nfeat_stn"], prelast_do=0)
    net.load_state_dict(sub(g, "sd0."))
    net.to(dev).train()
    x, xg = t(g["x"], dev), t(g["xg"], dev)
    out = net(x, xg)
    close(out, g["out_train"])
    out.backward(t(g["g"], dev))
    close_grads({k: p.grad for k, p in net.named_parameters()}, sub(g, "grad."), 3e-4)
    sd1 = sub(g, "sd1.")
    now = net.state_dict()
    for k, v in sd1.items():
        if k.endswith("num_batches_tracked"):
            assert int(now[k]) == int(v)
        elif not nets_ref.is_param(k):
            close(now[k], v, 1e-5, 1e-7)
    net.eval()
    with torch.no_grad():
        close(net(x, xg), g["out_eval"])
        close(net.stn(x[:, :cfg["nfeat_stn"]].contiguous()), g["T_eval"])


def test_pointnet_ragged_csr(golden_dir, dev):
    """PointNet.forward_ragged (CSR offset array, no resample-to-ptn_npts): (1) with equal segment lengths
    it reproduces the reference's golden outputs and gradients; (2) with unequal lengths (1..300 points)
    it matches the oracle's ragged restatement, forward and backward (incl. the gradient w.r.t. the
    global input), S3DIS widths."""
    from superpoint_graph_b200.spg_pointnet import PointNet
    g = load(golden_dir, "pointnet_small.npz")
    cfg = json.loads(str(g["cfg"]))
    net = PointNet(cfg["nf_conv"], cfg["nf_fc"], cfg["nf_conv_stn"], cfg["nf_fc_stn"], cfg["nfeat"],
                   cfg["nfeat_stn"], prelast_do=0)
    net.load_state_dict(sub(g, "sd0."))
    net.to(dev).train()
    x, xg = t(g["x"]), t(g["xg"], dev)
    B, F, L = x.shape
    pts = x.permute(0, 2, 1).reshape(B * L, F).contiguous().to(dev)
    offs = (torch.arange(B + 1) * L).to(dev)
    out = net.forward_ragged(pts, offs, xg)
    close(out, g["out_train"])
    out.backward(t(g["g"], dev))
    close_grads({k: p.grad for k, p in net.named_parameters()}, sub(g, "grad."), 3e-4)
    net.eval()
    with torch.no_grad():
        close(net.forward_ragged(pts, offs, xg), g["out_eval"])
    # (2) unequal lengths, S3DIS widths
    torch.manual_seed(6)
    net = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=0)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
    sd = {k: v.clone().requires_grad_(nets_ref.is_param(k)) for k, v in net.state_dict().items()}
    rng = np.random.default_rng(6)
    lens = rng.integers(1, 301, size=97)
    lens[[3, 50]] = 1
    offsets = np.concatenate([[0], np.cumsum(lens)])
    P = int(offsets[-1])
    points = torch.randn(P, 14) * 0.4
    glob = torch.rand(97) * 3
    glob_ref, glob_dev = glob.clone().requires_grad_(True), glob.to(dev).requires_grad_(True)
    pcfg = dict(n_conv=5, n_fc=3, n_conv_stn=3, n_fc_stn=2, nfeat_stn=14)
    ref = nets_ref.pointnet_forward_ragged(points, offsets, glob_ref, sd, pcfg, True)
    gy = torch.randn(97, 32)
    ref.backward(gy)
    net.to(dev).train()
    out = net.forward_ragged(points.to(dev), torch.from_numpy(offsets).to(dev), glob_dev)
    close(out, ref)
    out.backward(gy.to(dev))
    assert glob_dev.grad is not None, "missing gradient for input_global"
    close(glob_dev.grad, glob_ref.grad, 1e-3)
    # (float32 oracle, BatchNorm over 1.5e4 points, max-pool ties: see tests/test_gpu_shapes.py's docstring)
    close_grads({k: p.grad for k, p in net.named_parameters()},
                {k: v.grad for k, v in sd.items() if v.requires_grad}, 3e-2)


def test_pointnet_s3dis_widths_vs_oracle(dev):
    """The S3DIS architecture (main.py:104-107) at L=128, training-mode forward+backward."""
    from superpoint_graph_b200.spg_pointnet import PointNet
    net = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=0)
    torch.manual_seed(8)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
        net.stn.proj.bias.normal_(0, 0.05)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    for k, v in sd.items():
        if nets_ref.is_param(k):
            v.requires_grad_(True)
    B = 48
    x, xg = torch.randn(B, 14, 128) * 0.4, torch.rand(B) * 3
    gout = torch.randn(B, 32)
    pcfg = dict(n_conv=5, n_fc=3, n_conv_stn=3, n_fc_stn=2, nfeat_stn=14)
    ref = nets_ref.pointnet_forward(x, xg, sd, pcfg, True)
    ref.backward(gout)
    net.to(dev).train()
    out = net(x.to(dev), xg.to(dev))
    close(out, ref)
    out.backward(gout.to(dev))
    close_grads({k: p.grad for k, p in net.named_parameters()},
                {k: v.grad for k, v in sd.items() if v.requires_grad}, 5e-4)


MCFG = {
    "vv": dict(fnet_widths=[13, 32, 128, 64, 32], bnidx=2, nrepeats=3, layernorm=True, ingate=True, cat_all=False),
    "cat": dict(fnet_widths=[13, 32, 128, 64, 32], bnidx=2, nrepeats=2, layernorm=True, ingate=True, cat_all=True),
    "mat": dict(fnet_widths=[13, 32, 128, 64, 1024], bnidx=2, nrepeats=2, layernorm=True, ingate=True, cat_all=True),
}


@pytest.mark.parametrize("tag,fused", [("vv", True), ("vv", False), ("cat", True), ("cat", False),
                                       ("mat", False)])
def test_graphnet_golden(golden_dir, dev, tag, fused, monkeypatch):
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    monkeypatch.setattr(ops, "USE_FUSED_RNN", [fused])
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    g = load(golden_dir, "graphnet_%s.npz" % tag)
    net = GraphNetwork(str(g["config"]), 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0, cuda=True)
    net.load_state_dict(sub(g, "sd0."))
    net.to(dev).train()
    gi = GraphConvInfo.from_arrays(g["idxn"], g["degs"], g["edgefeats"])
    net.set_info([gi], True)
    emb = t(g["emb"], dev).requires_grad_(True)
    out = net(emb)
    close(out, g["out_train"])
    ncls = out.shape[1]
    labels = t(g["labels"])
    if ncls < 13:
        labels = labels.clamp(max=ncls - 1)
    cw = t(g["cw"])[:ncls]
    loss = torch.nn.functional.cross_entropy(out, labels.to(dev), weight=cw.to(dev))
    loss.backward()
    if "loss" in g:
        close(loss, g["loss"])
        close(emb.grad, g["gemb"], 3e-4, 1e-7)
        close_grads({k: p.grad for k, p in net.named_parameters()}, sub(g, "grad."), 3e-4)
    else:  # matrix filters: the reference's backward no longer runs; the pinned oracle decides
        sd = sub(g, "sd0.")
        for k, v in sd.items():
            if nets_ref.is_param(k):
                v.requires_grad_(True)
        e2 = t(g["emb"]).requires_grad_(True)
        ro = nets_ref.graphnet_forward(e2, t(g["edgefeats"]), t(g["idxn"]), t(g["degs"]), sd, MCFG[tag], True)
        torch.nn.functional.cross_entropy(ro, labels, weight=cw).backward()
        close(emb.grad, e2.grad, 3e-4, 1e-7)
        close_grads({k: p.grad for k, p in net.named_parameters()},
                    {k: v.grad for k, v in sd.items() if v.requires_grad}, 3e-4)
    net.eval()
    with torch.no_grad():
        close(net(emb.detach()), g["out_eval"])


def test_two_training_steps_golden(golden_dir, dev):
    """Two complete reference training steps (loss, logits, updated parameters)."""
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    g = load(golden_dir, "train_steps.npz")
    args = make_args(model_config="gru_3_1_1_1_0,f_13", ptn_widths=[[16, 16, 32], [32, 16, 8]],
                     ptn_widths_stn=[[8, 16], [16, 8]], ptn_nfeat_stn=6, node_feats=6,
                     fnet_widths=[16, 32, 16])
    model = create_model(args)
    model.ecc.load_state_dict(sub(g, "ecc0."))
    model.ptn.load_state_dict(sub(g, "ptn0."))
    model.to(dev)
    tr = Trainer(model, args)
    batch = dict(clouds=t(g["clouds"]), clouds_global=t(g["cglob"]), clouds_flag=t(g["flag"]),
                 edgefeats=t(g["edgefeats"]), idxn=t(g["idxn"]), degs=t(g["degs"]), labels=t(g["labels"]))
    hb = HostBatch(batch)
    db = hb.to_device(dev)
    l0, o0 = tr.train_step(db)
    l1, o1 = tr.train_step(db)
    close(o0, g["out0"])
    close(torch.stack([l0[0], l1[0]]), g["losses"], 1e-4)
    close(o1, g["out1"], 3e-3)
    sd = model.ecc.state_dict()
    for k, v in sub(g, "ecc2.").items():
        if nets_ref.is_param(k):
            close(sd[k], v, 5e-3, 2.1e-2 if k == "0._fnet.4.bias" else 1e-5)


def test_cpu_tensors_are_rejected(dev):
    from superpoint_graph_b200 import ops
    with pytest.raises(RuntimeError):
        ops.gemm(torch.randn(4, 4), 4, True, torch.randn(4, 4), 4, True, 4, 4, 4)


def test_cuda_graph_replay_matches_eager(dev):
    """Trainer.capture()/replay(): three replayed steps == three eager steps (same kernels, same
    order; the Adam step count lives in device memory so nothing is baked into the graph)."""
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config="gru_3_1_1_1_0,f_13")
    batch = make_batch(n_nodes=200, seed=11)
    results = []
    for mode in ("eager", "graph"):
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        losses = []
        if mode == "eager":
            for _ in range(3):
                loss, logits = tr.train_step(db)
                losses.append(float(loss[0]))
        else:
            # capture() is free of side effects (warm-up runs on a snapshot): 3 replays == 3 eager steps
            key = tr.capture(db, warmup=1)
            losses = []
            for _ in range(3):
                loss, logits = tr.replay(key)
                losses.append(float(loss[0]))
        torch.cuda.synchronize()
        results.append((losses, tr.flat.clone(), logits.clone()))
    (l_e, p_e, o_e), (l_g, p_g, o_g) = results
    assert int(torch.isfinite(p_g).all())
    close(torch.tensor(l_g), torch.tensor(l_e), 1e-5)
    close(o_g, o_e, 1e-4)
    close(p_g, p_e, 1e-4, 2.1e-2 * 4)  # noise-driven (pre-BN bias) parameters random-walk by +-lr


def test_eval_chunking_matches_unchunked(dev, monkeypatch):
    """Eval-mode PointNet slices huge inputs (Semantic3D-scale inference, configs[2]); BatchNorm in
    eval mode is per-sample, so slicing must not change anything."""
    from superpoint_graph_b200 import spg_pointnet
    net = spg_pointnet.PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 11, 11, prelast_do=0)
    torch.manual_seed(3)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    B = 301
    x, xg = torch.randn(B, 11, 128) * 0.4, torch.rand(B) * 3
    pcfg = dict(n_conv=5, n_fc=3, n_conv_stn=3, n_fc_stn=2, nfeat_stn=11)
    ref = nets_ref.pointnet_forward(x, xg, sd, pcfg, False)
    net.to(dev).eval()
    with torch.no_grad():
        whole = net(x.to(dev), xg.to(dev))
        monkeypatch.setattr(spg_pointnet, "_EVAL_CHUNK", 64)
        sliced = net(x.to(dev), xg.to(dev))
    close(whole, ref)
    close(sliced, ref)
    assert torch.equal(whole, sliced)


@pytest.mark.parametrize("F,B", [(14, 301), (11, 64), (9, 1)])
def test_fused_eval_trunk_vs_oracle(dev, monkeypatch, F, B):
    """Eval-mode PointNet with both point-wise chains fused into one kernel each (input tile -> STN chain /
    xy transform + 5 layers -> max-pool, BatchNorm folded, activations never in HBM) against the oracle
    and against the layer-by-layer path; the fused kernel must actually be the one that ran."""
    from superpoint_graph_b200 import ops, spg_pointnet
    net = spg_pointnet.PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], F, F, prelast_do=0)
    torch.manual_seed(3 + F)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    x, xg = torch.randn(B, F, 128) * 0.4, torch.rand(B) * 3
    pcfg = dict(n_conv=5, n_fc=3, n_conv_stn=3, n_fc_stn=2, nfeat_stn=F)
    ref = nets_ref.pointnet_forward(x, xg, sd, pcfg, False)
    net.to(dev).eval()
    ops.prof_reset()
    with torch.no_grad():
        fused = net(x.to(dev), xg.to(dev))
        assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 2  # STN chain + main chain
        monkeypatch.setattr(ops, "USE_FUSED_EVAL", [False])
        layered = net(x.to(dev), xg.to(dev))
    close(fused, ref)
    close(layered, ref)
    close(fused, layered, 2e-5)


def test_local_cloud_embedder_tiny_clouds(dev):
    """Learned-partition embedder (configs[3] first half, pointnet.py:182-207): external STN on 2
    features, 20-point clouds, global features + flattened T, L2-normalised 4-D output."""
    from types import SimpleNamespace
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder, PointNet, STNkD
    torch.manual_seed(4)
    model = torch.nn.Module()
    model.stn = STNkD(2, [16, 64], [32, 16])
    model.ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=0, nfeat_global=11 + 4)
    with torch.no_grad():
        model.stn.proj.weight.normal_(0, 0.1)
    sd_stn = {k: v.clone() for k, v in model.stn.state_dict().items()}
    sd_ptn = {k: v.clone() for k, v in model.ptn.state_dict().items()}
    B, L = 700, 20
    clouds, glob = torch.randn(B, 6, L) * 0.5, torch.randn(B, 11)
    T = nets_ref.stn_forward(clouds[:, :2], sd_stn, "", 2, 2, True)
    xy = torch.bmm(clouds[:, :2].transpose(1, 2), T).transpose(1, 2)
    c2 = torch.cat([xy, clouds[:, 2:]], 1)
    g2 = torch.cat([glob, T.view(-1, 4)], 1)
    pcfg = dict(n_conv=2, n_fc=4, n_conv_stn=0, n_fc_stn=0, nfeat_stn=0)
    ref = torch.nn.functional.normalize(nets_ref.pointnet_forward(c2, g2, sd_ptn, pcfg, True))
    model.to(dev).train()
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    out = emb.run_batch(model, clouds.to(dev), glob.to(dev))
    close(out, ref, 2e-4)
    # backward through the whole embedder (STN -> xy transform -> global features -> PointNet -> L2
    # normalisation) against autograd of the oracle on the same state (supervized_partition.py:411-434 trains it)
    sd_s = {k: v.clone().requires_grad_(nets_ref.is_param(k)) for k, v in sd_stn.items()}
    sd_p = {k: v.clone().requires_grad_(nets_ref.is_param(k)) for k, v in sd_ptn.items()}
    T = nets_ref.stn_forward(clouds[:, :2], sd_s, "", 2, 2, True)
    xy = torch.bmm(clouds[:, :2].transpose(1, 2), T).transpose(1, 2)
    ref2 = torch.nn.functional.normalize(nets_ref.pointnet_forward(
        torch.cat([xy, clouds[:, 2:]], 1), torch.cat([glob, T.view(-1, 4)], 1), sd_p, pcfg, True))
    gy = torch.randn(B, 4)
    ref2.backward(gy)
    model.zero_grad()
    out.backward(gy.to(dev))
    close_grads({"stn." + k: p.grad for k, p in model.stn.named_parameters()},
                {"stn." + k: v.grad for k, v in sd_s.items() if v.requires_grad}, 2e-3)
    close_grads({"ptn." + k: p.grad for k, p in model.ptn.named_parameters()},
                {"ptn." + k: v.grad for k, v in sd_p.items() if v.requires_grad}, 2e-3)


def test_cloud_embedder_mem_monger_same_gradients(dev):
    """ptn_mem_monger=1 (no-grad forward + full recomputation in bw_hook, pointnet.py:160-180) must
    give the gradients of the plain path; only the running statistics see two updates per step."""
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    batch = make_batch(n_nodes=150, seed=21)
    grads = []
    for monger in (0, 1):
        args = make_args(model_config="gru_2_1_1_1_0,f_13", ptn_mem_monger=monger)
        torch.manual_seed(9)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        # CloudEmbedder API as main.py:202-208 drives it
        model.train()
        model.ecc.gconvs[0].set_info(db.gi)
        emb = tr.embedder.run(model, None, batch["clouds_flag"], batch["clouds"], batch["clouds_global"])
        out = model.ecc(emb)
        loss = torch.nn.functional.cross_entropy(out, db.labels)
        loss.backward()
        tr.embedder.bw_hook()
        grads.append({k: p.grad.clone() for k, p in model.named_parameters()})
    close_grads(grads[1], grads[0], 1e-5)


def test_graph_conv_module_matrix_filters(dev):
    """ecc.GraphConvModule (GraphConvModule.py:156-193): filter net -> [E,in,out] -> function."""
    from superpoint_graph_b200.spg_ecc import GraphConvInfo, GraphConvModule
    from superpoint_graph_b200.spg_graphnet import create_fnet
    rng = np.random.default_rng(2)
    N, cin, cout = 90, 8, 12
    degs_np = rng.integers(0, 6, size=N)
    E = int(degs_np.sum())
    idxn = rng.integers(0, N, size=E)
    ef = rng.standard_normal((E, 5)).astype(np.float32)
    torch.manual_seed(2)
    fnet = create_fnet([5, 16, cin * cout], True, True)
    sd = {k: v.clone().requires_grad_(True) for k, v in fnet.state_dict().items()}
    x = torch.randn(N, cin)
    w_ref = nets_ref.fnet_forward(t(ef), sd, "", [5, 16, cin * cout], -1, True).view(E, cin, cout)
    ref = ecc_ref.graph_conv_forward(x, w_ref, t(idxn), None, t(degs_np))
    gout = torch.randn(N, cout)
    ref.backward(gout)
    mod = GraphConvModule(cin, cout, fnet, GraphConvInfo.from_arrays(idxn, degs_np, ef)).to(dev).train()
    mod._gci.cuda()
    xg = x.to(dev).requires_grad_(True)
    out = mod(xg)
    close(out, ref)
    out.backward(gout.to(dev))
    close_grads({k: p.grad for k, p in fnet.named_parameters()}, {k: v.grad for k, v in sd.items()}, 3e-4)


@pytest.mark.parametrize("cat_all", [False, True])
@pytest.mark.parametrize("n_nodes", [37, 1024, 5000])
@pytest.mark.parametrize("cell", ["GRUCellEx", "LSTMCellEx"])
def test_fused_recurrence_is_bit_identical_to_per_step_kernels(dev, monkeypatch, cell, n_nodes, cat_all):
    """One-kernel R x {ECC, cell} loop (grid barrier between steps) vs. the 2R / 3R separate
    launches, for both cells: the ECC rows (ecc_rows.cuh) and the cell rows are the same device
    functions in both paths, so the sums run in the same order -> identical bits, forward and
    backward."""
    from superpoint_graph_b200 import ops, spg_modules, synthetic
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_graphnet import create_fnet
    torch.manual_seed(3)
    b = synthetic.make_batch(n_nodes, k=8, seed=11, npts=8, minpts=4)
    gi = GraphConvInfo.from_arrays(b["idxn"].numpy(), b["degs"].numpy(), b["edgefeats"].numpy())
    gi.cuda()
    fnet = create_fnet([13, 32, 128, 64, 32], True, 0, 2)
    cell_mod = getattr(spg_modules, cell)(32, 32, bias=True, layernorm=True, ingate=True)
    mod = spg_modules.RNNGraphConvModule(cell_mod, fnet, 32, vv=True, gc_info=gi, nrepeats=10,
                                         cat_all=cat_all, use_pyg=False, cuda=True).to(dev).train()
    x0 = torch.randn(n_nodes, 32, device=dev)
    results = []
    for fused in (True, False):
        monkeypatch.setattr(ops, "USE_FUSED_RNN", [fused])
        assert ops.rnn_vv_supported(torch.empty(1, 32, device=dev), gi.graph(), n_nodes, 32) == fused
        mod.zero_grad()
        x = x0.clone().requires_grad_(True)
        y = mod(x)
        (y * torch.linspace(-1, 1, y.numel(), device=dev).view_as(y)).sum().backward()
        results.append([y.detach(), x.grad] + [p.grad.clone() for p in mod.parameters()])
    for a, c in zip(*results):
        assert torch.equal(a, c)


@pytest.mark.parametrize("graph", [False, True])
def test_side_stream_gives_identical_steps(dev, monkeypatch, graph):
    """Trainer runs the recurrent block's parameter gradients on a second stream underneath the
    PointNet backward; the kernels and their order per stream are unchanged, so three steps must be
    bit-identical to the single-stream run (eager and CUDA-graph replay)."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config="gru_4_1_1_1_1,f_13")
    batch = make_batch(n_nodes=300, seed=4)
    results = []
    for side in (True, False):
        monkeypatch.setattr(ops, "USE_SIDE_STREAM", [side])
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        assert (tr._side is not None) == side
        tr.side_in_eager = True  # default: only captured steps use the second stream
        db = HostBatch(batch).to_device(dev)
        losses = []
        if graph:
            key = tr.capture(db, warmup=2)
            for _ in range(3):
                loss, logits = tr.replay(key)
                losses.append(float(loss[0]))
        else:
            for _ in range(5):
                loss, logits = tr.train_step(db)
                losses.append(float(loss[0]))
        torch.cuda.synchronize()
        results.append((losses, tr.flat.clone(), logits.clone(), tr.flat_grad.clone()))
    (l_a, p_a, o_a, g_a), (l_b, p_b, o_b, g_b) = results
    assert l_a == l_b
    assert torch.equal(g_a, g_b) and torch.equal(p_a, p_b) and torch.equal(o_a, o_b)


# ------------------------------------------------------------------ device-side graph build (f1)
@pytest.mark.parametrize("n,deg,seed", [(1, 0, 0), (7, 3, 1), (1024, 9, 2), (20000, 12, 3), (200000, 9, 4)])
def test_graph_build_device_is_bit_identical_to_host_builder(dev, n, deg, seed):
    """spg_graph_build (scan + stable radix sort + 3 kernels) against the numpy builder the CPU tests pin
    (tests/test_host_logic.py): every view bit-exact, including the order of equal sources in src_perm."""
    from superpoint_graph_b200 import ops
    rng = np.random.RandomState(seed)
    degs = rng.randint(0, 2 * deg + 1, size=n).astype(np.int64) if deg else np.zeros(n, dtype=np.int64)
    if n > 3:
        degs[rng.randint(0, n, size=max(1, n // 50))] = 0   # isolated targets
        degs[rng.randint(0, n)] = 40 * max(deg, 1)           # one hub
    E = int(degs.sum())
    idxn = rng.randint(0, n, size=E).astype(np.int64)
    if E > 10:
        idxn[: E // 4] = idxn[0]                              # many equal keys: stability matters
    want = ops.build_csr_host(idxn, degs, n)
    g = ops.EccGraph.from_device(t(idxn, dev), t(degs, dev), n_in=n, check=True)
    got = g.to(dev)
    for k in ops.EccGraph.GRAPH_FIELDS:
        assert got[k].dtype == torch.int32
        assert np.array_equal(got[k].cpu().numpy(), want[k]), k
    assert int(got["status"].item()) == 0


def test_graph_build_device_rejects_bad_arrays(dev):
    from superpoint_graph_b200 import ops
    degs = torch.tensor([2, 1, 0], dtype=torch.int64, device=dev)
    with pytest.raises(ValueError, match="status 1"):
        ops.EccGraph.from_device(torch.tensor([0, 3, 1], dtype=torch.int64, device=dev), degs, n_in=3)
    with pytest.raises(ValueError, match="status 4"):
        ops.EccGraph.from_device(torch.tensor([0, 1], dtype=torch.int64, device=dev), degs, n_in=3)


def test_graphconvinfo_cuda_builds_on_device_and_matches_golden(golden_dir, dev):
    """GraphConvInfo.cuda() (the call learning/main.py makes through set_info) now derives the CSR views on
    the device; the convolution through it must equal the one through the host-built graph."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_ecc import GraphConvFunction, GraphConvInfo
    rng = np.random.RandomState(5)
    n = 500
    degs = rng.randint(0, 12, size=n).astype(np.int64)
    idxn = rng.randint(0, n, size=int(degs.sum())).astype(np.int64)
    ef = rng.randn(idxn.shape[0], 13).astype(np.float32)
    gi = GraphConvInfo.from_arrays(idxn, degs, ef)
    gi.cuda()
    assert gi.graph().host is None  # built on the device
    x = torch.randn(n, 32, device=dev)
    w = torch.randn(idxn.shape[0], 32, device=dev)
    a = GraphConvFunction.apply(x, w, 32, 32, gi.graph(), None, None, None)
    host = ops.EccGraph(t(idxn), None, t(degs), n_in=n)
    b = GraphConvFunction.apply(x, w, 32, 32, host, None, None, None)
    assert torch.equal(a, b)
    # raw reference-style argument list with CUDA tensors: cached device build
    bufs = gi.get_buffers()
    c = GraphConvFunction.apply(x, w, 32, 32, bufs[0], bufs[1], bufs[2], bufs[3])
    assert torch.equal(a, c)
