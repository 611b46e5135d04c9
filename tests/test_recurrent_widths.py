"""The recurrent ECC block (`gru_*` / `lstm_*` tokens: R x {ECC, cell}, ref: learning/modules.py:128-316) at
every hidden width H and cell option the kernels accept, kernel by kernel against float64.

H is the PointNet's last FC width (or that of an `f_<n>` token before the recurrent one), so it is not always 32.
At H != 32 the recurrence runs the per-step path: the generic ECC kernels, the cell kernels at the
instantiation their tiling selection picks, and the SIMT GEMMs of the cell's weight gradients.

CPU: a Python copy of the cell kernels' tiling selection (rnn_cell.cu: cell_weight_floats,
cell_scratch_floats, cell_smem_bytes, cell_rows_per_warp) and the table CELL_CASES of (cell, H, rows)
with one row set for every instantiation cell_bwd_kernel<Cell, NU, RW> that selection can make.
GPU:
  * the selection against the library at the widths where it stops accepting (forward and backward);
  * GRUCellEx / LSTMCellEx at every row of CELL_CASES and at all 8 {LAYERNORM, INGATE, BIAS}
    combinations, forward and backward, against float64 autograd through the oracle cells;
  * the generic ECC kernels (ecc.cu: ecc_generic_*) in fp32 against oracle/ecc_ref;
  * RNNGraphConvModule at H = 16 and 64, and one training step at H = 64, against the oracle.

Row counts: the cell kernels run at most 4 * 132 blocks of 8 warps, grid-strided.  With 1 row per warp
(RW = 1) one pass covers 4224 rows, so 4225 rows reach a second pass; 1 and 7 leave most warps idle.
With 4 rows per warp (RW = 4, from 8448 rows on) 8449 and 8451 leave the last warp 1 and 3 live rows
and 16897 is one row into the second pass.  Widths that are not a multiple of 32 (20, 48, 57, 72, 85, ...)
leave the last column group of each warp partly idle.
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import ecc_ref, lstm_ref, nets_ref
from test_gpu_parity import close, close_grads
from test_lstm import _cell_oracle as _lstm_oracle

# --------------------------------------------------------------------------------------------------
# Python copy of the cell kernels' tiling selection (rnn_cell.cu)
MAX_SMEM, CELL_WARPS, NUM_SMS = 227 * 1024, 8, 132
RW4_MIN_ROWS = NUM_SMS * CELL_WARPS * 4 * 2  # 8448: enough rows for 4 per warp to fill the GPU twice
GATES = {"gru": 3, "lstm": 4}
DY_SCRATCH = {"gru": 0, "lstm": 1}
FEWER_ROWS_IF_FULL = {"gru": False, "lstm": True}  # Cell::kFewerRowsIfFull


def cell_weight_floats(cell, H):
    return H * (H + 1) + 2 * H * (GATES[cell] * H + 1)


def cell_scratch_floats(cell, H, rw):
    return rw * (3 * H + (2 + DY_SCRATCH[cell]) * GATES[cell] * H)


def cell_smem_bytes(cell, H, rw):
    return 4 * (cell_weight_floats(cell, H) + CELL_WARPS * cell_scratch_floats(cell, H, rw))


def cell_rows_per_warp(cell, n, H):
    rw = 4 if n >= RW4_MIN_ROWS else 1
    if rw == 4 and FEWER_ROWS_IF_FULL[cell] and cell_smem_bytes(cell, H, 4) > MAX_SMEM:
        rw = 1
    return rw if cell_smem_bytes(cell, H, rw) <= MAX_SMEM else 0


def selection(cell, n, H):
    """(NU, RW) of the cell_bwd_kernel that runs (cell, n rows, width H); None: "not supported"."""
    if H > 128:
        return None
    rw = cell_rows_per_warp(cell, n, H)
    if rw == 0:
        return None
    return (1 if H <= 32 else 2 if H <= 64 else 4), rw


# (cell, H, rows) -> (NU, RW).  Every instantiation at the row counts of the module docstring; the
# H = 32 rows at 1, 3, 33 and 1027 (and 20000 for the LSTM, and H = 64 for the LSTM) were the cases of the
# earlier per-cell tests.  At >= 8448 rows the LSTM falls back to 1 row per warp from H = 58 on.
CELL_CASES = {
    # GRU
    ("gru", 32, 1): (1, 1), ("gru", 32, 3): (1, 1), ("gru", 32, 33): (1, 1), ("gru", 32, 1027): (1, 1),
    ("gru", 20, 7): (1, 1), ("gru", 20, 4225): (1, 1),
    ("gru", 32, 8448): (1, 4), ("gru", 20, 8449): (1, 4), ("gru", 32, 8451): (1, 4), ("gru", 32, 16897): (1, 4),
    ("gru", 48, 1): (2, 1), ("gru", 57, 7): (2, 1), ("gru", 64, 4225): (2, 1),
    ("gru", 48, 8448): (2, 4), ("gru", 64, 8449): (2, 4), ("gru", 57, 8451): (2, 4), ("gru", 40, 16897): (2, 4),
    ("gru", 85, 1): (4, 1), ("gru", 72, 7): (4, 1), ("gru", 85, 4225): (4, 1), ("gru", 73, 8447): (4, 1),
    ("gru", 72, 8448): (4, 4), ("gru", 65, 8449): (4, 4), ("gru", 72, 8451): (4, 4), ("gru", 70, 16897): (4, 4),
    # LSTM
    ("lstm", 32, 1): (1, 1), ("lstm", 32, 3): (1, 1), ("lstm", 32, 33): (1, 1), ("lstm", 32, 1027): (1, 1),
    ("lstm", 20, 7): (1, 1), ("lstm", 32, 4225): (1, 1),
    ("lstm", 32, 8448): (1, 4), ("lstm", 20, 8449): (1, 4), ("lstm", 32, 8451): (1, 4),
    ("lstm", 32, 16897): (1, 4), ("lstm", 32, 20000): (1, 4),
    ("lstm", 64, 1): (2, 1), ("lstm", 64, 3): (2, 1), ("lstm", 64, 33): (2, 1), ("lstm", 64, 1027): (2, 1),
    ("lstm", 48, 7): (2, 1), ("lstm", 57, 4225): (2, 1),
    ("lstm", 58, 8448): (2, 1), ("lstm", 60, 8451): (2, 1), ("lstm", 64, 20000): (2, 1),
    ("lstm", 48, 8448): (2, 4), ("lstm", 57, 8449): (2, 4), ("lstm", 40, 8451): (2, 4), ("lstm", 57, 16897): (2, 4),
    ("lstm", 73, 1): (4, 1), ("lstm", 72, 7): (4, 1), ("lstm", 73, 4225): (4, 1), ("lstm", 73, 8449): (4, 1),
    ("lstm", 65, 16897): (4, 1),
}

ALL_FLAGS = list(itertools.product((True, False), repeat=3))
FLAG_H = 48                  # NU = 2 for both cells
FLAG_ROWS = (4225, 8451)     # RW = 1 and RW = 4 at that width


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("key", sorted(CELL_CASES), ids=lambda k: "%s-H%d-n%d" % k)
def test_cell_case_table_matches_selection(key):
    cell, H, n = key
    assert selection(cell, n, H) == CELL_CASES[key]


def test_cell_case_table_reaches_every_instantiation():
    """Between them the rows reach every (cell, NU, RW) the selection makes for H in 1..128, on both sides
    of the row-count threshold, and every row-count stress point of the module docstring."""
    reachable = {(cell, ) + s for cell in GATES for H in range(1, 129)
                 for n in (1, RW4_MIN_ROWS - 1, RW4_MIN_ROWS) for s in [selection(cell, n, H)] if s}
    covered = {(cell, ) + s for (cell, H, n), s in CELL_CASES.items()}
    assert covered == reachable
    assert len(reachable) == 11
    for cell, nu, rw in reachable:
        rows = {n for (c, H, n), s in CELL_CASES.items() if c == cell and s == (nu, rw)}
        if rw == 1:
            assert {1, 7, 4225} <= rows, (cell, nu, rw)
        elif rw == 4:
            assert {8448, 8449, 8451, 16897} <= rows, (cell, nu, rw)
    # the LSTM's fallback to 1 row per warp at >= 8448 rows, and widths off the 32-lane column groups
    assert any(c == "lstm" and n >= RW4_MIN_ROWS and s[1] == 1 for (c, H, n), s in CELL_CASES.items())
    assert {H % 32 for (c, H, n) in CELL_CASES} - {0}
    for fl in (FLAG_ROWS[0], FLAG_ROWS[1]):
        assert selection("gru", fl, FLAG_H)[0] == selection("lstm", fl, FLAG_H)[0] == 2
    assert [selection(c, n, FLAG_H)[1] for c in GATES for n in FLAG_ROWS] == [1, 4, 1, 4]


def test_selection_boundaries():
    """The widths where the cells stop being served (the GPU test pins these to the library)."""
    assert RW4_MIN_ROWS == 8448
    assert selection("gru", 100, 85) == (4, 1) and selection("gru", 100, 86) is None
    assert selection("gru", 8448, 72) == (4, 4) and selection("gru", 8448, 73) is None
    assert selection("gru", 8447, 73) == (4, 1)
    for n in (100, 8448):
        assert selection("lstm", n, 73) == (4, 1) and selection("lstm", n, 74) is None
    assert selection("lstm", 8448, 57) == (2, 4) and selection("lstm", 8448, 58) == (2, 1)
    assert all(selection(c, n, 129) is None for c in GATES for n in (1, 8448))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _cell_weights(G, H, dev):
    return [torch.randn(G * H, H, device=dev) * H ** -0.5, torch.randn(G * H, H, device=dev) * H ** -0.5,
            torch.randn(G * H, device=dev) * 0.3, torch.randn(G * H, device=dev) * 0.3,
            torch.randn(H, H, device=dev) * 2 * H ** -0.5, torch.randn(H, device=dev) * 0.3]


# (cell, rows, H, accepted): the last accepted and the first rejected width of each selection branch
BOUNDARIES = [("gru", 100, 85, True), ("gru", 100, 86, False), ("gru", 8448, 72, True), ("gru", 8448, 73, False),
              ("gru", 8447, 73, True), ("lstm", 100, 73, True), ("lstm", 100, 74, False),
              ("lstm", 8448, 73, True), ("lstm", 8448, 74, False),
              # inside the branches: a GRU width served with 1 row per warp only, the LSTM's fallback
              ("gru", 100, 80, True), ("gru", 9000, 80, False), ("lstm", 9000, 73, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("cell,n,H,accepted", BOUNDARIES)
def test_selection_boundaries_match_library(dev, cell, n, H, accepted):
    """ops.gru_fwd / lstm_fwd and the backward (cell_bwd, a separate entry with its own check) accept
    exactly the widths the Python selection accepts."""
    from superpoint_graph_b200 import ops
    assert (selection(cell, n, H) is not None) == accepted
    torch.manual_seed(H + n)
    flags = ops.GRU_LAYERNORM | ops.GRU_INGATE | ops.GRU_BIAS
    G = GATES[cell]
    w = _cell_weights(G, H, dev)
    x, h, c, gy = (torch.randn(n, H, device=dev) for _ in range(4))
    bufs = [torch.empty(n, G * H, device=dev), torch.empty(n, G * H, device=dev),
            torch.empty(n, H, device=dev), torch.empty(n, H, device=dev)]
    if cell == "gru":
        fwd = lambda: ops.gru_fwd(x, h, *w, flags)
        bwd = lambda: ops.gru_bwd(x, h, gy, *w, flags, *bufs, torch.empty(n, 4 * H, device=dev))
    else:
        fwd = lambda: ops.lstm_fwd(x, h, c, *w, flags)
        bwd = lambda: ops.lstm_bwd(x, h, c, gy, gy, *w, flags, *bufs)
    if accepted:
        outs = fwd() if cell == "lstm" else (fwd(),)
        grads = bwd()
        torch.cuda.synchronize()
        assert all(torch.isfinite(t).all() for t in tuple(outs) + tuple(grads))
    else:
        with pytest.raises(RuntimeError, match="not supported"):
            fwd()
        with pytest.raises(RuntimeError, match="not supported"):
            bwd()


def _make_cell(cell, H, ln, ig, bias, seed, offset=False):
    """The module and a float32 copy of its state: non-zero biases N(0, 0.3) and an input gate whose
    weights N(0, 4/H) spread sigmoid(q) over (0.1, 0.9) rather than about 0.5.  offset: every row of the
    three weight matrices is centred, and the gate weights' rows are then shifted by 1/H, so that with
    inputs around +30 each hidden-side gate pre-activation carries a common offset of about 30 over a
    spread of about 0.6 (the layer norm must cancel it) while the input gate stays off saturation."""
    from superpoint_graph_b200.spg_modules import GRUCellEx, LSTMCellEx
    torch.manual_seed(seed)
    mod = (GRUCellEx if cell == "gru" else LSTMCellEx)(H, H, bias=bias, layernorm=ln, ingate=ig)
    with torch.no_grad():
        for k, p in mod.named_parameters():
            if "bias" in k:
                p.normal_(0, 0.3)
        if ig:
            mod.ig.weight.normal_(0, 2 * H ** -0.5)
        if offset:
            for p in (mod.weight_ih, mod.weight_hh) + ((mod.ig.weight,) if ig else ()):
                p.sub_(p.mean(1, keepdim=True))
            mod.weight_ih.add_(1.0 / H)
            mod.weight_hh.add_(1.0 / H)
    sd = {k: v.clone() for k, v in mod.state_dict().items()}
    return mod, sd


def _gru_oracle(sd, x, h, g, ln, ig):
    """float64 autograd through nets_ref.gru_cell_ex: hy and the gradients of <hy, g>."""
    sd = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    x, h = (v.double().clone().requires_grad_(True) for v in (x, h))
    hy = nets_ref.gru_cell_ex(x, h, sd, "", ln, ig)
    (hy * g.double()).sum().backward()
    return hy.detach(), x.grad, h.grad, {k: v.grad for k, v in sd.items()}


def _check_cell(dev, cell, H, n, ln=True, ig=True, bias=True, offset=False):
    mod, sd = _make_cell(cell, H, ln, ig, bias, seed=1000 * H + n + 7 * ln + 3 * ig + bias + 11 * offset,
                         offset=offset)
    G = GATES[cell] * H
    if not bias:  # the oracles add the biases unconditionally (GRU) or take them if present (LSTM)
        sd["bias_ih"], sd["bias_hh"] = torch.zeros(G), torch.zeros(G)
    x, h, c, g, gc = (torch.randn(n, H) for _ in range(5))
    if offset:
        x, h = x + 30, h + 30
    mod.to(dev)
    xd, hd, cd = (v.to(dev).requires_grad_(True) for v in (x, h, c))
    if cell == "gru":
        hy_r, gx_r, gh_r, grads_r = _gru_oracle(sd, x, h, g, ln, ig)
        hy = mod(xd, hd)
        close(hy, hy_r, 1e-4)
        (hy * g.to(dev)).sum().backward()
    else:
        hy_r, cy_r, gx_r, gh_r, gc_r, grads_r = _lstm_oracle(sd, x, h, c, g, gc, ln, ig)
        hy, cy = mod(xd, (hd, cd))
        close(hy, hy_r, 1e-4)
        close(cy, cy_r, 1e-4)
        ((hy * g.to(dev)).sum() + (cy * gc.to(dev)).sum()).backward()
        close(cd.grad, gc_r, 3e-4)
    close(xd.grad, gx_r, 3e-4)
    close(hd.grad, gh_r, 3e-4)
    have = {k: p.grad for k, p in mod.named_parameters()}
    want = {k: v for k, v in grads_r.items() if bias or "bias_" not in k}
    assert set(have) == set(want), (sorted(have), sorted(want))  # bias off: no bias gradients
    close_grads(have, want, 3e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(CELL_CASES), ids=lambda k: "%s-H%d-n%d" % k)
def test_cell_vs_float64(dev, key):
    """Every (cell, NU, RW) instantiation at ragged row counts and widths off the column groups, all
    options on: hy (and cy), dL/dx, dL/dh (and dL/dc, from both hy and cy) and every parameter gradient."""
    from superpoint_graph_b200 import ops
    cell, H, n = key
    ops.prof_reset()
    _check_cell(dev, cell, H, n)
    assert ops.prof_collect()["%s_cell_bwd" % cell][0] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("n", FLAG_ROWS)
@pytest.mark.parametrize("ln,ig,bias", ALL_FLAGS, ids=lambda v: str(int(v)))
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_cell_flags_vs_float64(dev, cell, ln, ig, bias, n):
    """All 8 {LAYERNORM, INGATE, BIAS} combinations at H = 48 (NU = 2), with 1 and 4 rows per warp.  BIAS
    off: the reference computes with zero biases and the module has no bias parameters."""
    _check_cell(dev, cell, FLAG_H, n, ln, ig, bias)


@pytest.mark.gpu
@pytest.mark.parametrize("n", FLAG_ROWS)
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_cell_layernorm_cancels_common_offset(dev, cell, n):
    """Gate pre-activations around 30 with a spread of about 0.6: the layer norm's two-pass statistics
    cancel the offset (E[y^2] - E[y]^2 in float32 would lose about 3 of the 7 digits here)."""
    _check_cell(dev, cell, FLAG_H, n, offset=True)


# ------------------------------------------------------------------------------------- generic ECC
def _heavy_tailed_graph(rng, n_out, n_in, unread=()):
    """Degrees 0..200 (geometric, mean ~7: many nodes of degree 1..9; a few of 0 and of 200); sources
    drawn from [0, n_in) except `unread`."""
    degs = np.minimum(rng.geometric(0.12, size=n_out) - 1, 200)
    degs[:5] = 0
    degs[5:9] = 200
    rng.shuffle(degs)
    E = int(degs.sum())
    pool = np.setdiff1d(np.arange(n_in), np.asarray(unread, dtype=np.int64))
    idxn = pool[rng.integers(0, len(pool), size=E)]
    return torch.from_numpy(degs.astype(np.int64)), torch.from_numpy(idxn.astype(np.int64))


GRAPHS = {"square": (700, 700, ()), "bipartite": (500, 820, tuple(range(0, 820, 7)) + tuple(range(760, 820)))}


def _ecc_case(kind, mat, c_in, c_out, idxe, seed):
    rng = np.random.default_rng(seed)
    n_out, n_in, unread = GRAPHS[kind]
    degs, idxn = _heavy_tailed_graph(rng, n_out, n_in, unread)
    E = idxn.numel()
    n_w = 37 if idxe else E
    ie = torch.from_numpy(rng.integers(0, n_w, size=E).astype(np.int64)) if idxe else None
    if idxe:
        ie[:n_w] = torch.arange(n_w)  # every filter is used
    torch.manual_seed(seed)
    w = torch.randn(n_w, c_in, c_out) * c_in ** -0.5 if mat else torch.randn(n_w, c_in)
    return degs, idxn, ie, w, n_in, unread


def _ecc_kernels_ran(ops):
    return {k for k in ops.prof_collect() if k.startswith("ecc_")}


ECC_SHAPES = [(False, 1, 1), (False, 13, 13), (False, 31, 31), (False, 33, 33), (False, 64, 64),
              (True, 8, 12), (True, 13, 13), (True, 64, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("idxe", [False, True])
@pytest.mark.parametrize("kind", sorted(GRAPHS))
@pytest.mark.parametrize("mat,c_in,c_out", ECC_SHAPES, ids=lambda v: str(int(v)))
def test_ecc_generic_vs_oracle(dev, mat, c_in, c_out, kind, idxe):
    """ecc_generic_{fwd,bwd_x,bwd_w}_kernel<float> on heavy-tailed degrees, square and bipartite
    (n_in > n_out, sources no edge reads), with and without idxe (filter gradient by atomics): forward,
    grad_x with no / one / both addends, grad_w over 1 and 3 iterations and accumulated onto itself.
    fp32 sums of at most 200 products per output (x 64 for matrix filters): 1e-5 of the maximum."""
    from superpoint_graph_b200 import ops
    seed = 17 * c_in + c_out + 1000 * mat + 100 * idxe + (7 if kind == "bipartite" else 0)
    degs, idxn, ie, w, n_in, unread = _ecc_case(kind, mat, c_in, c_out, idxe, seed)
    graph = ops.EccGraph(idxn, ie, degs, n_in=n_in)
    xs = torch.randn(3, n_in, c_in)
    gs = torch.randn(3, degs.numel(), c_out)
    wd = w.to(dev)

    ops.prof_reset()
    out = ops.ecc_fwd(xs[0].to(dev), wd, graph, c_out)
    assert _ecc_kernels_ran(ops) == {"ecc_generic_fwd"}
    close(out, ecc_ref.graph_conv_forward(xs[0].double(), w.double(), idxn, ie, degs), 1e-5)

    rgx, _ = ecc_ref.graph_conv_backward(xs[0].double(), w.double(), idxn, ie, degs, gs[0].double())
    a0, a1 = torch.randn(n_in, c_in), torch.randn(n_in, c_in)
    for add0, add1 in ((None, None), (a0, None), (None, a1), (a0, a1)):
        ops.prof_reset()
        gx = ops.ecc_bwd_x(wd, gs[0].to(dev), graph, c_in, add0=None if add0 is None else add0.to(dev),
                           add1=None if add1 is None else add1.to(dev))
        assert _ecc_kernels_ran(ops) == {"ecc_generic_bwd_x"}
        adds = torch.zeros(n_in, c_in)
        for a in (add0, add1):
            if a is not None:
                adds = adds + a
        close(gx, rgx + adds.double(), 1e-5)
        if unread:
            assert torch.equal(gx.cpu()[list(unread)], adds[list(unread)])

    for n_iter in (1, 3):
        rgw = sum(ecc_ref.graph_conv_backward(xs[r].double(), w.double(), idxn, ie, degs, gs[r].double())[1]
                  for r in range(n_iter))
        xin, gin = (xs[0], gs[0]) if n_iter == 1 else (xs, gs)
        ops.prof_reset()
        gw = ops.ecc_bwd_w(xin.to(dev), gin.to(dev), graph, tuple(w.shape), n_iter=n_iter)
        close(gw, rgw, 1e-5)
        gw2 = ops.ecc_bwd_w(xin.to(dev), gin.to(dev), graph, tuple(w.shape), n_iter=n_iter, out=gw.clone(),
                            accumulate=True)
        assert _ecc_kernels_ran(ops) == {"ecc_generic_bwd_w"}
        close(gw2, 2 * rgw, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("mat", [False, True])
def test_ecc_32_channels_misaligned_takes_generic_path(dev, mat):
    """C = 32 with every operand at a 4-byte storage offset: the dispatcher's 16-byte alignment check
    sends the problem to the generic kernels, which agree with the fast path on aligned copies (and both
    with the oracle) to 1e-5 of the maximum."""
    from superpoint_graph_b200 import ops
    rng = np.random.default_rng(5 + mat)
    degs, idxn = _heavy_tailed_graph(rng, 600, 600)
    graph = ops.EccGraph(idxn, None, degs, n_in=600)
    E, C = idxn.numel(), 32
    torch.manual_seed(6)
    w = torch.randn(E, C, C) * C ** -0.5 if mat else torch.randn(E, C)
    xs, gs = torch.randn(3, 600, C), torch.randn(3, 600, C)
    a0, a1 = torch.randn(600, C), torch.randn(600, C)

    def off(t):  # the same values 4 bytes past a 16-byte boundary
        buf = torch.empty(t.numel() + 4, device=dev)
        v = buf[1:1 + t.numel()].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.data_ptr() % 16 == 4
        return v

    fast = "ecc_mat_" if mat else "ecc_vv_"
    res = {}
    for path, put in (("fast", lambda t: t.to(dev)), ("generic", off)):
        ops.prof_reset()
        fwd = ops.ecc_fwd(put(xs[0]), put(w), graph, C)
        gx = ops.ecc_bwd_x(put(w), put(gs[0]), graph, C, add0=put(a0), add1=put(a1))
        gw = ops.ecc_bwd_w(put(xs), put(gs), graph, tuple(w.shape), n_iter=3)
        ran = _ecc_kernels_ran(ops)
        prefix = "ecc_generic_" if path == "generic" else fast
        assert ran == {prefix + s for s in ("fwd", "bwd_x", "bwd_w")}, ran
        res[path] = (fwd, gx, gw)
    rgx, _ = ecc_ref.graph_conv_backward(xs[0].double(), w.double(), idxn, None, degs, gs[0].double())
    want = (ecc_ref.graph_conv_forward(xs[0].double(), w.double(), idxn, None, degs),
            rgx + a0.double() + a1.double(),
            sum(ecc_ref.graph_conv_backward(xs[r].double(), w.double(), idxn, None, degs, gs[r].double())[1]
                for r in range(3)))
    for f, g, r in zip(res["fast"], res["generic"], want):
        close(g, f, 1e-5)
        close(g, r, 1e-5)


# ------------------------------------------------------------------------------ block and training step
def _block(cell, H, mat, cat_all, n, seed):
    from superpoint_graph_b200 import synthetic
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_graphnet import create_fnet
    from superpoint_graph_b200.spg_modules import GRUCellEx, LSTMCellEx, RNNGraphConvModule
    torch.manual_seed(seed)
    b = synthetic.make_batch(n, k=8, seed=seed, npts=8, minpts=4)
    gi = GraphConvInfo.from_arrays(b["idxn"].numpy(), b["degs"].numpy(), b["edgefeats"].numpy())
    gi.cuda()
    widths = [13, 32, 128, 64, H * H if mat else H]
    fnet = create_fnet(widths, True, 0, 2)
    cmod = (GRUCellEx if cell == "gru" else LSTMCellEx)(H, H, bias=True, layernorm=True, ingate=True)
    with torch.no_grad():
        for k, p in cmod.named_parameters():
            if "bias" in k:
                p.normal_(0, 0.3)
        cmod.ig.weight.normal_(0, 2 * H ** -0.5)
    mod = RNNGraphConvModule(cmod, fnet, H, vv=not mat, gc_info=gi, nrepeats=3, cat_all=cat_all,
                             use_pyg=False, cuda=True)
    mcfg = dict(fnet_widths=widths, bnidx=2, nrepeats=3, layernorm=True, ingate=True, cat_all=cat_all)
    return mod, gi, b, mcfg


BLOCK_CASES = [(cell, H, mat, cat_all, 1000) for cell in ("gru", "lstm") for H in (16, 64) for mat in (False, True)
               for cat_all in (False, True) if not (mat and H == 64)] + [("gru", 64, False, False, 9000)]


@pytest.mark.gpu
@pytest.mark.parametrize("cell,H,mat,cat_all,n", BLOCK_CASES)
def test_recurrent_block_vs_float64(dev, cell, H, mat, cat_all, n):
    """RNNGraphConvModule at H != 32 (the per-step path: generic ECC, cell kernels, SIMT weight-gradient
    GEMMs), 3 repeats, against the float64 oracle: output, dL/dx and every filter-network and cell parameter
    gradient.  9000 nodes run the recurrence's cells with 4 rows per warp."""
    from superpoint_graph_b200 import ops
    mod, gi, b, mcfg = _block(cell, H, mat, cat_all, n, seed=H + n + 2 * mat + cat_all)
    sd = {"0." + k: v.double().clone().requires_grad_(nets_ref.is_param(k)) for k, v in mod.state_dict().items()}
    mod.to(dev).train()
    wshape = (1, H, H) if mat else (1, H)
    assert not ops.rnn_vv_supported(torch.empty(wshape, device=dev), gi.graph(), n, H)
    x0 = torch.randn(n, H)
    x = x0.to(dev).requires_grad_(True)
    ops.prof_reset()
    y = mod(x)
    gout = torch.linspace(-1, 1, y.numel()).view(y.shape)
    (y * gout.to(dev)).sum().backward()
    ran = ops.prof_collect()
    assert not any(k.startswith("rnn_ecc_") for k in ran), ran
    assert ran["ecc_generic_fwd"][0] == 3 and ran["ecc_generic_bwd_x"][0] == 3 and ran["ecc_generic_bwd_w"][0] == 1
    assert ran["%s_cell_fwd" % cell][0] == 3 and ran["%s_cell_bwd" % cell][0] == 3
    xr = x0.double().requires_grad_(True)
    ef = b["edgefeats"].double()
    if cell == "gru":
        yr = nets_ref.rnn_ecc_forward(xr, ef, b["idxn"], b["degs"], sd, "0.", mcfg, True)
    else:
        yr = lstm_ref.rnn_ecc_forward(xr, ef, b["idxn"], b["degs"], sd, "0.", mcfg, True, cell="lstm")
    (yr * gout.double()).sum().backward()
    close(y, yr, 1e-4)
    close(x.grad, xr.grad, 3e-4, 1e-5 * float(xr.grad.abs().max()))
    want = {k[2:]: v.grad for k, v in sd.items() if nets_ref.is_param(k[2:])}
    have = {k: p.grad for k, p in mod.named_parameters()}
    assert set(have) == set(want)
    close_grads(have, want, 3e-4)


@pytest.mark.gpu
def test_train_step_hidden_width_64_vs_oracle(dev):
    """One Trainer.train_step of s3dis_train's flags with ptn_widths [[64, 64, 128, 128, 256], [256, 64, 64]],
    so H = 64 and the recurrence runs per step: loss, logits and every gradient against the float64
    RefTrainer, with test_gpu_shapes' bounds."""
    from superpoint_graph_b200 import ops, workloads
    from superpoint_graph_b200.trainer import HostBatch
    from test_gpu_shapes import _check_grads, _f64, _model_and_oracle, _ref_grads
    w = workloads.get("s3dis_train")
    w["margs"].ptn_widths = [[64, 64, 128, 128, 256], [256, 64, 64]]
    batch = workloads.batch(w, 2)
    model, tr, ref, skip = _model_and_oracle(w, dev)
    assert model.ecc.state_dict()["0._cell.weight_hh"].shape == (3 * 64, 64)
    db = HostBatch(batch).to_device(dev)
    assert not ops.rnn_vv_supported(torch.empty(1, 64, device=dev), db.gi.graph(), w["nodes"], 64)
    loss, logits = tr.train_step(db)
    ref_loss, ref_logits = ref.step(_f64(batch))
    close(logits, ref_logits, 1e-4)
    assert abs(float(loss[0]) - ref_loss) <= 1e-4 * abs(ref_loss)
    _check_grads(model, _ref_grads(ref), skip)
