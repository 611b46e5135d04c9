"""Recurrent ECC module and GRUCellEx with the reference's signatures (ref:
learning/modules.py:128-183, 205-259), executed as ONE autograd node over the sm_90a kernels:

  filters  = fnet(edge features)                      (once, fused Linear/BN/ReLU chain)
  repeat R: input = ECC(h, filters); h = GRUCellEx(input, h)
  backward: per step GRU-cell backward + ECC grad_input (source-CSR, no atomics); the filter
            gradient of all R steps is produced by one batched kernel, the cell's weight
            gradients by three GEMMs over the R*N stacked per-row factors.

The reference builds ~25 autograd nodes per recurrent step and sums R separate [E,C(,C)]
filter-gradient tensors; nothing of that is materialised here.
"""
import torch
import torch.nn as nn

from . import ops
from .dense import Deferred, chain_backward, chain_forward, parse_sequential


class GRUCellEx(nn.GRUCell):
    """GRU cell with layer normalisation of both gate pre-activations and an input gate
    (ref: learning/modules.py:205-259).  Parameter names/shapes are those of nn.GRUCell plus
    `ig.weight`, `ig.bias`; `ini`/`inh` exist for state-dict/printing parity only."""

    def __init__(self, input_size, hidden_size, bias=True, layernorm=True, ingate=True):
        super(GRUCellEx, self).__init__(input_size, hidden_size, bias)
        self._layernorm = layernorm
        self._ingate = ingate
        if layernorm:
            self.add_module('ini', nn.InstanceNorm1d(1, eps=1e-5, affine=False, track_running_stats=False))
            self.add_module('inh', nn.InstanceNorm1d(1, eps=1e-5, affine=False, track_running_stats=False))
        if ingate:
            self.add_module('ig', nn.Linear(hidden_size, input_size, bias=True))

    def flags(self):
        f = 0
        if self._layernorm:
            f |= ops.GRU_LAYERNORM
        if self._ingate:
            f |= ops.GRU_INGATE
        if self.bias:
            f |= ops.GRU_BIAS
        return f

    def cell_params(self):
        """[weight_ih, weight_hh, bias_ih|None, bias_hh|None, ig.weight|None, ig.bias|None]"""
        ig = self._modules['ig'] if self._ingate else None
        return [self.weight_ih, self.weight_hh,
                self.bias_ih if self.bias else None, self.bias_hh if self.bias else None,
                ig.weight if ig is not None else None, ig.bias if ig is not None else None]

    def forward(self, input, hidden):
        if self.input_size != self.hidden_size:
            raise NotImplementedError("GRUCellEx kernels need input_size == hidden_size "
                                      "(always true for graphnet.py:74)")
        p = self.cell_params()
        present = [q for q in p if q is not None]
        return _GRUCellFunction.apply(input, hidden, self.flags(), *present)

    def __repr__(self):
        s = super(GRUCellEx, self).__repr__() + '('
        if self._ingate:
            s += 'ingate'
        if self._layernorm:
            s += ' layernorm'
        return s + ')'


def _unpack_cell(flags, present):
    """present (list of tensors) -> (w_ih, w_hh, b_ih, b_hh, w_ig, b_ig) with None holes."""
    it = iter(present)
    w_ih, w_hh = next(it), next(it)
    b_ih = b_hh = w_ig = b_ig = None
    if flags & ops.GRU_BIAS:
        b_ih, b_hh = next(it), next(it)
    if flags & ops.GRU_INGATE:
        w_ig, b_ig = next(it), next(it)
    return w_ih, w_hh, b_ih, b_hh, w_ig, b_ig


def _cell_weight_grads(flags, d_gi, d_gh, d_q, xprime, hs, dpre, rows, H):
    """Parameter gradients of the cell from the stacked per-row factors ([rows, .])."""
    g_wih = ops.gemm(d_gi, 3 * H, False, xprime, H, False, 3 * H, H, rows)
    g_whh = ops.gemm(d_gh, 3 * H, False, hs, H, False, 3 * H, H, rows)
    out = [g_wih, g_whh]
    if flags & ops.GRU_BIAS:
        cs = ops.colsum(dpre, 4 * H, rows, 4 * H)
        g_bih = cs[:3 * H].contiguous()
        g_bhh = torch.cat([cs[:2 * H], cs[3 * H:]])
        out += [g_bih, g_bhh]
    if flags & ops.GRU_INGATE:
        g_wig = ops.gemm(d_q, H, False, hs, H, False, H, H, rows)
        g_big = ops.colsum(d_q, H, rows, H)
        out += [g_wig, g_big]
    return out


class _GRUCellFunction(torch.autograd.Function):
    """Stand-alone cell (API parity); the recurrent module below does not go through it."""

    @staticmethod
    def forward(ctx, x, h, flags, *present):
        x, h = x.contiguous(), h.contiguous()
        w = _unpack_cell(flags, present)
        hy = ops.gru_fwd(x, h, *w, flags)
        ctx.save_for_backward(x, h)
        ctx.flags, ctx.present = flags, present
        return hy

    @staticmethod
    def backward(ctx, gy):
        x, h = ctx.saved_tensors
        flags = ctx.flags
        n, H = h.shape
        dev = h.device
        w = _unpack_cell(flags, ctx.present)
        d_gi = torch.empty((n, 3 * H), device=dev)
        d_gh = torch.empty((n, 3 * H), device=dev)
        d_q = torch.empty((n, H), device=dev)
        xp = torch.empty((n, H), device=dev)
        dpre = torch.empty((n, 4 * H), device=dev)
        d_x, d_h = ops.gru_bwd(x, h, gy.contiguous(), *w, flags, d_gi, d_gh, d_q, xp, dpre)
        grads = _cell_weight_grads(flags, d_gi, d_gh, d_q, xp, h, dpre, n, H)
        return (d_x, d_h, None) + tuple(grads)


class RNNGraphConvModule(nn.Module):
    """Recurrent graph convolution: filters from `filter_net` (evaluated once), `nrepeats` x
    {ECC -> RNN cell} with shared weights (ref: learning/modules.py:128-183)."""

    def __init__(self, cell, filter_net, nfeat, vv=True, gc_info=None, nrepeats=1, cat_all=False,
                 edge_mem_limit=1e20, use_pyg=True, cuda=True):
        super(RNNGraphConvModule, self).__init__()
        self._cell = cell
        self._isLSTM = 'LSTM' in type(cell).__name__
        self._fnet = filter_net
        self._nrepeats = nrepeats
        self._cat_all = cat_all
        self._edge_mem_limit = edge_mem_limit
        self.set_info(gc_info)
        self.use_pyg = use_pyg
        if use_pyg:
            raise NotImplementedError(
                "use_pyg=1 selects the reference's torch_geometric path; the sm_90a kernels "
                "implement the native ECC path (use --use_pyg 0)")
        if self._isLSTM:
            raise NotImplementedError("lstm_* model configs are outside the accelerated path")

    def set_info(self, gc_info):
        self._gci = gc_info
        self._prefetched = None

    def prefetch_filters(self, inline=False):
        """Evaluate the filter network now — it depends on the edge features alone.  Trainer (ops.SIDE
        installed): on the side stream, underneath the PointNet forward; forward() picks the result up and
        joins the stream.  inline=True: on the current stream (the pipelined inference path runs it while
        the point clouds are still being uploaded)."""
        side = None if inline else ops.SIDE[0]
        if (side is None and not inline) or self._gci is None:
            return
        edgefeats = self._gci.get_buffers()[4]
        fspecs, fparams = parse_sequential(self._fnet, self.training)
        if side is None:
            self._prefetched = (self._gci, self.training, False) + _filter_bank(edgefeats, fspecs, fparams,
                                                                                self.training)
            return
        with side.fork(edgefeats):
            self._prefetched = (self._gci, self.training, True) + _filter_bank(edgefeats, fspecs, fparams,
                                                                               self.training)

    def forward(self, hx):
        idxn, idxe, degs, degs_gpu, edgefeats = self._gci.get_buffers()
        graph = self._gci.graph()
        cell = self._cell
        fspecs, fparams = parse_sequential(self._fnet, self.training)
        cparams = [q for q in cell.cell_params() if q is not None]
        pre, self._prefetched = self._prefetched, None
        if pre is not None:
            if pre[0] is not self._gci or pre[1] != self.training or (pre[2] and ops.SIDE[0] is None):
                raise RuntimeError("prefetch_filters() result does not belong to this forward")
            if pre[2]:
                ops.SIDE[0].join()
            pre = pre[3:]
        return _RecurrentECCFunction.apply(hx, edgefeats, graph, fspecs, len(fparams), cell.flags(),
                                           self._nrepeats, self._cat_all, self.training, pre,
                                           *(fparams + cparams))


def _filter_bank(edgefeats, fspecs, fparams, training):
    """fnet(edgefeats) -> (weights [E, width], saved activations, pending BN state)."""
    edgefeats = edgefeats.contiguous()
    if edgefeats.dtype != torch.float32:
        edgefeats = edgefeats.float()
    E, Fe = edgefeats.shape
    fsaved = [] if training else None
    wdef = chain_forward(Deferred(edgefeats, Fe, Fe), E, fspecs, fparams, training, fsaved)
    return wdef.materialise(E), fsaved, wdef.pending


class _RecurrentECCFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, hx, edgefeats, graph, fspecs, n_fparams, flags, nrepeats, cat_all, training,
                pre, *params):
        fparams, cpresent = params[:n_fparams], params[n_fparams:]
        hx = hx.contiguous()
        N, H = hx.shape
        E = edgefeats.shape[0]
        dev = hx.device
        # 1) filter bank, once (possibly evaluated ahead of time on the side stream)
        weights, fsaved, w_pending = pre if pre is not None else _filter_bank(edgefeats, fspecs,
                                                                              fparams, training)
        assert weights.size(1) in (H, H * H)
        if weights.size(1) != H:
            weights = weights.view(E, H, H)
        # 2) R x {ECC, cell}; all hidden states live in one [R+1, N, H] buffer
        w = _unpack_cell(flags, cpresent)
        hs = torch.empty((nrepeats + 1, N, H), dtype=torch.float32, device=dev)
        hs[0].copy_(hx)
        fused = nrepeats > 0 and ops.rnn_vv_supported(weights, graph, N, H)
        inps = (torch.empty((nrepeats, N, H), dtype=torch.float32, device=dev)
                if training or fused else None)
        if fused:
            ops.rnn_vv_fwd(hs, inps, weights, graph, w, flags)
        else:
            for r in range(nrepeats):
                inp = ops.ecc_fwd(hs[r], weights, graph, H, out=inps[r] if training else None)
                ops.gru_fwd(inp, hs[r], *w, flags, out=hs[r + 1])
        if training:
            ctx.save_for_backward(hs, inps, weights)
        ctx.meta = (graph, fspecs, n_fparams, flags, nrepeats, cat_all, training, fsaved,
                    w_pending, params, N, H, E)
        if cat_all:
            return hs.permute(1, 0, 2).reshape(N, (nrepeats + 1) * H)
        return hs[nrepeats].clone()

    @staticmethod
    def backward(ctx, gout):
        (graph, fspecs, n_fparams, flags, R, cat_all, training, fsaved, w_pending, params, N, H,
         E) = ctx.meta
        if not training:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        hs, inps, weights = ctx.saved_tensors
        fparams, cpresent = params[:n_fparams], params[n_fparams:]
        w = _unpack_cell(flags, cpresent)
        dev = hs.device
        gout = gout.contiguous()
        if cat_all:
            gcat = gout.view(N, R + 1, H).permute(1, 0, 2).contiguous()  # [R+1, N, H]
            gh = gcat[R]
        else:
            gcat = None
            gh = gout
        d_gi = torch.empty((R, N, 3 * H), device=dev)
        d_gh = torch.empty((R, N, 3 * H), device=dev)
        d_q = torch.empty((R, N, H), device=dev)
        xp = torch.empty((R, N, H), device=dev)
        dpre = torch.empty((R, N, 4 * H), device=dev)
        ginp = torch.empty((R, N, H), device=dev)
        if R > 0 and ops.rnn_vv_supported(weights, graph, N, H):
            gh = ops.rnn_vv_bwd(hs, inps, weights, graph, w, flags, gh, gcat, ginp, d_gi, d_gh, d_q,
                                xp, dpre)
        else:
            for r in range(R - 1, -1, -1):
                d_x, d_h = ops.gru_bwd(inps[r], hs[r], gh, *w, flags, d_gi[r], d_gh[r], d_q[r],
                                       xp[r], dpre[r], d_x=ginp[r])
                # gradient w.r.t. h_r: through the cell (d_h), through the ECC (source-CSR gather)
                # and, with cat_all, the direct gradient of the concatenated output
                gh = ops.ecc_bwd_x(weights, d_x, graph, H, add0=d_h,
                                   add1=None if gcat is None else gcat[r])
        g_hx = gh if ctx.needs_input_grad[0] else None

        def parameter_grads():
            # filter gradient of all R steps in one pass
            g_w = ops.ecc_bwd_w(hs[:R], ginp, graph, tuple(weights.shape), n_iter=R)
            grads_f = [None] * n_fparams
            chain_backward(g_w.view(E, -1), g_w.numel() // E, E, fspecs, fparams, fsaved, False,
                           grads_f, own_g=True)
            grads_c = _cell_weight_grads(flags, d_gi.view(R * N, 3 * H), d_gh.view(R * N, 3 * H),
                                         d_q.view(R * N, H), xp.view(R * N, H),
                                         hs[:R].view(R * N, H), dpre.view(R * N, 4 * H), R * N, H)
            return tuple(grads_f) + tuple(grads_c)

        side = ops.SIDE[0]
        if side is None:
            return (g_hx, None, None, None, None, None, None, None, None, None) + parameter_grads()
        # Trainer mode: the parameter gradients of this block do not feed anything upstream, so
        # they run on the side stream underneath the PointNet backward that follows.  They are
        # written to .grad here (the autograd engine must not touch tensors another stream is
        # still producing); Trainer.compute_gradients joins the stream before it reads them.
        with side.fork(hs, inps, weights, ginp, d_gi, d_gh, d_q, xp, dpre, fsaved, gout):
            grads = parameter_grads()
            for prm, g in zip(params, grads):
                if g is not None and prm.requires_grad:
                    prm.grad = g if prm.grad is None else prm.grad + g
        return (g_hx,) + (None,) * (9 + len(params))


class ECC_CRFModule(nn.Module):
    """Signature kept (ref: learning/modules.py:185-202); `crf_*` configs are outside the
    accelerated path of this round."""

    def __init__(self, propagation, nrepeats=1):
        super(ECC_CRFModule, self).__init__()
        raise NotImplementedError("crf_* model configs are outside the accelerated path")


class LSTMCellEx(nn.LSTMCell):
    """Signature kept (ref: learning/modules.py:262-316); not on the accelerated path."""

    def __init__(self, input_size, hidden_size, bias=True, layernorm=True, ingate=True):
        super(LSTMCellEx, self).__init__(input_size, hidden_size, bias)
        raise NotImplementedError("lstm_* model configs are outside the accelerated path")
