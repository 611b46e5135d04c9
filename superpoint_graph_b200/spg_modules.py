"""Recurrent ECC module, ECC_CRFModule, GRUCellEx and LSTMCellEx with the reference's signatures (ref:
learning/modules.py:128-316); the recurrent module is executed as ONE autograd node over the sm_90a
kernels (the CRF module likewise, see ECC_CRFModule):

  filters  = fnet(edge features)                      (once, fused Linear/BN/ReLU chain)
  repeat R: input = ECC(h, filters); h = GRUCellEx(input, h)   or   (h, c) = LSTMCellEx(input, (h, c))
  backward: per step cell backward + ECC grad_input (source-CSR, no atomics); the filter
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

    # ---- what the recurrent module needs to know about the cell (see _RecurrentECCFunction)
    N_GATES = 3

    @staticmethod
    def _new_state(R, N, H, dev):
        return None

    @staticmethod
    def _new_dpre(R, N, H, dev):
        return torch.empty((R, N, 4 * H), device=dev)

    @staticmethod
    def _step_forward(inp, hs, cs, r, w, flags):
        ops.gru_fwd(inp, hs[r], *w, flags, out=hs[r + 1])

    @staticmethod
    def _step_backward(inps, hs, cs, r, gh, dc, w, flags, d_gi, d_gh, d_q, xp, dpre, ginp):
        """Cell backward of step r into ginp[r]; returns dL/dh_r through the cell."""
        return ops.gru_bwd(inps[r], hs[r], gh, *w, flags, d_gi[r], d_gh[r], d_q[r], xp[r], dpre[r],
                           d_x=ginp[r])[1]

    @staticmethod
    def _bias_grads(d_gi, d_gh, dpre, rows, H):
        cs = ops.colsum(dpre, 4 * H, rows, 4 * H)
        return [cs[:3 * H].contiguous(), torch.cat([cs[:2 * H], cs[3 * H:]])]

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


def _cell_weight_grads(cell_cls, flags, d_gi, d_gh, d_q, xprime, hs, dpre, rows, H):
    """Parameter gradients of the cell from the stacked per-row factors ([rows, .])."""
    G = cell_cls.N_GATES * H
    g_wih = ops.gemm(d_gi, G, False, xprime, H, False, G, H, rows)
    g_whh = ops.gemm(d_gh, G, False, hs, H, False, G, H, rows)
    out = [g_wih, g_whh]
    if flags & ops.GRU_BIAS:
        out += cell_cls._bias_grads(d_gi, d_gh, dpre, rows, H)
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
        grads = _cell_weight_grads(GRUCellEx, flags, d_gi, d_gh, d_q, xp, h, dpre, n, H)
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
        return _RecurrentECCFunction.apply(hx, edgefeats, graph, fspecs, len(fparams), type(cell),
                                           cell.flags(), self._nrepeats, self._cat_all, self.training,
                                           pre, *(fparams + cparams))


def _filter_bank(edgefeats, fspecs, fparams, training, bn_repeats=1):
    """fnet(edgefeats) -> (weights [E, width], saved activations, pending BN state)."""
    edgefeats = edgefeats.contiguous()
    if edgefeats.dtype != torch.float32:
        edgefeats = edgefeats.float()
    E, Fe = edgefeats.shape
    fsaved = [] if training else None
    wdef = chain_forward(Deferred(edgefeats, Fe, Fe), E, fspecs, fparams, training, fsaved, bn_repeats)
    return wdef.materialise(E), fsaved, wdef.pending


class _RecurrentECCFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, hx, edgefeats, graph, fspecs, n_fparams, cell_cls, flags, nrepeats, cat_all,
                training, pre, *params):
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
        # 2) R x {ECC, cell}; all hidden states live in one [R+1, N, H] buffer, the LSTM's cell
        #    states in another (c_0 = 0, ref: modules.py:168-169)
        w = _unpack_cell(flags, cpresent)
        hs = torch.empty((nrepeats + 1, N, H), dtype=torch.float32, device=dev)
        hs[0].copy_(hx)
        cs = cell_cls._new_state(nrepeats, N, H, dev)
        fused = nrepeats > 0 and ops.rnn_vv_supported(weights, graph, N, H)
        inps = (torch.empty((nrepeats, N, H), dtype=torch.float32, device=dev)
                if training or fused else None)
        if fused:
            ops.rnn_vv_fwd(hs, inps, weights, graph, w, flags, cs=cs)
        else:
            for r in range(nrepeats):
                inp = ops.ecc_fwd(hs[r], weights, graph, H, out=inps[r] if training else None)
                cell_cls._step_forward(inp, hs, cs, r, w, flags)
        if training:
            ctx.save_for_backward(hs, inps, weights, cs)
        ctx.meta = (graph, fspecs, n_fparams, cell_cls, flags, nrepeats, cat_all, training, fsaved,
                    w_pending, params, N, H, E)
        if cat_all:
            return hs.permute(1, 0, 2).reshape(N, (nrepeats + 1) * H)
        return hs[nrepeats].clone()

    @staticmethod
    def backward(ctx, gout):
        (graph, fspecs, n_fparams, cell_cls, flags, R, cat_all, training, fsaved, w_pending, params,
         N, H, E) = ctx.meta
        if not training:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        hs, inps, weights, cs = ctx.saved_tensors
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
        G = cell_cls.N_GATES * H
        d_gi = torch.empty((R, N, G), device=dev)
        d_gh = torch.empty((R, N, G), device=dev)
        d_q = torch.empty((R, N, H), device=dev)
        xp = torch.empty((R, N, H), device=dev)
        dpre = cell_cls._new_dpre(R, N, H, dev)
        ginp = torch.empty((R, N, H), device=dev)
        if R > 0 and ops.rnn_vv_supported(weights, graph, N, H):
            gh = ops.rnn_vv_bwd(hs, inps, weights, graph, w, flags, gh, gcat, ginp, d_gi, d_gh, d_q,
                                xp, dpre, cs=cs)
        else:
            dc = None if cs is None else torch.empty((N, H), device=dev)  # dL/dc, node-local
            for r in range(R - 1, -1, -1):
                d_h = cell_cls._step_backward(inps, hs, cs, r, gh, dc, w, flags, d_gi, d_gh, d_q, xp,
                                              dpre, ginp)
                # gradient w.r.t. h_r: through the cell (d_h), through the ECC (source-CSR gather)
                # and, with cat_all, the direct gradient of the concatenated output
                gh = ops.ecc_bwd_x(weights, ginp[r], graph, H, add0=d_h,
                                   add1=None if gcat is None else gcat[r])
        g_hx = gh if ctx.needs_input_grad[0] else None

        def parameter_grads():
            # filter gradient of all R steps in one pass
            g_w = ops.ecc_bwd_w(hs[:R], ginp, graph, tuple(weights.shape), n_iter=R)
            grads_f = [None] * n_fparams
            chain_backward(g_w.view(E, -1), g_w.numel() // E, E, fspecs, fparams, fsaved, False,
                           grads_f, own_g=True)
            grads_c = _cell_weight_grads(cell_cls, flags, d_gi.view(R * N, G), d_gh.view(R * N, G),
                                         d_q.view(R * N, H), xp.view(R * N, H), hs[:R].view(R * N, H),
                                         None if dpre is None else dpre.view(R * N, 4 * H), R * N, H)
            return tuple(grads_f) + tuple(grads_c)

        side = ops.SIDE[0]
        if side is None:
            return (g_hx,) + (None,) * 10 + parameter_grads()
        # Trainer mode: the parameter gradients of this block do not feed anything upstream, so
        # they run on the side stream underneath the PointNet backward that follows.  They are
        # written to .grad here (the autograd engine must not touch tensors another stream is
        # still producing); Trainer.compute_gradients joins the stream before it reads them.
        with side.fork(hs, inps, weights, ginp, d_gi, d_gh, d_q, xp, dpre, fsaved, gout):
            grads = parameter_grads()
            for prm, g in zip(params, grads):
                if g is not None and prm.requires_grad:
                    prm.grad = g if prm.grad is None else prm.grad + g
        return (g_hx,) + (None,) * (10 + len(params))


def _fnet_width(fnet):
    """Output width of a filter network (its last Linear layer)."""
    lins = [m for m in fnet.modules() if isinstance(m, nn.Linear)]
    return lins[-1].out_features if lins else None


class ECC_CRFModule(nn.Module):
    """ECC as a CRF mean-field recurrence (ref: learning/modules.py:185-202):

      Q = softmax(U);  repeat R: Q = U - propagation(Q), softmax except after the last step

    with `propagation` the package's GraphConvModule(C, C, fnet) over [E, C, C] matrix filters,
    C <= 32 (what GraphNetwork builds for `crf_<R>`).  Runs as ONE autograd node: the filter network
    is evaluated once (the R banks of the reference are identical; its BatchNorm running statistics
    still take R updates), one kernel per iteration in each direction, and the filter gradient of
    all R iterations comes from one pass."""

    def __init__(self, propagation, nrepeats=1):
        super(ECC_CRFModule, self).__init__()
        from .spg_ecc import GraphConvModule
        if not isinstance(propagation, GraphConvModule):
            raise NotImplementedError(
                "ECC_CRFModule runs with the package's GraphConvModule(C, C, fnet) as propagation "
                "(got %s)" % type(propagation).__name__)
        C = propagation._in_channels
        if propagation._out_channels != C or _fnet_width(propagation._fnet) != C * C:
            raise NotImplementedError(
                "ECC_CRFModule needs a GraphConvModule(C, C, fnet) with [E, C, C] matrix filters "
                "(fnet output width C*C); vector filters and C_in != C_out are not supported")
        if C > ops.CRF_MAX_C:
            raise NotImplementedError("the ECC-CRF kernels serve C <= %d classes (got C = %d)"
                                      % (ops.CRF_MAX_C, C))
        self._propagation = propagation
        self._nrepeats = nrepeats

    def forward(self, input):
        prop = self._propagation
        _, idxe, _, _, edgefeats = prop._gci.get_buffers()
        if idxe is not None:
            raise NotImplementedError("the ECC-CRF kernels do not take idxe (edge-feature compaction)")
        fspecs, fparams = parse_sequential(prop._fnet, self.training)
        return _CRFFunction.apply(input, edgefeats, prop._gci.graph(), fspecs, len(fparams),
                                  self._nrepeats, self.training, *fparams)


class _CRFFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, U, edgefeats, graph, fspecs, n_fparams, R, training, *fparams):
        U = U.contiguous()
        if U.dtype != torch.float32:
            raise TypeError("ECC_CRFModule runs in float32 (got %s)" % U.dtype)
        N, C = U.shape
        dev = U.device
        weights = fsaved = None
        if R == 0:  # softmax(U); the filter network never runs (ref: modules.py:196-202)
            out = ops.crf_softmax(U)
            qs = out.view(1, N, C)
        else:
            # Q_0 .. Q_{R-1}: all kept for the backward in training, two ping-pong buffers in eval
            qs = torch.empty((R if training else min(R, 2), N, C), dtype=torch.float32, device=dev)
            ops.crf_softmax(U, out=qs[0])
            weights, fsaved, _ = _filter_bank(edgefeats, fspecs, fparams, training, bn_repeats=R)
            E = weights.shape[0]
            if weights.shape[1] != C * C:
                raise ValueError("filter bank of width %d for C = %d" % (weights.shape[1], C))
            weights = weights.view(E, C, C)
            out = torch.empty((N, C), dtype=torch.float32, device=dev)
            for r in range(1, R + 1):
                src = qs[r - 1] if training else qs[(r - 1) % 2]
                dst = out if r == R else (qs[r] if training else qs[r % 2])
                ops.crf_fwd_step(U, src, weights, graph, dst, softmax=r < R)
        if training:
            ctx.save_for_backward(qs, weights)
        ctx.meta = (graph, fspecs, n_fparams, R, training, fsaved, fparams)
        return out

    @staticmethod
    def backward(ctx, gout):
        graph, fspecs, n_fparams, R, training, fsaved, fparams = ctx.meta
        if not training:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        qs, weights = ctx.saved_tensors
        gout = gout.contiguous()
        nones = (None,) * 6  # edgefeats, graph, fspecs, n_fparams, R, training
        if R == 0:
            return (ops.crf_softmax(qs[0], gout),) + nones + (None,) * n_fparams
        _, N, C = qs.shape
        E = weights.shape[0]
        # gps[r-1] = dL/dP_r (P_r: the propagation output of iteration r; Z_r = U - P_r)
        gps = torch.empty((R, N, C), dtype=torch.float32, device=qs.device)
        torch.neg(gout, out=gps[R - 1])
        g_u = torch.empty((N, C), dtype=torch.float32, device=qs.device)
        du_in = gout  # Z_R = U - P_R: the top gradient reaches U directly
        for r in range(R, 0, -1):
            ops.crf_bwd_step(weights, gps[r - 1], qs[r - 1], du_in, g_u, gps[r - 2] if r > 1 else None, graph)
            du_in = g_u

        def parameter_grads():
            # filter gradient of all R iterations in one pass: sum_r (1/deg) Q_{r-1}[src]^T (x) dL/dP_r[tgt]
            g_w = ops.ecc_bwd_w(qs, gps, graph, (E, C, C), n_iter=R)
            grads_f = [None] * n_fparams
            chain_backward(g_w.view(E, C * C), C * C, E, fspecs, fparams, fsaved, False, grads_f, own_g=True)
            return tuple(grads_f)

        side = ops.SIDE[0]
        if side is None:
            return (g_u,) + nones + parameter_grads()
        # Trainer mode: as _RecurrentECCFunction.backward, the filter-network gradients go on the side
        # stream, straight to .grad
        with side.fork(qs, weights, gps, fsaved, gout):
            for prm, g in zip(fparams, parameter_grads()):
                if g is not None and prm.requires_grad:
                    prm.grad = g if prm.grad is None else prm.grad + g
        return (g_u,) + nones + (None,) * n_fparams


class LSTMCellEx(nn.LSTMCell):
    """LSTM cell with layer normalisation of both gate pre-activations and an input gate
    (ref: learning/modules.py:262-316).  Parameter names/shapes are those of nn.LSTMCell plus
    `ig.weight`, `ig.bias`; `ini`/`inh` exist for state-dict/printing parity only.  Unlike GRUCellEx
    the biases enter inside the linears, before the norm (ref: :296-297)."""

    def __init__(self, input_size, hidden_size, bias=True, layernorm=True, ingate=True):
        super(LSTMCellEx, self).__init__(input_size, hidden_size, bias)
        self._layernorm = layernorm
        self._ingate = ingate
        if layernorm:
            self.add_module('ini', nn.InstanceNorm1d(1, eps=1e-5, affine=False, track_running_stats=False))
            self.add_module('inh', nn.InstanceNorm1d(1, eps=1e-5, affine=False, track_running_stats=False))
        if ingate:
            self.add_module('ig', nn.Linear(hidden_size, input_size, bias=True))

    flags = GRUCellEx.flags
    cell_params = GRUCellEx.cell_params

    def forward(self, input, hidden):
        if self.input_size != self.hidden_size:
            raise NotImplementedError("LSTMCellEx kernels need input_size == hidden_size "
                                      "(always true for graphnet.py:74)")
        h, c = hidden
        present = [q for q in self.cell_params() if q is not None]
        return _LSTMCellFunction.apply(input, h, c, self.flags(), *present)

    # ---- what the recurrent module needs to know about the cell (see _RecurrentECCFunction)
    N_GATES = 4

    @staticmethod
    def _new_state(R, N, H, dev):
        cs = torch.empty((R + 1, N, H), dtype=torch.float32, device=dev)
        cs[0].zero_()
        return cs

    @staticmethod
    def _new_dpre(R, N, H, dev):
        return None

    @staticmethod
    def _step_forward(inp, hs, cs, r, w, flags):
        ops.lstm_fwd(inp, hs[r], cs[r], *w, flags, out=hs[r + 1], out_c=cs[r + 1])

    @staticmethod
    def _step_backward(inps, hs, cs, r, gh, dc, w, flags, d_gi, d_gh, d_q, xp, dpre, ginp):
        """Cell backward of step r into ginp[r]; dc: dL/dc_{r+1} in, dL/dc_r out (c_R has no
        gradient: only the h states leave the module).  Returns dL/dh_r through the cell."""
        last = r == hs.shape[0] - 2
        return ops.lstm_bwd(inps[r], hs[r], cs[r], gh, None if last else dc, *w, flags, d_gi[r], d_gh[r],
                            d_q[r], xp[r], d_x=ginp[r], d_c=dc)[1]

    @staticmethod
    def _bias_grads(d_gi, d_gh, dpre, rows, H):
        return [ops.colsum(d_gi, 4 * H, rows, 4 * H), ops.colsum(d_gh, 4 * H, rows, 4 * H)]

    def __repr__(self):
        s = super(LSTMCellEx, self).__repr__() + '('
        if self._ingate:
            s += 'ingate'
        if self._layernorm:
            s += ' layernorm'
        return s + ')'


class _LSTMCellFunction(torch.autograd.Function):
    """Stand-alone cell (API parity); the recurrent module does not go through it."""

    @staticmethod
    def forward(ctx, x, h, c, flags, *present):
        x, h, c = x.contiguous(), h.contiguous(), c.contiguous()
        w = _unpack_cell(flags, present)
        hy, cy = ops.lstm_fwd(x, h, c, *w, flags)
        ctx.save_for_backward(x, h, c)
        ctx.flags, ctx.present = flags, present
        return hy, cy

    @staticmethod
    def backward(ctx, gy, gc):
        x, h, c = ctx.saved_tensors
        flags = ctx.flags
        n, H = h.shape
        dev = h.device
        w = _unpack_cell(flags, ctx.present)
        if gy is None:
            gy = torch.zeros_like(h)
        d_gi = torch.empty((n, 4 * H), device=dev)
        d_gh = torch.empty((n, 4 * H), device=dev)
        d_q = torch.empty((n, H), device=dev)
        xp = torch.empty((n, H), device=dev)
        d_x, d_h, d_c = ops.lstm_bwd(x, h, c, gy.contiguous(), None if gc is None else gc.contiguous(), *w,
                                     flags, d_gi, d_gh, d_q, xp)
        grads = _cell_weight_grads(LSTMCellEx, flags, d_gi, d_gh, d_q, xp, h, None, n, H)
        return (d_x, d_h, d_c, None) + tuple(grads)
