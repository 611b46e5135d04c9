"""Typed Python wrappers over the C-ABI (include/spg_b200.h).

Every function takes CUDA tensors, validates shape/dtype/contiguity on the host and enqueues
on torch's current stream.  CPU tensors are rejected: there is no CPU implementation in the
product (the CPU restatement lives in oracle/ and is test infrastructure only).
"""
import os
import weakref

import numpy as np
import torch

from . import _lib

F32, F64 = 0, 1
GRU_LAYERNORM, GRU_INGATE, GRU_BIAS = 1, 2, 4


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "superpoint_graph_b200 ops run on sm_90a CUDA tensors only (got a CPU tensor); "
                "there is no CPU fallback")


def _dt(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.float64:
        return F64
    raise TypeError("unsupported dtype %s" % t.dtype)


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


_workspaces = {}
_retired_workspaces = []  # outgrown buffers are never freed: a captured CUDA graph may hold their address


def workspace(nfloats, device, slot=0):
    """Per (device, stream, slot) scratch buffer; stream order makes reuse across calls safe.
    Slots keep buffers that are live in the SAME kernel apart (0: split-K / partial products,
    1: statistics partials).  A buffer that has to grow is replaced by one at least twice as large
    and the old one is kept alive for the life of the process (Trainer.capture bakes workspace
    addresses into CUDA graphs; geometric growth bounds the retired total by the final size)."""
    key = (device.index, _lib.current_stream(), slot)
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nfloats:
        grow = 0 if buf is None else 2 * buf.numel()
        if buf is not None:
            _retired_workspaces.append(buf)
        buf = torch.empty(max(int(nfloats), grow, 1 << 16), dtype=torch.float32, device=device)
        _workspaces[key] = buf
    return buf


def _workspace(query, device, *sizes):
    """uint8 scratch of the bytes that the C-ABI query `query` reports for `sizes` (torch's allocations are
    256-byte aligned, as the entry points require)."""
    nbytes = torch.zeros(1, dtype=torch.int64)
    _lib.call(query, *[int(n) for n in sizes], nbytes)
    return torch.empty(int(nbytes[0]), dtype=torch.uint8, device=device)


WEIGHTS_GENERATION = [0]


def weights_written():
    """Called by every wrapper that writes parameters or BatchNorm running statistics through a raw pointer
    (the optimizer kernels, the BatchNorm folds given running statistics).  Such writes bump no tensor version
    counter, so caches of values derived from the weights (the folded images of pointnet_fused_image) compare
    this generation instead."""
    WEIGHTS_GENERATION[0] += 1


def zero_(t):
    _need_cuda(t)
    assert t.is_contiguous()
    _lib.call("spg_zero", t, t.numel() * t.element_size(), _lib.current_stream())
    return t


# ------------------------------------------------------------------ graph structure
class EccGraph(object):
    """Device-side CSR views of one batched graph, shared by all ECC kernels.

    Derived from the reference's `(idxn, idxe, degs)` triple (ref: learning/ecc/GraphConvInfo.py:48-69):
    `tgt_rowptr` is the exclusive scan of the in-degrees, `edge_tgt` the target of every edge,
    `(src_rowptr, src_perm)` a stable source-sorted CSR used by the atomic-free grad_input kernel.
    CUDA inputs: `EccGraph.from_device` (spg_graph_build, on the device); host inputs: this constructor
    (numpy), which the CPU tests pin and the GPU tests compare the device builder with, bit for bit.
    """

    def __init__(self, idxn, idxe, degs, n_in=None):
        idxn_np = idxn.detach().cpu().numpy().astype(np.int64, copy=False)
        degs_np = degs.detach().cpu().numpy().astype(np.int64, copy=False)
        self.n_out = int(degs_np.shape[0])
        self.n_edges = int(idxn_np.shape[0])
        if int(degs_np.sum()) != self.n_edges:
            raise ValueError("sum(degs)=%d does not match the number of edges %d"
                             % (int(degs_np.sum()), self.n_edges))
        if n_in is None:
            n_in = max(self.n_out, int(idxn_np.max()) + 1 if self.n_edges else 0)
        self.n_in = int(n_in)
        if self.n_edges and (idxn_np.min() < 0 or idxn_np.max() >= self.n_in):
            raise ValueError("idxn out of range")
        host = build_csr_host(idxn_np, degs_np, self.n_in)
        self.host = host
        self.idxe_host = None if idxe is None else idxe.detach().cpu().numpy().astype(np.int32)
        self._dev = {}

    GRAPH_FIELDS = ("tgt_rowptr", "idxn", "edge_tgt", "src_rowptr", "src_perm")

    @classmethod
    def from_device(cls, idxn, degs, n_in=None, check=True, idxe=None):
        """Builds the views ON THE DEVICE from the reference's collated pair (int64 CUDA tensors, as
        GraphConvInfo.cuda() holds them, GraphConvInfo.py:71-77) — spg_graph_build: a scan, a stable radix
        sort and three small kernels instead of host numpy; bit-identical to the host builder.
        check=True reads the device status word back (one synchronisation) and raises like the host
        builder does; callers that validated the host arrays already pass check=False."""
        _need_cuda(idxn, degs)
        g = cls.__new__(cls)
        g.n_out, g.n_edges = int(degs.numel()), int(idxn.numel())
        g.n_in = int(n_in if n_in is not None else g.n_out)
        g.host, g.idxe_host = None, None
        dev = graph_build_alloc(g.n_out, g.n_in, g.n_edges, idxn.device)
        graph_build_into(dev, idxn, degs, g.n_in)
        if idxe is not None:
            dev["idxe"] = idxe.to(device=idxn.device, dtype=torch.int32)
        if check:
            st = int(dev["status"].item())
            if st:
                raise ValueError("graph build rejected the arrays (status %d: 1 = idxn out of range, "
                                 "2 = bad degree, 4 = sum(degs) != number of edges)" % st)
        g._dev = {(idxn.device.type, idxn.device.index): dev}
        return g

    def to(self, device):
        device = torch.device(device)
        key = (device.type, device.index)
        if key not in self._dev:
            if self.host is None:
                raise RuntimeError("this graph was built on %s; it has no host copy to move" % (list(self._dev),))
            d = {k: torch.from_numpy(v).to(device) for k, v in self.host.items()}
            d["idxe"] = None if self.idxe_host is None else torch.from_numpy(self.idxe_host).to(device)
            self._dev[key] = d
        return self._dev[key]


def graph_build_alloc(n_out, n_in, n_edges, device):
    """Output tensors + status word + workspace of spg_graph_build (static addresses: a captured CUDA graph
    reads them, HostBatch.copy_into rebuilds into them)."""
    i32 = dict(dtype=torch.int32, device=device)
    return {"tgt_rowptr": torch.empty(n_out + 1, **i32), "idxn": torch.empty(n_edges, **i32),
            "edge_tgt": torch.empty(n_edges, **i32), "src_rowptr": torch.empty(n_in + 1, **i32),
            "src_perm": torch.empty(n_edges, **i32), "idxe": None, "status": torch.zeros(1, **i32),
            "_ws": _workspace("spg_graph_build_workspace", device, n_out, n_in, n_edges)}


def graph_build_into(dev, idxn, degs, n_in):
    """Runs spg_graph_build on the current stream into the tensors of graph_build_alloc()."""
    _need_cuda(idxn, degs)
    assert idxn.dtype == torch.int64 and degs.dtype == torch.int64 and idxn.is_contiguous() and degs.is_contiguous()
    ws = dev["_ws"]
    _lib.call("spg_graph_build", idxn, degs, degs.numel(), int(n_in), idxn.numel(), dev["idxn"], dev["tgt_rowptr"],
              dev["edge_tgt"], dev["src_rowptr"], dev["src_perm"], dev["status"], ws, ws.numel(),
              _lib.current_stream())


def build_csr_host(idxn, degs, n_in):
    """Pure-numpy structure builder (also exercised by the CPU tests)."""
    n_edges = idxn.shape[0]
    tgt_rowptr = np.zeros(degs.shape[0] + 1, dtype=np.int64)
    np.cumsum(degs, out=tgt_rowptr[1:])
    edge_tgt = np.repeat(np.arange(degs.shape[0], dtype=np.int64), degs)
    src_perm = np.argsort(idxn, kind="stable")
    src_counts = np.bincount(idxn, minlength=n_in) if n_edges else np.zeros(n_in, dtype=np.int64)
    src_rowptr = np.zeros(n_in + 1, dtype=np.int64)
    np.cumsum(src_counts, out=src_rowptr[1:])
    if n_edges >= 2 ** 31 or n_in >= 2 ** 31:
        raise ValueError("graph too large for int32 indices")
    return {
        "tgt_rowptr": tgt_rowptr.astype(np.int32),
        "idxn": idxn.astype(np.int32),
        "edge_tgt": edge_tgt.astype(np.int32),
        "src_rowptr": src_rowptr.astype(np.int32),
        "src_perm": src_perm.astype(np.int32),
    }


# ------------------------------------------------------------------------------ ECC
def ecc_fwd(x, w, graph, c_out, out=None):
    _need_cuda(x, w)
    x, w = _c(x), _c(w)
    g = graph.to(x.device)
    is_mat = int(w.dim() == 3)
    c_in = x.shape[1]
    if x.shape[0] != graph.n_in:
        raise ValueError("input has %d rows, graph has %d nodes" % (x.shape[0], graph.n_in))
    n_w = g["idxe"].max().item() + 1 if g["idxe"] is not None else graph.n_edges
    if w.shape[0] < n_w:
        raise ValueError("weights has %d rows, graph needs %d" % (w.shape[0], n_w))
    if out is None:
        out = torch.empty((graph.n_out, c_out), dtype=x.dtype, device=x.device)
    _lib.call("spg_ecc_fwd", x, w, g["tgt_rowptr"], g["idxn"], g["idxe"], out, graph.n_out,
              graph.n_edges, c_in, c_out, is_mat, _dt(x), _lib.current_stream())
    return out


def ecc_bwd_w(xs, gs, graph, w_shape, n_iter=1, out=None, accumulate=False):
    """xs: [n_iter, n_in, c_in] (or [n_in, c_in]); gs: [n_iter, n_out, c_out]."""
    _need_cuda(xs, gs)
    xs, gs = _c(xs), _c(gs)
    g = graph.to(xs.device)
    is_mat = int(len(w_shape) == 3)
    c_in, c_out = xs.shape[-1], gs.shape[-1]
    if out is None:
        if g["idxe"] is not None:
            out = torch.zeros(w_shape, dtype=xs.dtype, device=xs.device)
        else:
            out = torch.empty(w_shape, dtype=xs.dtype, device=xs.device)
    x_stride = xs.shape[-2] * c_in if xs.dim() == 3 else 0
    g_stride = gs.shape[-2] * c_out if gs.dim() == 3 else 0
    _lib.call("spg_ecc_bwd_w", xs, gs, x_stride, g_stride, n_iter, g["tgt_rowptr"], g["idxn"],
              g["idxe"], g["edge_tgt"], out, graph.n_out, graph.n_edges, c_in, c_out, is_mat,
              int(accumulate), _dt(xs), _lib.current_stream())
    return out


def ecc_bwd_x(w, g_out, graph, c_in, add0=None, add1=None):
    _need_cuda(w, g_out, add0, add1)
    w, g_out = _c(w), _c(g_out)
    add0 = None if add0 is None else _c(add0)
    add1 = None if add1 is None else _c(add1)
    g = graph.to(w.device)
    is_mat = int(w.dim() == 3)
    c_out = g_out.shape[1]
    gx = torch.empty((graph.n_in, c_in), dtype=w.dtype, device=w.device)
    _lib.call("spg_ecc_bwd_x", w, g_out, g["tgt_rowptr"], g["src_rowptr"], g["src_perm"],
              g["edge_tgt"], g["idxe"], add0, add1, gx, graph.n_in, graph.n_edges, c_in, c_out,
              is_mat, _dt(w), _lib.current_stream())
    return gx


# -------------------------------------------------------------------------- ECC-CRF
CRF_MAX_C = 32  # widest class count the CRF kernels serve (filters [E, C, C])


def _crf_graph(graph, n, device):
    if graph.idxe_host is not None or graph.n_in != n or graph.n_out != n:
        raise ValueError("the CRF kernels need a square graph of %d nodes without idxe" % n)
    return graph.to(device)


def crf_softmax(x, g=None, out=None):
    """softmax(x) over rows, or (g given, x a softmax output) its backward x * (g - <g, x>)."""
    _need_cuda(x, g)
    x = _c(x)
    n, C = x.shape
    if out is None:
        out = torch.empty_like(x)
    _lib.call("spg_crf_softmax", x, None if g is None else _c(g), out, n, C, _lib.current_stream())
    return out


def crf_fwd_step(u, q_prev, w, graph, out, softmax):
    """out = softmax(Z) if softmax else Z, Z = u - ECC(q_prev, w) (matrix filters w [E, C, C])."""
    _need_cuda(u, q_prev, w, out)
    n, C = u.shape
    g = _crf_graph(graph, n, u.device)
    _lib.call("spg_crf_fwd_step", u, q_prev, w, g["tgt_rowptr"], g["idxn"], out, n, graph.n_edges, C,
              int(softmax), _lib.current_stream())
    return out


def crf_bwd_step(w, gp, q_prev, du_in, du_out, gp_out, graph):
    """From gp = dL/dP_r: du_out = du_in + dL/dZ_{r-1}; gp_out (if given) = dL/dP_{r-1} = -dL/dZ_{r-1}."""
    _need_cuda(w, gp, q_prev, du_in, du_out, gp_out)
    n, C = q_prev.shape
    g = _crf_graph(graph, n, w.device)
    _lib.call("spg_crf_bwd_step", w, gp, q_prev, du_in, du_out, gp_out, g["tgt_rowptr"], g["src_rowptr"],
              g["src_perm"], g["edge_tgt"], n, graph.n_edges, C, _lib.current_stream())
    return du_out


# ------------------------------------------------------------------------------ GRU
def gru_fwd(x, h, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, flags, out=None):
    _need_cuda(x, h, w_ih, w_hh)
    x, h = _c(x), _c(h)
    n, H = h.shape
    assert x.shape == h.shape and w_ih.shape == (3 * H, H) and w_hh.shape == (3 * H, H)
    if out is None:
        out = torch.empty_like(h)
    _lib.call("spg_gru_fwd", x, h, _c(w_ih), _c(w_hh), b_ih, b_hh,
              None if w_ig is None else _c(w_ig), b_ig, out, n, H, flags, _lib.current_stream())
    return out


def gru_bwd(x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, flags, d_gi, d_gh, d_q, xprime, dpre,
            d_x=None, d_h=None):
    _need_cuda(x, h, gy)
    x, h, gy = _c(x), _c(h), _c(gy)
    n, H = h.shape
    if d_x is None:
        d_x = torch.empty_like(h)
    if d_h is None:
        d_h = torch.empty_like(h)
    _lib.call("spg_gru_bwd", x, h, gy, _c(w_ih), _c(w_hh), b_ih, b_hh,
              None if w_ig is None else _c(w_ig), b_ig, d_x, d_h, d_gi, d_gh, d_q, xprime, dpre,
              n, H, flags, _lib.current_stream())
    return d_x, d_h


# ----------------------------------------------------------------------------- LSTM
def lstm_fwd(x, h, c, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, flags, out=None, out_c=None):
    """(hy, cy) of LSTMCellEx (ref: learning/modules.py:281-308); flags: the GRU_* bits."""
    _need_cuda(x, h, c, w_ih, w_hh)
    x, h, c = _c(x), _c(h), _c(c)
    n, H = h.shape
    assert x.shape == h.shape == c.shape and w_ih.shape == (4 * H, H) and w_hh.shape == (4 * H, H)
    if out is None:
        out = torch.empty_like(h)
    if out_c is None:
        out_c = torch.empty_like(h)
    _lib.call("spg_lstm_fwd", x, h, c, _c(w_ih), _c(w_hh), b_ih, b_hh,
              None if w_ig is None else _c(w_ig), b_ig, out, out_c, n, H, flags, _lib.current_stream())
    return out, out_c


def lstm_bwd(x, h, c, gy, gc, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, flags, d_gi, d_gh, d_q, xprime,
             d_x=None, d_h=None, d_c=None):
    """Returns (d_x, d_h, d_c); gc = dL/dcy or None (zero).  d_c may be gc itself."""
    _need_cuda(x, h, c, gy, gc)
    x, h, c, gy = _c(x), _c(h), _c(c), _c(gy)
    n, H = h.shape
    d_x = torch.empty_like(h) if d_x is None else d_x
    d_h = torch.empty_like(h) if d_h is None else d_h
    d_c = torch.empty_like(h) if d_c is None else d_c
    _lib.call("spg_lstm_bwd", x, h, c, gy, None if gc is None else _c(gc), _c(w_ih), _c(w_hh), b_ih, b_hh,
              None if w_ig is None else _c(w_ig), b_ig, d_x, d_h, d_c, d_gi, d_gh, d_q, xprime,
              n, H, flags, _lib.current_stream())
    return d_x, d_h, d_c


def rnn_vv_supported(weights, graph, n, H):
    """True when the fused recurrence kernels apply (vector filters, H == 32, no idxe, training-batch
    sizes); everything else runs the per-step kernels."""
    return (USE_FUSED_RNN[0] and weights.dim() == 2 and weights.dtype == torch.float32
            and graph.idxe_host is None and graph.n_in == n and graph.n_out == n
            and bool(_lib.lib().spg_rnn_vv_supported(n, H)))


def rnn_vv_fwd(hs, inps, weights, graph, cell, flags, cs=None):
    """hs [R+1,n,H] with hs[0] set, inps [R,n,H]; fills hs[1:], inps (ref: learning/modules.py:160-180).
    cs [R+1,n,H] with cs[0] set selects the LSTM cell (ref: :167-181) and fills cs[1:]; None: the GRU."""
    _need_cuda(hs, inps, weights, cs)
    R, n, H = inps.shape
    g = graph.to(hs.device)
    w_ih, w_hh, b_ih, b_hh, w_ig, b_ig = cell
    bar = torch.empty(4, dtype=torch.int32, device=hs.device)
    w = (_c(weights), g["tgt_rowptr"], g["idxn"], _c(w_ih), _c(w_hh), b_ih, b_hh,
         None if w_ig is None else _c(w_ig), b_ig, n, H, R, flags, bar, _lib.current_stream())
    if cs is None:
        _lib.call("spg_rnn_vv_fwd", hs, inps, *w)
    else:
        _lib.call("spg_rnn_vv_lstm_fwd", hs, cs, inps, *w)


def rnn_vv_bwd(hs, inps, weights, graph, cell, flags, gtop, gcat, ginp, d_gi, d_gh, d_q, xp, dpre, cs=None):
    """Backward of rnn_vv_fwd; returns the gradient w.r.t. hs[0].  With cs (the LSTM), dpre is unused."""
    _need_cuda(hs, inps, weights, gtop, cs)
    R, n, H = inps.shape
    g = graph.to(hs.device)
    w_ih, w_hh, b_ih, b_hh, w_ig, b_ig = cell
    bar = torch.empty(4, dtype=torch.int32, device=hs.device)
    dh = torch.empty((n, H), dtype=torch.float32, device=hs.device)
    gh0 = torch.empty((n, H), dtype=torch.float32, device=hs.device)
    head = (_c(weights), gtop, gcat, g["tgt_rowptr"], g["src_rowptr"], g["src_perm"], g["edge_tgt"],
            _c(w_ih), _c(w_hh), b_ih, b_hh, None if w_ig is None else _c(w_ig), b_ig, ginp, dh)
    tail = (n, H, R, flags, bar, _lib.current_stream())
    if cs is None:
        _lib.call("spg_rnn_vv_bwd", hs, inps, *head, gh0, d_gi, d_gh, d_q, xp, dpre, *tail)
    else:
        dc = torch.empty((n, H), dtype=torch.float32, device=hs.device)
        _lib.call("spg_rnn_vv_lstm_bwd", hs, cs, inps, *head, dc, gh0, d_gi, d_gh, d_q, xp, *tail)
    return gh0


# ---------------------------------------------------------------------------- dense
GEMM_TRACE = None  # set to [] to record (description, start, end) events of every SIMT gemm call
GEMM_FLOPS = [0]  # algorithmic FLOPs (2*M*N*K) issued through gemm(); read by bench.py


def _auto_split(M, N, K):
    tiles = ((M + 127) // 128) * ((N + 63) // 64)
    if tiles >= 132 or K < 256:
        return 1
    split = min((2 * 132 + tiles - 1) // tiles, max(1, K // 64))
    return max(1, split)


def _merge_stats(sws, tiles, N, M, dev, fold):
    """(mean, var) or, with fold=(gamma, beta, eps, rm, rv, nbt, momentum), (mean, var, scale, shift)."""
    mean = torch.empty(N, dtype=torch.float32, device=dev)
    var = torch.empty(N, dtype=torch.float32, device=dev)
    if fold is None:
        _lib.call("spg_colstats_merge", sws, tiles, N, mean, var, _lib.current_stream())
        return mean, var
    gamma, beta, eps, rm, rv, nbt, mom = fold
    if rm is not None:
        weights_written()
    scale = torch.empty(N, dtype=torch.float32, device=dev)
    shift = torch.empty(N, dtype=torch.float32, device=dev)
    _lib.call("spg_colstats_merge_fold", sws, tiles, N, mean, var, gamma, beta, float(eps), scale, shift,
              rm, rv, nbt, float(mom), int(M), _lib.current_stream())
    return mean, var, scale, shift


def gemm(A, lda, a_kmajor, B, ldb, b_kmajor, M, N, K, bias=None, out=None, ldc=None,
         a_aff=None, b_aff=None, split_k=None, stats=False, fold=None):
    """C[M,N] = opA(A) opB(B) + bias.  a_aff/b_aff = (scale|None, shift|None, relu)."""
    _need_cuda(A, B)
    dev = A.device
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=dev)
        ldc = N
    elif ldc is None:
        ldc = out.stride(0)
    a_s, a_t, a_r = a_aff if a_aff is not None else (None, None, False)
    b_s, b_t, b_r = b_aff if b_aff is not None else (None, None, False)
    GEMM_FLOPS[0] += 2 * M * N * K
    if GEMM_TRACE is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev0.record()
    if split_k is None:
        split_k = 1 if stats else _auto_split(M, N, K)
    ws = workspace(split_k * M * N, dev) if split_k > 1 else None
    tiles = (M + 127) // 128
    sws = workspace((tiles + tiles // 256 + 2) * N * 3, dev, slot=1) if stats else None
    _lib.call("spg_gemm", A, lda, int(a_kmajor), B, ldb, int(b_kmajor), bias, out, ldc, M, N, K,
              a_s, a_t, int(bool(a_r)), b_s, b_t, int(bool(b_r)), split_k, ws, sws,
              _lib.current_stream())
    if GEMM_TRACE is not None:
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        GEMM_TRACE.append(("M=%d N=%d K=%d a%d b%d split=%d" % (M, N, K, int(a_kmajor), int(b_kmajor), split_k),
                           ev0, ev1))
    if stats:
        return (out,) + _merge_stats(sws, tiles, N, M, dev, fold)
    return out


USE_TC = [os.environ.get("SPG_TC", "1") != "0"]  # tensor-core (wgmma) path for the large point-wise layers
USE_FUSED_RNN = [os.environ.get("SPG_FUSED_RNN", "1") != "0"]  # one-kernel R x {ECC, cell} loop
USE_FUSED_BNBWD = [os.environ.get("SPG_FUSED_BNBWD", "1") != "0"]  # BatchNorm backward inside the dX GEMM (prologue + epilogue sums)
USE_FUSED_EVAL = [os.environ.get("SPG_FUSED_EVAL", "1") != "0"]  # eval-mode PointNet trunk as one kernel per chain
def set_pdl(mode):
    """Programmatic dependent launch policy of the library (spg_set_pdl): 1 = every kernel is scheduled while
    its predecessor on the stream still runs and waits on the device for it (measured -1.5 ... -4.5 % on the
    single-stream inference workloads), 0 = plain stream order (the two-stream training schedule is 2 % faster
    that way: early-resident GEMM CTAs take SMs from the weight-gradient stream).  An explicit SPG_PDL in the
    environment wins."""
    if "SPG_PDL" not in os.environ:
        _lib.call("spg_set_pdl", int(mode))


USE_SIDE_STREAM = [os.environ.get("SPG_SIDE_STREAM", "1") != "0"]  # Trainer: block-local weight gradients on a 2nd stream


def tc_supported(M, N, K, lda=0, ldc=0):
    return (USE_TC[0] and M >= 512 and lda % 4 == 0 and ldc % 4 == 0
            and bool(_lib.lib().spg_tc_gemm_supported(int(M), int(N), int(K))))


PACK_CACHE = {}   # (W ptr, ldw, transpose, N, K, k_valid) -> image, valid until the weights change
_PACK_TABLES = {}  # tuple of job keys -> (device table, images, total)
PACK_LEARN = [None]  # dict owned by a Trainer: images packed on demand in its step, batched from the next step on


def prepack(jobs):
    """Packs the weight images of many layers with ONE launch and publishes them in PACK_CACHE.
    jobs: [(W, ldw, transpose, N, K, k_valid)].  The caller clears PACK_CACHE when the weights
    change (Trainer does after every backward)."""
    if not jobs:
        return
    keys = tuple((W.data_ptr(), int(ldw), int(bool(tr)), int(N), int(K), int(kv)) for W, ldw, tr, N, K, kv in jobs)
    ent = _PACK_TABLES.get(keys)
    dev = jobs[0][0].device
    if ent is None:
        rows, imgs, total = [], [], 0
        for (ptr, ldw, tr, N, K, kv) in keys:
            img = torch.empty(2 * N * K, dtype=torch.float32, device=dev)
            imgs.append(img)
            rows.append([ptr, ldw, tr, N, K, kv, img.data_ptr(), total])
            total += N * K
        table = torch.tensor(rows, dtype=torch.int64).to(dev)
        ent = _PACK_TABLES[keys] = (table, imgs, total)
    table, imgs, total = ent
    _lib.call("spg_tc_pack_weights_multi", table, len(keys), total, _lib.current_stream())
    for k, img in zip(keys, imgs):
        PACK_CACHE[k] = img


def _weight_image(W, ldw, transpose, N, K, kv, dev):
    key = (W.data_ptr(), int(ldw), int(bool(transpose)), int(N), int(K), int(kv))
    img = PACK_CACHE.get(key)
    if img is None:
        img = torch.empty(2 * N * K, dtype=torch.float32, device=dev)
        _lib.call("spg_tc_pack_weights", W, ldw, int(bool(transpose)), N, K, kv, img, _lib.current_stream())
        if PACK_LEARN[0] is not None:
            PACK_LEARN[0][key] = (W, int(ldw), bool(transpose), int(N), int(K), kv)
    return img


def tc_gemm(A, lda, W, ldw, transpose, M, N, K, bias=None, a_aff=None, stats=False, k_valid=None,
            fold=None, bnbwd=None, bnred=None):
    """C[M,N] = f(A)[M,K] B[N,K]^T + bias on the wgmma 3xTF32 kernel (spg_tc_gemm_ex).
    transpose=False: B = W ([N,K], ld ldw); True: B = W^T with W [K,N].

    stats / fold: batch statistics of C (and the BatchNorm fold) finished inside the kernel; returns
        (C, mean, var[, scale, shift]).
    bnbwd = (Y, ldy, scale, shift, relu, mean, var, s12, eps, want_dy): A is dL/d(activation) of a
        BatchNorm+ReLU layer whose raw output is Y; the prologue turns it into dL/dY on the fly.
        With want_dy the kernel also stores dL/dY [M,K] (for the weight-gradient kernel).
    bnred = (Y2, ldy2, scale2, shift2, mean2, var2, eps2, relu2): C is dL/d(activation) of the layer
        below; its BatchNorm-backward sums s1|s2 [2N] come out of the epilogue.
    Returns C, or a tuple (C, [mean, var, [scale, shift]], [dY], [s12]) in that order."""
    _need_cuda(A, W)
    dev = A.device
    kv = int(K if k_valid is None else k_valid)
    img = _weight_image(W, ldw, transpose, N, K, kv, dev)
    out = torch.empty((M, N), dtype=torch.float32, device=dev)
    a_s, a_t, a_r = a_aff if a_aff is not None else (None, None, False)
    a2 = a_mean = a_var = a_s12 = dy = None
    lda2 = lddy = 0
    a_eps = 0.0
    if bnbwd is not None:
        a2, lda2, a_s, a_t, a_r, a_mean, a_var, a_s12, a_eps, want_dy = bnbwd
        if want_dy:
            dy = torch.empty((M, K), dtype=torch.float32, device=dev)
            lddy = K
    epi, ws = 0, None
    mean = var = scale = shift = gamma = beta = rm = rv = nbt = None
    eps = mom = 0.0
    e = (None, 0, None, None, None, None, 0.0, False)
    s12 = None
    if stats:
        epi = 1
        mean = torch.empty(N, dtype=torch.float32, device=dev)
        var = torch.empty(N, dtype=torch.float32, device=dev)
        if fold is not None:
            gamma, beta, eps, rm, rv, nbt, mom = fold
            if rm is not None:
                weights_written()
            scale = torch.empty(N, dtype=torch.float32, device=dev)
            shift = torch.empty(N, dtype=torch.float32, device=dev)
    elif bnred is not None:
        epi = 2
        e = bnred
        s12 = torch.empty(2 * N, dtype=torch.float32, device=dev)
    if epi:
        ws = workspace(MAX_TC_PARTIALS[0] * N * 3, dev, slot=1)
    GEMM_FLOPS[0] += 2 * M * N * K
    TC_FLOPS[0] += 2 * M * N * K
    _lib.call("spg_tc_gemm_ex", A, lda, img, bias, out, N, M, N, K, a_s, a_t, int(bool(a_r)),
              a2, lda2, a_mean, a_var, a_s12, float(a_eps), dy, lddy, epi, ws,
              mean, var, gamma, beta, float(eps), scale, shift, rm, rv, nbt, float(mom),
              e[0], e[1], e[2], e[3], e[4], e[5], float(e[6]), int(bool(e[7])), s12,
              _lib.current_stream())
    res = [out]
    if stats:
        res += [mean, var] + ([scale, shift] if fold is not None else [])
    if dy is not None:
        res.append(dy)
    if s12 is not None:
        res.append(s12)
    return res[0] if len(res) == 1 else tuple(res)


MAX_TC_PARTIALS = [132]  # spg_tc_gemm_max_partials(): CTAs along the rows = partials per column

TC_FLOPS = [0]  # algorithmic FLOPs through tc_gemm (forward + data gradients)
DW_FLOPS = [0]  # algorithmic FLOPs through tc_dw (weight gradients)


def tc_dw_supported(M, co, ci, lddy, ldp):
    return (USE_TC[0] and M >= 2048 and lddy % 4 == 0 and ldp % 4 == 0
            and bool(_lib.lib().spg_tc_dw_supported(int(M), int(co), int(ci))))


def tc_dw(dY, lddy, P, ldp, M, co, ci, p_aff=None):
    """dW[co,ci] = dY^T [co,M] f(P)[M,ci] on the wgmma 3xTF32 kernel (ci may be the padded
    leading dimension of P; the caller slices the valid columns)."""
    _need_cuda(dY, P)
    dev = dY.device
    ctas = int(_lib.lib().spg_tc_dw_ctas(int(M)))
    ws = workspace(ctas * co * ci, dev)
    out = torch.empty((co, ci), dtype=torch.float32, device=dev)
    p_s, p_t, p_r = p_aff if p_aff is not None else (None, None, False)
    GEMM_FLOPS[0] += 2 * M * co * ci
    DW_FLOPS[0] += 2 * M * co * ci
    _lib.call("spg_tc_dw", dY, lddy, P, ldp, p_s, p_t, int(bool(p_r)), out, ws, M, co, ci,
              _lib.current_stream())
    return out


def _chunks(M):
    return max(1, (M + 255) // 256)


def bn_fold(mean, var, gamma, beta, eps, running_mean=None, running_var=None, momentum=0.1, M=0,
            num_batches_tracked=None):
    _need_cuda(mean, var)
    if running_mean is not None:
        weights_written()
    C = mean.numel()
    scale = torch.empty(C, dtype=torch.float32, device=mean.device)
    shift = torch.empty(C, dtype=torch.float32, device=mean.device)
    _lib.call("spg_bn_fold", mean, var, gamma, beta, float(eps), scale, shift, running_mean,
              running_var, num_batches_tracked, float(momentum), int(M), C, _lib.current_stream())
    return scale, shift


def _drop(drop):
    """drop = (p, slot) of a training-mode dropout, or None -> the (p, drop_slot) arguments of the C-ABI."""
    if drop is None:
        return 0.0, None
    _need_cuda(drop[1])
    return float(drop[0]), drop[1]


def affine_act(Y, ldy, M, C, scale=None, shift=None, relu=False, out=None, ldo=None, drop=None):
    """relu?(Y*scale+shift) -> [M, C]; with drop = (p, slot), dropout of that, mask from `slot`."""
    _need_cuda(Y)
    if out is None:
        out = torch.empty((M, C), dtype=torch.float32, device=Y.device)
        ldo = C
    _lib.call("spg_affine_act", Y, ldy, scale, shift, int(bool(relu)), out, ldo, M, C, *_drop(drop),
              _lib.current_stream())
    return out


def colsum(X, ldx, M, C):
    _need_cuda(X)
    out = torch.empty(C, dtype=torch.float32, device=X.device)
    ws = workspace(C * _chunks(M), X.device)
    _lib.call("spg_colsum", X, ldx, M, C, out, ws, _lib.current_stream())
    return out


def act_bwd_reduce(G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, M, C, drop=None):
    """-> s12 [2C]: s1 = s12[:C] (sum of the masked gradient), s2 = s12[C:] (same, weighted by xhat).
    With drop = (p, slot), the gradient is first turned into G*m/(1-p), m regenerated from `slot`."""
    _need_cuda(G, Y)
    s12 = torch.empty(2 * C, dtype=torch.float32, device=G.device)
    ws = workspace(2 * C * _chunks(M), G.device)
    _lib.call("spg_act_bwd_reduce", G, ldg, Y, ldy, scale, shift, mean, var, float(eps),
              int(bool(relu)), s12, ws, M, C, *_drop(drop), _lib.current_stream())
    return s12


def act_bwd_apply(G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, has_bn, s1, s2, M, C,
                  out=None, ldo=None, drop=None):
    """BatchNorm/ReLU backward -> dY [M, C]; drop as in act_bwd_reduce."""
    _need_cuda(G)
    if out is None:
        out = torch.empty((M, C), dtype=torch.float32, device=G.device)
        ldo = C
    _lib.call("spg_act_bwd_apply", G, ldg, Y, ldy, scale, shift, mean, var, float(eps),
              int(bool(relu)), int(bool(has_bn)), s1, s2, out, ldo, M, C, *_drop(drop),
              _lib.current_stream())
    return out


# -------------------------------------------------------------------------- dropout
_DROPOUT_RNG = {}  # device index -> int64[2] (seed, counter) on that device
DROPOUT_KEY_XOR = {}  # device index -> value folded into the key (data-parallel rank, see Trainer)


def _device(device):
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    return torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())


def dropout_rng_state(device=None, create=True):
    """The device's dropout generator state, an int64[2] (seed, counter) tensor that the kernels read and
    advance.  Created on first use with a seed drawn from torch's default generator (so torch.manual_seed
    makes runs reproducible) and counter 0; with create=False, None if it does not exist yet."""
    dev = _device(device)
    st = _DROPOUT_RNG.get(dev.index)
    if st is None and create:
        seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64))
        st = torch.tensor([seed, 0], dtype=torch.int64).to(dev)
        _DROPOUT_RNG[dev.index] = st
    return st


def _int64(v):
    v = int(v) & (2 ** 64 - 1)
    return v - 2 ** 64 if v >= 2 ** 63 else v


def dropout_manual_seed(seed, device=None):
    """Resets the device's dropout generator to (seed, counter 0)."""
    dev = _device(device)
    st = _DROPOUT_RNG.get(dev.index)
    if st is None:
        _DROPOUT_RNG[dev.index] = torch.tensor([_int64(seed), 0], dtype=torch.int64).to(dev)
    else:
        st[0].fill_(_int64(seed))
        st[1].zero_()


def dropout_slot(device):
    """Takes the next counter of the device's generator: returns a fresh int64[2] slot (seed ^ key fold,
    counter) in device memory, filled on the current stream (spg_dropout_rng_next)."""
    dev = _device(device)
    st = dropout_rng_state(dev)
    slot = torch.empty(2, dtype=torch.int64, device=dev)
    _lib.call("spg_dropout_rng_next", st, slot, _int64(DROPOUT_KEY_XOR.get(dev.index, 0)), _lib.current_stream())
    return slot


def dropout_fwd(Y, ldy, M, C, scale, shift, relu, p, slot):
    """dropout(relu?(Y*scale+shift)) -> [M, C], mask from `slot` (affine_act with drop=(p, slot))."""
    return affine_act(Y, ldy, M, C, scale, shift, relu, drop=(p, slot))


def dropout_mask(slot, p, M, C):
    """uint8 [M, C] keep mask of (slot = (seed, ctr), p)."""
    _need_cuda(slot)
    mask = torch.empty((M, C), dtype=torch.uint8, device=slot.device)
    _lib.call("spg_dropout_mask", _c(slot), float(p), M, C, mask, _lib.current_stream())
    return mask


# ------------------------------------------------------------------------- PointNet
def cloud_rows(clouds, T, ld, add_eye=False):
    _need_cuda(clouds, T)
    clouds = _c(clouds)
    B, F, L = clouds.shape
    rows = torch.empty((B * L, ld), dtype=torch.float32, device=clouds.device)
    _lib.call("spg_cloud_rows", clouds, None if T is None else _c(T), int(bool(add_eye)), rows, ld,
              B, F, L, _lib.current_stream())
    return rows


def rows_to_clouds(rows, ld, B, F, L):
    _need_cuda(rows)
    out = torch.empty((B, F, L), dtype=torch.float32, device=rows.device)
    _lib.call("spg_rows_to_clouds", rows, ld, out, B, F, L, _lib.current_stream())
    return out


def _seg_rows(seg):
    """Row count of a segment description seg = (B, L, offsets, row_seg): B segments of L rows if offsets
    is None, else CSR segments [offsets[b], offsets[b+1]) (int64 [B+1]) with row_seg the int32 segment of
    every row."""
    B, L, offsets, row_seg = seg
    if offsets is None:
        return B * L
    assert offsets.dtype == torch.int64 and offsets.is_contiguous() and row_seg.dtype == torch.int32
    return row_seg.numel()


def segmax_fwd(Y, ldy, seg, C, scale, shift, relu, pooled, ldp):
    """Max-pool of relu?(Y*scale+shift) over each segment of seg into pooled[:, :C]; returns the int32
    argmax within the segment (-1 for an empty segment, whose pooled value is 0)."""
    B, L, offsets, _ = seg
    _need_cuda(Y, pooled, offsets)
    assert offsets is None or (offsets.dtype == torch.int64 and offsets.is_contiguous())
    argmax = torch.empty((B, C), dtype=torch.int32, device=Y.device)
    _lib.call("spg_segmax_fwd", Y, ldy, scale, shift, int(bool(relu)), pooled, ldp, argmax, B, L, offsets, C,
              _lib.current_stream())
    return argmax


def segmax_bwd(g_pooled, ldg, argmax, seg, C):
    _need_cuda(g_pooled, argmax)
    B, L, offsets, row_seg = seg
    M = _seg_rows(seg)
    G = torch.empty((M, C), dtype=torch.float32, device=g_pooled.device)
    _lib.call("spg_segmax_bwd", g_pooled, ldg, argmax, G, C, B, L, offsets, row_seg, M, C, _lib.current_stream())
    return G


def segmax_bn_bwd(g_pooled, ldg, argmax, Y, ldy, scale, shift, mean, var, eps, relu, seg, C):
    """Fused max-pool backward + BatchNorm/ReLU backward; returns (s1, s2, dY[rows, C])."""
    _need_cuda(g_pooled, argmax, Y)
    dev = Y.device
    B, L, offsets, row_seg = seg
    M = _seg_rows(seg)
    s12 = torch.empty(2 * C, dtype=torch.float32, device=dev)
    dY = torch.empty((M, C), dtype=torch.float32, device=dev)
    ws = workspace(2 * C * ((B + 255) // 256), dev)
    _lib.call("spg_segmax_bn_bwd", g_pooled, ldg, argmax, Y, ldy, scale, shift, mean, var, float(eps),
              int(bool(relu)), s12, dY, C, ws, B, L, offsets, row_seg, M, C, _lib.current_stream())
    return s12[:C], s12[C:], dY


def row_segs(M):
    """The segment description of M rows that are each their own sample (an FC layer's rows)."""
    return (M, 1, None, None)


def group_norm_fwd(Y, ldy, seg, C, groups, gamma, beta, eps, relu, drop=None, out=None, ldo=None):
    """GroupNorm(groups, C) of Y [rows, C] over each segment of seg (as segmax_fwd), then ReLU if relu, then
    dropout with drop = (p, slot) (as affine_act).  Returns (out [rows, C], mean [B, groups, 2], rstd [B, groups]);
    the mean is a pair of floats (hi, lo) whose sum is the group's mean."""
    B, L, offsets, _ = seg
    _need_cuda(Y, gamma, beta, offsets)
    M = _seg_rows(seg)
    dev = Y.device
    if out is None:
        out = torch.empty((M, C), dtype=torch.float32, device=dev)
        ldo = C
    mean = torch.empty((B, groups, 2), dtype=torch.float32, device=dev)
    rstd = torch.empty((B, groups), dtype=torch.float32, device=dev)
    _lib.call("spg_group_norm_fwd", Y, ldy, _c(gamma), _c(beta), float(eps), int(bool(relu)), out, ldo, mean, rstd,
              B, L, offsets, C, groups, *_drop(drop), _lib.current_stream())
    return out, mean, rstd


def group_norm_bwd(G, ldg, Y, ldy, mean, rstd, gamma, beta, seg, C, groups, relu, drop=None):
    """Backward of group_norm_fwd from G = dL/d(out): returns (dY [rows, C], d_gamma [C], d_beta [C])."""
    B, L, offsets, _ = seg
    _need_cuda(G, Y, gamma, beta, offsets)
    M = _seg_rows(seg)
    dev = G.device
    dY = torch.empty((M, C), dtype=torch.float32, device=dev)
    dbg = torch.empty(2 * C, dtype=torch.float32, device=dev)
    ws = workspace(2 * C * int(_lib.lib().spg_group_norm_partials(int(B))), dev)
    _lib.call("spg_group_norm_bwd", G, ldg, Y, ldy, mean, rstd, _c(gamma), _c(beta), int(bool(relu)), dY, C, dbg,
              ws, B, L, offsets, C, groups, *_drop(drop), _lib.current_stream())
    return dY, dbg[C:], dbg[:C]


def stn_apply_bwd(clouds, dXrows, ld):
    _need_cuda(clouds, dXrows)
    clouds = _c(clouds)
    B, F, L = clouds.shape
    dT = torch.empty((B, 4), dtype=torch.float32, device=clouds.device)
    _lib.call("spg_stn_apply_bwd", clouds, dXrows, ld, dT, B, F, L, _lib.current_stream())
    return dT


def rows_scatter(src, idx, n_rows_out):
    _need_cuda(src, idx)
    src = _c(src)
    n, C = src.shape
    dst = torch.empty((n_rows_out, C), dtype=torch.float32, device=src.device)
    zero_(dst)
    _lib.call("spg_rows_scatter", src, idx, dst, n, C, _lib.current_stream())
    return dst


def rows_gather(src, idx):
    _need_cuda(src, idx)
    src = _c(src)
    n = idx.numel()
    C = src.shape[1]
    dst = torch.empty((n, C), dtype=torch.float32, device=src.device)
    _lib.call("spg_rows_gather", src, idx, dst, n, C, _lib.current_stream())
    return dst


# ----------------------------------------------------------------------------- step
def ce_loss(logits, target, class_weight=None, ignore_index=-100, need_grad=True):
    _need_cuda(logits, target, class_weight)
    logits = _c(logits)
    n, C = logits.shape
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    d_logits = torch.empty_like(logits) if need_grad else None
    ws = torch.empty(2, dtype=torch.float64, device=logits.device)
    _lib.call("spg_ce_loss", logits, _c(target), class_weight, int(ignore_index), loss, d_logits,
              ws, n, C, _lib.current_stream())
    return loss, d_logits


def clamp_adam_(param, grad, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-8,
                weight_decay=0.0, grad_clip=0.0, grad_scale=1.0):
    _need_cuda(param, grad, exp_avg, exp_avg_sq)
    weights_written()
    _lib.call("spg_clamp_adam", param, grad, exp_avg, exp_avg_sq, param.numel(), float(lr),
              float(beta1), float(beta2), float(eps), float(weight_decay), float(grad_clip),
              float(grad_scale), int(step), _lib.current_stream())


def clamp_adam_dev_(param, grad, exp_avg, exp_avg_sq, step_counter, lr, beta1=0.9, beta2=0.999,
                    eps=1e-8, weight_decay=0.0, grad_clip=0.0, grad_scale=1.0):
    """clamp + Adam with the step count in device memory (int64 scalar tensor, incremented here)."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq, step_counter)
    weights_written()
    _lib.call("spg_clamp_adam_dev", param, grad, exp_avg, exp_avg_sq, param.numel(), float(lr),
              float(beta1), float(beta2), float(eps), float(weight_decay), float(grad_clip),
              float(grad_scale), step_counter, _lib.current_stream())


class FusedAllreduce(object):
    """Symmetric-memory plumbing of spg_allreduce_clamp_adam: a two-half staging buffer and the flag words are
    allocated with torch.distributed._symmetric_memory (CUDA VMM handles exchanged through the process
    group's store) so that every rank holds device pointers to every peer's copy over NVLink.  `grad` — the
    flat gradient the step writes — is ordinary local memory; the kernel stages it itself."""

    def __init__(self, n, device, group):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.grad = torch.zeros(n, dtype=torch.float32, device=device)
        self.stage = symm_mem.empty(int(_lib.lib().spg_allreduce_stage_floats(int(n))), dtype=torch.float32,
                                    device=device)
        self.stage.zero_()
        words = int(_lib.lib().spg_allreduce_flag_words(self.world))
        self.flags = symm_mem.empty(words, dtype=torch.int32, device=device)
        self.flags.zero_()
        self._h_stage = symm_mem.rendezvous(self.stage, group)
        self._h_flags = symm_mem.rendezvous(self.flags, group)
        self.stage_ptrs = int(self._h_stage.buffer_ptrs_dev)
        self.flag_ptrs = int(self._h_flags.buffer_ptrs_dev)
        self.state = torch.zeros(2, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group=group)  # every rank's zero-fill has landed before anybody's first kernel

    def step_(self, param, exp_avg, exp_avg_sq, step_counter, lr, beta1=0.9, beta2=0.999, eps=1e-8,
              weight_decay=0.0, grad_clip=0.0):
        _need_cuda(param, exp_avg, exp_avg_sq, step_counter)
        weights_written()
        _lib.call("spg_allreduce_clamp_adam", self.grad, self.stage_ptrs, self.flag_ptrs, self.rank, self.world,
                  param, exp_avg, exp_avg_sq, param.numel(), float(lr), float(beta1), float(beta2), float(eps),
                  float(weight_decay), float(grad_clip), 1.0 / self.world, step_counter, self.state,
                  _lib.current_stream())


USE_FUSED_ALLREDUCE = [os.environ.get("SPG_FUSED_ALLREDUCE", "1") != "0"]


# ------------------------------------------------------------------------ profiling
def prof_enable(on):
    _lib.lib().spg_prof_enable(int(on))


def prof_reset():
    _lib.lib().spg_prof_reset()


def prof_collect():
    """Returns {kernel_name: (launches, total_ms)} for kernels launched since the last reset."""
    import ctypes

    L = _lib.lib()
    L.spg_prof_collect()
    out = {}
    for k in range(L.spg_prof_num_kernels()):
        n = ctypes.c_int64(0)
        ms = ctypes.c_double(0.0)
        L.spg_prof_kernel_stats(k, ctypes.byref(n), ctypes.byref(ms))
        if n.value:
            out[L.spg_prof_kernel_name(k).decode()] = (int(n.value), float(ms.value))
    return out


def total_launches():
    return int(_lib.lib().spg_prof_total_launches())


# ------------------------------------------------------------------ side stream (Trainer only)
class SideStream(object):
    """A second stream for work nobody waits for until the gradients are gathered: the filter-net
    and cell weight gradients of the recurrent ECC block are chains of small, latency-bound kernels
    that are independent of the (large) PointNet backward which follows them on the main stream.
    `fork()` orders the side stream after everything enqueued so far, `join()` orders the current
    stream after the side stream.  Tensors handed to fork() are kept alive until join(): the
    caching allocator would otherwise recycle main-stream blocks the side kernels still read.
    Only the Trainer installs one (SIDE[0]) — a caller who does not know about join() never forks."""

    def __init__(self, device):
        self.stream = torch.cuda.Stream(device=device)
        self.keep = []
        self.active = False

    def fork(self, *keep):
        self.stream.wait_stream(torch.cuda.current_stream())
        self.keep.append(keep)
        self.active = True
        return torch.cuda.stream(self.stream)

    def join(self):
        if self.active:
            torch.cuda.current_stream().wait_stream(self.stream)
            self.active = False
        self.keep = []


SIDE = [None]


# ------------------------------------------------------------- either side of the path
def cloud_build(points, sp_start, sp_count, sample_idx, columns, n_points, normalize, xform, jitter,
                jitter_sigma, jitter_clip, seed, clouds, diameters):
    """Resample / normalise / select / augment superpoints straight into the [Nv, F, L] PointNet
    input (ref: learning/spg.py:198-260); see include/spg_b200.h spg_cloud_build."""
    _need_cuda(points, sp_start, sp_count, sample_idx, columns, xform, jitter, clouds, diameters)
    assert points.dtype == torch.float32 and points.is_contiguous()
    assert sp_start.dtype == torch.int64 and sp_count.dtype == torch.int32 and columns.dtype == torch.int32
    assert sample_idx is None or (sample_idx.dtype == torch.int32 and sample_idx.is_contiguous())
    assert xform is None or (xform.dtype == torch.float64 and xform.is_contiguous())
    assert jitter is None or (jitter.dtype == torch.float32 and jitter.is_contiguous())
    nv, F, L = clouds.shape
    assert L == n_points and columns.numel() == F
    _lib.call("spg_cloud_build", points, points.shape[1], sp_start, sp_count, sample_idx, columns, F,
              L, int(bool(normalize)), xform, jitter, float(jitter_sigma), float(jitter_clip),
              int(seed), clouds, diameters, nv, _lib.current_stream())
    return clouds, diameters


def confusion_count(logits, label_mode, label_vec, confusion, counters, want_predictions=False):
    """confusion[:, argmax(logits_i)] += label_vec[i] for the labelled nodes (ref: learning/main.py:
    257-262, metrics.py:16-18); returns the predictions of all nodes if asked."""
    _need_cuda(logits, label_mode, label_vec, confusion, counters)
    logits = _c(logits)
    label_mode, label_vec = _c(label_mode), _c(label_vec)
    n, C = logits.shape
    assert logits.dtype == torch.float32 and label_mode.dtype == torch.int64
    assert label_vec.dtype == torch.int64 and label_vec.shape == (n, C)
    assert confusion.dtype == torch.int64 and confusion.shape == (C, C) and confusion.is_contiguous()
    pred = torch.empty(n, dtype=torch.int64, device=logits.device) if want_predictions else None
    _lib.call("spg_confusion_count", logits, C, label_mode, label_vec, C, confusion, counters, pred,
              n, C, _lib.current_stream())
    return pred


def labels_to_points(labels_red, comp_ptr, point_ids, n_ver):
    _need_cuda(labels_red, comp_ptr, point_ids)
    assert labels_red.dtype == torch.int64 and comp_ptr.dtype == torch.int64 and point_ids.dtype == torch.int64
    out = torch.empty(n_ver, dtype=torch.uint8, device=labels_red.device)
    _lib.call("spg_labels_to_points", _c(labels_red), _c(comp_ptr), _c(point_ids), comp_ptr.numel() - 1, out,
              n_ver, _lib.current_stream())
    return out


def nn1_interpolate(xyz_ref, xyz_query, labels_ref=None, want_index=False):
    """Exact 1-NN (float64 distances) of every query point among the reference points."""
    _need_cuda(xyz_ref, xyz_query, labels_ref)
    assert xyz_ref.dtype == torch.float32 and xyz_query.dtype == torch.float32
    assert xyz_ref.shape[1] == 3 and xyz_query.shape[1] == 3
    xyz_ref, xyz_query = _c(xyz_ref), _c(xyz_query)
    m = xyz_query.shape[0]
    lab = torch.empty(m, dtype=torch.int64, device=xyz_ref.device) if labels_ref is not None else None
    idx = torch.empty(m, dtype=torch.int32, device=xyz_ref.device) if (want_index or labels_ref is None) else None
    _lib.call("spg_nn1_interpolate", xyz_ref, xyz_ref.shape[0], xyz_query, m,
              None if labels_ref is None else _c(labels_ref), lab, idx, _lib.current_stream())
    return lab, idx


# ------------------------------------------------------------------ ragged (CSR) superpoints
def rows_xy_transform(rows, T, row_seg, add_eye=True):
    _need_cuda(rows, T, row_seg)
    assert rows.is_contiguous() and row_seg.dtype == torch.int32
    out = torch.empty_like(rows)
    _lib.call("spg_rows_xy_transform", rows, _c(T), int(bool(add_eye)), row_seg, out, rows.shape[0], rows.shape[1],
              _lib.current_stream())
    return out


def rows_xy_transform_bwd(rows, d_out, offsets):
    _need_cuda(rows, d_out, offsets)
    B = offsets.numel() - 1
    dT = torch.empty((B, 4), dtype=torch.float32, device=rows.device)
    d_out = _c(d_out)
    _lib.call("spg_rows_xy_transform_bwd", rows, rows.shape[1], d_out, d_out.shape[1], offsets, dT, B,
              _lib.current_stream())
    return dT


# ------------------------------------------------------------------ fused eval-mode PointNet trunk
def pointnet_fused_supported(F, L, widths):
    w = torch.tensor(list(widths), dtype=torch.int32)
    return USE_FUSED_EVAL[0] and bool(_lib.lib().spg_pointnet_fused_supported(int(F), int(L), len(widths), w.data_ptr()))


EVAL_BF16 = [False]  # eval-mode PointNet trunk in bf16 arithmetic (Trainer(dtype="bf16") sets it around eval_step)
_FUSED_IMAGES = {}  # (F, bf16, ids of the source tensors) -> _FusedImage
FUSED_RECORD = [None]  # a list while Trainer.capture_eval records the images its graph reads


def _fused_sources(layers):
    """The tensors a folded image is computed from: per layer W, bias, running mean and variance, gamma, beta
    (None where absent)."""
    out = []
    for W, b, bn in layers:
        out += [W, b] + ([bn.running_mean, bn.running_var, bn.weight, bn.bias] if bn is not None else [None] * 4)
    return out


class _FusedImage(object):
    """One folded chain: the weight image, the folded bias and the widths, plus what decides whether they still
    match their sources.  The sources are held by weak reference: an entry never keeps a model alive, and a new
    tensor that happens to get a freed one's id or address is not mistaken for it.  The stamp is the weights
    generation and every source's (address, version): torch's in-place operations bump the versions, the
    library's raw-pointer writers the generation.  A stale entry is refolded in place, so that a captured eval
    graph, which holds the image's and bias's addresses, reads the refreshed values."""

    def __init__(self, layers, F, bf16):
        self.F, self.bf16 = int(F), bool(bf16)
        self.refs = [None if t is None else weakref.ref(t) for t in _fused_sources(layers)]
        self.bn_refs = [None if bn is None else weakref.ref(bn) for _, _, bn in layers]
        self.shapes = [tuple(W.shape) for W, _, _ in layers]
        dev = layers[0][0].device
        L = _lib.lib()
        self.widths = torch.tensor([int(W.shape[0]) for W, _, _ in layers], dtype=torch.int32)
        if bf16:
            rows = int(L.spg_pointnet_fused_bf16_image_rows(self.F, len(layers), self.widths.data_ptr()))
            self.image = torch.empty(rows * 64, dtype=torch.bfloat16, device=dev)
        else:
            rows = int(L.spg_pointnet_fused_image_rows(self.F, len(layers), self.widths.data_ptr()))
            self.image = torch.empty(rows * 32, dtype=torch.float32, device=dev)
        self.bias = torch.empty(int(self.widths.sum()), dtype=torch.float32, device=dev)
        self._fold(layers)

    def same_sources(self, layers):
        srcs = _fused_sources(layers)
        return (len(srcs) == len(self.refs) and [tuple(W.shape) for W, _, _ in layers] == self.shapes
                and all((r is None and t is None) or (r is not None and r() is t) for r, t in zip(self.refs, srcs)))

    @staticmethod
    def _stamp(layers):
        return (WEIGHTS_GENERATION[0],) + tuple(None if t is None else (t.data_ptr(), t._version)
                                                for t in _fused_sources(layers))

    def refresh(self, layers=None):
        """Refolds in place if a source changed since the last fold; layers=None: the entry's own sources
        (nothing to do once they are gone)."""
        if layers is None:
            layers = []
            for i, bnr in enumerate(self.bn_refs):
                W, b = (None if r is None else r() for r in self.refs[6 * i:6 * i + 2])
                bn = None if bnr is None else bnr()
                if W is None or (self.refs[6 * i + 1] is not None and b is None) or (bnr is not None and bn is None):
                    return
                layers.append((W, b, bn))
            if not self.same_sources(layers):
                return
        if self._stamp(layers) != self.stamp:
            self._fold(layers)

    def _fold(self, layers):
        self.stamp = self._stamp(layers)
        image, bias, bf16 = self.image, self.bias, self.bf16
        kc = 64 if bf16 else 32
        row, boff, K = 0, 0, kc
        for W, b, bn in layers:
            N, kv = int(W.shape[0]), int(W.shape[1])
            scale = shift = None
            if bn is not None:
                scale, shift = bn_fold(bn.running_mean, bn.running_var, bn.weight, bn.bias, bn.eps)
            if bf16:
                _lib.call("spg_tc_pack_weights_bf16", W, W.stride(0), scale, N, K, kv, image[row * 64:],
                          _lib.current_stream())
                row += (K // 64) * N
            else:
                _lib.call("spg_tc_pack_weights_scaled", W, W.stride(0), scale, N, K, kv, image[row * 32:],
                          _lib.current_stream())
                row += (K // 32) * 2 * N
            bsl = bias[boff:boff + N]
            if b is not None:
                affine_act(b.detach().reshape(1, N), N, 1, N, scale, shift, False, out=bsl, ldo=N)
            elif shift is not None:
                bsl.copy_(shift)
            else:
                zero_(bsl)
            boff += N
            K = max(N, kc) if bf16 else N


def pointnet_fused_image(layers, F, bf16=False):
    """layers: [(W [N,K] or Conv1d weight [N,K,1], bias|None, bn_module|None)] of a Conv1d(k=1)+BatchNorm+ReLU
    chain in eval mode.  Returns (image, bias, widths): BatchNorm folded into weights and bias
    (scale = gamma/sqrt(rv+eps), bias' = bias*scale + beta - rm*scale), packed for spg_pointnet_fused_eval
    (fp32: tf32 hi|lo blocks of 32 floats) or spg_pointnet_fused_eval_bf16 (bf16 blocks of 64 elements).
    Cached per source tensors (see _FusedImage): pass the same tensor objects on every call (the module's
    parameters, not fresh views of them), and the image is refolded only when they have changed."""
    key = (int(F), bool(bf16)) + tuple(None if t is None else id(t) for t in _fused_sources(layers))
    ent = _FUSED_IMAGES.get(key)
    if ent is None or not ent.same_sources(layers):
        ent = _FusedImage(layers, F, bf16)
        if len(_FUSED_IMAGES) > 64:
            _FUSED_IMAGES.clear()
        _FUSED_IMAGES[key] = ent
    else:
        ent.refresh(layers)
    if FUSED_RECORD[0] is not None:
        FUSED_RECORD[0].append(ent)
    return ent.image, ent.bias, ent.widths


def pointnet_fused_eval(clouds, T, image, bias, widths, pooled, ldp):
    """pooled[b, :widths[-1]] = max over points of the folded conv chain on clouds[b] (xy transformed by T+I);
    the image's dtype selects the arithmetic (float32 image: 3xTF32, bfloat16 image: bf16)."""
    _need_cuda(clouds, image, bias, pooled, T)
    B, F, L = clouds.shape
    name = "spg_pointnet_fused_eval_bf16" if image.dtype == torch.bfloat16 else "spg_pointnet_fused_eval"
    _lib.call(name, clouds, B, F, L, None if T is None else _c(T), 1, image, bias,
              int(widths.numel()), widths.data_ptr(), pooled, ldp, _lib.current_stream())
    k = int(F)
    for n in widths.tolist():  # algorithmic FLOPs of the chain (valid K of the first layer, no padding)
        FUSED_FLOPS[0] += 2 * B * L * k * int(n)
        k = int(n)
    return pooled


FUSED_FLOPS = [0]  # algorithmic FLOPs through the fused eval trunk; read by bench.py


# ------------------------------------------------------------------ learned partition (csrc/partition.cu)
LP_DIST = {"euclidian": 0, "intrinsic": 1, "scalar": 2}
LP_INTRA = {"tv": 0, "laplacian": 1, "TVH": 2}
LP_INTER = {None: -1, "zhang": 0, "TVminus": 1}


def lp_incidence(src, tgt, n_ver):
    """Per-vertex CSR of the edge endpoints: (rowptr int32 [V+1], entry int32 [2E]); entry j < E is the source
    side of edge j, j >= E the target side of edge j - E."""
    _need_cuda(src, tgt)
    dev, E = src.device, src.numel()
    i32 = dict(dtype=torch.int32, device=dev)
    rowptr, entry = torch.empty(n_ver + 1, **i32), torch.empty(2 * E, **i32)
    ws = _workspace("spg_lp_workspace", dev, n_ver, E, 0)
    _lib.call("spg_lp_incidence", src, tgt, n_ver, E, rowptr, entry, ws, ws.numel(), _lib.current_stream())
    return rowptr, entry


def lp_dist_fwd(emb, src, tgt, dist_type):
    """(diff [E], coef [E] or None): compute_dist and the factor d diff / d <x_s, x_t> of its backward."""
    _need_cuda(emb, src, tgt)
    assert emb.dtype == torch.float32 and emb.dim() == 2 and emb.is_contiguous()
    assert src.dtype == torch.int64 and tgt.dtype == torch.int64
    E, dev = src.numel(), emb.device
    dt = LP_DIST[dist_type]
    diff = torch.empty(E, dtype=torch.float32, device=dev)
    coef = None if dt == 0 else torch.empty(E, dtype=torch.float32, device=dev)
    _lib.call("spg_lp_dist_fwd", emb, emb.shape[0], emb.shape[1], src, tgt, E, dt, diff, coef, _lib.current_stream())
    return diff, coef


def lp_dist_bwd(emb, src, tgt, dist_type, coef, gdiff, incidence):
    _need_cuda(emb, src, tgt, coef, gdiff)
    rowptr, entry = incidence
    gemb = torch.empty_like(emb)
    _lib.call("spg_lp_dist_bwd", emb, emb.shape[0], emb.shape[1], src, tgt, src.numel(), LP_DIST[dist_type], coef,
              _c(gdiff), rowptr, entry, gemb, _lib.current_stream())
    return gemb


def lp_loss_fwd(diff, weights, is_transition, intra, inter, dist_type):
    """float32 [2] = (loss1, loss2) of compute_loss; is_transition uint8."""
    _need_cuda(diff, weights, is_transition)
    assert diff.dtype == torch.float32 and weights.dtype == torch.float32 and is_transition.dtype == torch.uint8
    dev = diff.device
    part = torch.empty(2 * int(_lib.lib().spg_lp_loss_partials()), dtype=torch.float64, device=dev)
    loss = torch.empty(2, dtype=torch.float32, device=dev)
    _lib.call("spg_lp_loss_fwd", _c(diff), _c(weights), _c(is_transition), diff.numel(), LP_INTRA[intra],
              LP_INTER[inter], LP_DIST[dist_type], part, loss, _lib.current_stream())
    return loss


def lp_loss_bwd(diff, weights, is_transition, intra, inter, dist_type, gloss):
    _need_cuda(diff, weights, is_transition, gloss)
    gdiff = torch.empty_like(diff)
    _lib.call("spg_lp_loss_bwd", _c(diff), _c(weights), _c(is_transition), diff.numel(), LP_INTRA[intra],
              LP_INTER[inter], LP_DIST[dist_type], _c(gloss), gdiff, _lib.current_stream())
    return gdiff


def lp_xpart(src, tgt, is_transition, pred_in_component, n_ver, transition_factor):
    """crosspartition weights: (weights float32 [E], in_component_x int32 [V], comp_size int32 [V] (the first
    n_comp are used), n_comp int32 [1]), all on the device."""
    _need_cuda(src, tgt, is_transition, pred_in_component)
    dev, E = src.device, src.numel()
    i32 = dict(dtype=torch.int32, device=dev)
    w = torch.empty(E, dtype=torch.float32, device=dev)
    inx, size, ncomp = torch.empty(n_ver, **i32), torch.empty(n_ver, **i32), torch.empty(1, **i32)
    ws = _workspace("spg_lp_workspace", dev, n_ver, E, 0)
    _lib.call("spg_lp_xpart", src, tgt, is_transition, pred_in_component, n_ver, E, float(transition_factor), w, inx,
              size, ncomp, ws, ws.numel(), _lib.current_stream())
    return w, inx, size, ncomp


def lp_seal(src, tgt, is_transition, pred_in_component, objects, n_comp, transition_factor):
    """SEAL weights: (weights float32 [E], w_per_component int32 [n_comp])."""
    _need_cuda(src, tgt, is_transition, pred_in_component, objects)
    dev, E, V = src.device, src.numel(), pred_in_component.numel()
    w, wc = torch.empty(E, dtype=torch.float32, device=dev), torch.empty(n_comp, dtype=torch.int32, device=dev)
    ws = _workspace("spg_lp_workspace", dev, V, E, n_comp)
    _lib.call("spg_lp_seal", src, tgt, is_transition, pred_in_component, objects, V, E, n_comp,
              float(transition_factor), w, wc, ws, ws.numel(), _lib.current_stream())
    return w, wc


def lp_fill_weights(is_transition, w_other, w_transition):
    _need_cuda(is_transition)
    w = torch.empty(is_transition.numel(), dtype=torch.float32, device=is_transition.device)
    _lib.call("spg_lp_fill_weights", is_transition, is_transition.numel(), float(w_other), float(w_transition), w,
              _lib.current_stream())
    return w


def lp_count(truth, pred=None):
    """int64 [2] on the device: (#(truth and pred), #truth) of uint8 masks."""
    _need_cuda(truth, pred)
    counts = torch.empty(2, dtype=torch.int64, device=truth.device)
    _lib.call("spg_lp_count", _c(truth), None if pred is None else _c(pred), truth.numel(), counts,
              _lib.current_stream())
    return counts


def lp_edge_weight(diff, threshold):
    _need_cuda(diff)
    out = torch.empty(diff.numel(), dtype=torch.float64, device=diff.device)
    _lib.call("spg_lp_edge_weight", _c(diff), diff.numel(), float(threshold), out, _lib.current_stream())
    return out


def lp_relax(relaxed, src, tgt, n_ver, tolerance):
    """relax_edge_binary in place on the uint8 mask `relaxed`; returns the status word (1: numpy's IndexError)."""
    _need_cuda(relaxed, src, tgt)
    assert relaxed.dtype == torch.uint8 and relaxed.is_contiguous()
    dev = relaxed.device
    mark = torch.empty(max(n_ver, 1), dtype=torch.uint8, device=dev)
    hit, status = torch.empty(1, dtype=torch.int32, device=dev), torch.empty(1, dtype=torch.int32, device=dev)
    _lib.call("spg_lp_relax", relaxed, src, tgt, n_ver, relaxed.numel(), int(tolerance), mark, hit, status,
              _lib.current_stream())
    return status


def lp_perfect_prediction(comp_ptr, point_ids, labels, n_ver):
    """int64 [n_ver]: the first majority label of each point's component (labels int64 [V, 1 + C])."""
    _need_cuda(comp_ptr, point_ids, labels)
    assert labels.dtype == torch.int64 and labels.dim() == 2
    labels = _c(labels)
    pred = torch.empty(n_ver, dtype=torch.int64, device=labels.device)
    _lib.call("spg_lp_perfect_prediction", comp_ptr, point_ids, comp_ptr.numel() - 1, labels, labels.shape[1],
              labels.shape[1] - 1, n_ver, pred, _lib.current_stream())
    return pred


# ------------------------------------------------------------- learned-partition batch builder
LPL_GLOBAL_E, LPL_GLOBAL_RGB, LPL_GLOBAL_XYN, LPL_GLOBAL_XY = 1, 2, 4, 8


def lp_augment(xyz, rgb, rot, ref_index, noise_xyz, noise_rgb, device_noise, rgb_jitter, sigma, clip, seed,
               file_pos, xyz_out, rgb_out):
    """rgb / 255, rotation about the reference point and jitter of one file (ref: graph_processing.py:353,
    534-546); see include/spg_b200.h spg_lp_augment."""
    _need_cuda(xyz, rgb, rot, noise_xyz, noise_rgb, xyz_out, rgb_out)
    assert xyz.dtype == torch.float32 and rgb.dtype == torch.float32 and xyz.is_contiguous() and rgb.is_contiguous()
    assert rot is None or (rot.dtype == torch.float32 and rot.numel() == 9 and rot.is_contiguous())
    _lib.call("spg_lp_augment", xyz, rgb, xyz.shape[0], rot, int(ref_index), noise_xyz, noise_rgb,
              int(bool(device_noise)), int(bool(rgb_jitter)), float(sigma), float(clip), int(seed), int(file_pos),
              xyz_out, rgb_out, _lib.current_stream())


def lp_subgraph_select(mask, objects, src, tgt, new_index, selected, edge_pos, object_max):
    """Vertex / edge scans of a sub-graph mask and the object maximum (mask None: maximum only); see
    spg_lp_subgraph_select."""
    _need_cuda(mask, objects, src, tgt, new_index, selected, edge_pos, object_max)
    n, E = objects.numel(), src.numel()
    ws = None if mask is None else _workspace("spg_lp_subgraph_workspace", objects.device, n, E)
    _lib.call("spg_lp_subgraph_select", mask, objects, n, src, tgt, E, new_index, selected, edge_pos, object_max, ws,
              0 if ws is None else ws.numel(), _lib.current_stream())


def lp_subgraph_edges(src, tgt, is_transition, new_index, edge_pos, vertex_offset, src_out, tgt_out, tr_out):
    _need_cuda(src, tgt, is_transition, new_index, edge_pos, src_out, tgt_out, tr_out)
    _lib.call("spg_lp_subgraph_edges", src, tgt, is_transition, src.numel(), new_index, edge_pos, int(vertex_offset),
              src_out, tgt_out, tr_out, _lib.current_stream())


def lp_object_offsets(object_max, counts, offsets):
    _need_cuda(object_max, counts, offsets)
    assert counts.dtype == torch.int64 and offsets.dtype == torch.int64
    _lib.call("spg_lp_object_offsets", object_max, counts, counts.numel(), offsets, _lib.current_stream())


def lp_local_clouds(xyz, rgb, rgb_scale, local_geometry, k, selected, n_sel, elevation, xyn, labels, objects,
                    object_offset, use_rgb, global_flags, clouds, clouds_global, xyz_out, labels_out, objects_out):
    """Local clouds, global features and gathered rows of one file's kept vertices (ref: graph_processing.py:
    387-411,430); every output is that file's slice of the batch."""
    _need_cuda(xyz, rgb, local_geometry, selected, elevation, xyn, labels, objects, object_offset, clouds,
               clouds_global, xyz_out, labels_out, objects_out)
    assert local_geometry.dtype == torch.int32 and local_geometry.is_contiguous()
    assert clouds.dtype == torch.float32 and clouds.is_contiguous() and clouds_global.is_contiguous()
    _lib.call("spg_lp_local_clouds", xyz, rgb, int(bool(rgb_scale)), local_geometry, local_geometry.shape[1], int(k),
              selected, int(n_sel), elevation, xyn, labels, labels.shape[1], objects, object_offset,
              int(bool(use_rgb)), int(global_flags), clouds, clouds_global, clouds_global.shape[1], xyz_out,
              labels_out, objects_out, _lib.current_stream())


# ------------------------------------------------------------- k-NN graphs and geometric features
def knn_max_k():
    return int(_lib.lib().spg_knn_max_k())


def knn_bounds(xyz):
    """int32 [8] on the device: the order-preserving keys of the per-axis minimum (0-2) and maximum (3-5) of the
    finite coordinates, and the status word (6; 1: a non-finite coordinate); see spg_knn_bounds."""
    _need_cuda(xyz)
    assert xyz.dtype == torch.float32 and xyz.is_contiguous()
    words = torch.empty(8, dtype=torch.int32, device=xyz.device)
    _lib.call("spg_knn_bounds", xyz, xyz.shape[0], words, _lib.current_stream())
    return words


def knn_workspace(n, device):
    return _workspace("spg_knn_workspace", device, n)


def knn_grid(xyz, grid, ws):
    """Sorts the cloud into the cells of grid = (ox, oy, oz, cell, dim_x, dim_y, dim_z) inside `ws`; returns the
    number of occupied cells, int32 [1] on the device."""
    _need_cuda(xyz, ws)
    n_cells = torch.empty(1, dtype=torch.int32, device=xyz.device)
    ox, oy, oz, cell, dx, dy, dz = grid
    _lib.call("spg_knn_grid", xyz, xyz.shape[0], float(ox), float(oy), float(oz), float(cell), int(dx), int(dy),
              int(dz), ws, ws.numel(), n_cells, _lib.current_stream())
    return n_cells


def knn_query(n, k, k1, grid, ws, want_target2):
    """(source, target int64 [n k1], distances float32 [n k1], target2 int64 [n k] or None) from the sorted cloud
    that knn_grid left in `ws`."""
    _need_cuda(ws)
    dev = ws.device
    source = torch.empty(n * k1, dtype=torch.int64, device=dev)
    target = torch.empty(n * k1, dtype=torch.int64, device=dev)
    distances = torch.empty(n * k1, dtype=torch.float32, device=dev)
    target2 = torch.empty(n * k, dtype=torch.int64, device=dev) if want_target2 else None
    ox, oy, oz, cell, dx, dy, dz = grid
    _lib.call("spg_knn_query", int(n), int(k), int(k1), float(ox), float(oy), float(oz), float(cell), int(dx),
              int(dy), int(dz), ws, ws.numel(), source, target, distances, target2, _lib.current_stream())
    return source, target, distances, target2


def geof(xyz, target, k):
    """(geof float32 [n, 4], status int32 [1] on the device; 2: an id outside [0, n)); see spg_geof."""
    _need_cuda(xyz, target)
    assert xyz.dtype == torch.float32 and xyz.is_contiguous()
    assert target.dtype == torch.int64 and target.is_contiguous()
    n = xyz.shape[0]
    out = torch.empty((n, 4), dtype=torch.float32, device=xyz.device)
    status = torch.empty(1, dtype=torch.int32, device=xyz.device)
    _lib.call("spg_geof", xyz, n, target, int(k), out, status, _lib.current_stream())
    return out, status


# ------------------------------------------------------------- superpoint graph
def sp_scan(xyz, in_component):
    """int64 [2] on the device: max(in_component) + 1 and the status word (1: a non-finite coordinate, 4: a negative
    id); see spg_sp_scan."""
    _need_cuda(xyz, in_component)
    assert xyz.dtype == torch.float32 and xyz.is_contiguous()
    assert in_component.dtype == torch.int64 and in_component.is_contiguous()
    words = torch.empty(2, dtype=torch.int64, device=xyz.device)
    _lib.call("spg_sp_scan", xyz, in_component, xyz.shape[0], words, _lib.current_stream())
    return words


def sp_points(xyz, in_component, n_com, labels, label_mode, n_labels):
    """The superpoint features (centroids [n_com, 3], length, surface, volume [n_com, 1] float32, point_count
    [n_com, 1] int64, sp_labels [n_com, n_label_cols] int64 or None) and the status word (int32 [1]; 8: an empty
    component); see spg_sp_points.  labels: None, int64 [n] (label_mode 1) or int64 [n, L] (label_mode 2)."""
    _need_cuda(xyz, in_component, labels)
    assert in_component.dtype == torch.int64 and in_component.is_contiguous()
    dev, n = xyz.device, xyz.shape[0]
    ws = _workspace("spg_sp_points_workspace", dev, n)
    cols = 0
    if label_mode:
        assert labels.dtype == torch.int64 and labels.is_contiguous()
        cols = n_labels + 1 if label_mode == 1 else labels.shape[1]
    cen = torch.empty((n_com, 3), dtype=torch.float32, device=dev)
    f = [torch.empty((n_com, 1), dtype=torch.float32, device=dev) for _ in range(3)]
    count = torch.empty((n_com, 1), dtype=torch.int64, device=dev)
    sp_labels = torch.empty((n_com, cols), dtype=torch.int64, device=dev) if label_mode else None
    status = torch.empty(1, dtype=torch.int32, device=dev)
    _lib.call("spg_sp_points", xyz, in_component, int(n), int(n_com), labels, int(label_mode), int(cols),
              int(n_labels), ws, ws.numel(), cen, f[0], f[1], f[2], count, sp_labels, status, _lib.current_stream())
    return (cen, f[0], f[1], f[2], count, sp_labels), status


def sp_edges_count(in_component, simplices):
    """(tet_offsets int32 [T + 1], status int32 [1]; 2: an id outside [0, n)) on the device for simplices int32 or
    int64 [T, 4]; tet_offsets[T] is the number of candidate pairs.  See spg_sp_edges_count."""
    _need_cuda(in_component, simplices)
    assert simplices.dtype in (torch.int32, torch.int64) and simplices.is_contiguous()
    dev, t = in_component.device, simplices.shape[0]
    ws = _workspace("spg_sp_edges_workspace", dev, t, 0)
    offsets = torch.empty(t + 1, dtype=torch.int32, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    _lib.call("spg_sp_edges_count", in_component, in_component.shape[0], simplices,
              int(simplices.dtype == torch.int64), int(t), offsets, ws, ws.numel(), status, _lib.current_stream())
    return offsets, status


def sp_edges_build(xyz, in_component, simplices, offsets, n_cand, d_max):
    """(workspace, n_sedg int64 [1] on the device): the superedges' pairs grouped by component key; see
    spg_sp_edges_build."""
    _need_cuda(xyz, in_component, simplices, offsets)
    dev, t = xyz.device, simplices.shape[0]
    ws = _workspace("spg_sp_edges_workspace", dev, t, n_cand)
    n_sedg = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.call("spg_sp_edges_build", xyz, in_component, xyz.shape[0], simplices, int(simplices.dtype == torch.int64),
              int(t), offsets, int(n_cand), float(d_max), ws, ws.numel(), n_sedg, _lib.current_stream())
    return ws, n_sedg


def sp_edges_features(xyz, n_tets, n_cand, ws, n_sedg, sp):
    """dict of source, target [n_sedg, 1] (int64) and the se_* features (float32); see spg_sp_edges_features.
    sp = (centroids, length, surface, volume, point_count) from sp_points."""
    _need_cuda(xyz, ws, *sp)
    dev = xyz.device
    src = torch.empty((n_sedg, 1), dtype=torch.int64, device=dev)
    tgt = torch.empty((n_sedg, 1), dtype=torch.int64, device=dev)
    f3 = {k: torch.empty((n_sedg, 3), dtype=torch.float32, device=dev)
          for k in ("se_delta_mean", "se_delta_std", "se_delta_centroid")}
    f1 = {k: torch.empty((n_sedg, 1), dtype=torch.float32, device=dev)
          for k in ("se_delta_norm", "se_length_ratio", "se_surface_ratio", "se_volume_ratio", "se_point_count_ratio")}
    _lib.call("spg_sp_edges_features", xyz, int(n_tets), int(n_cand), ws, ws.numel(), int(n_sedg), *sp, src, tgt,
              f3["se_delta_mean"], f3["se_delta_std"], f1["se_delta_norm"], f3["se_delta_centroid"],
              f1["se_length_ratio"], f1["se_surface_ratio"], f1["se_volume_ratio"], f1["se_point_count_ratio"],
              _lib.current_stream())
    out = {"source": src, "target": tgt}
    out.update(f3)
    out.update(f1)
    return out


# ------------------------------------------------------------- voxel pruning
def prune_workspace(n, chunk_rows, device):
    return _workspace("spg_prune_workspace", device, n, chunk_rows)


def prune_bounds(xyz, chunk_rows, voxel_size, labels, n_labels, objects, n_objects, ws):
    """int64 [4] on the device: the status word (1: a non-finite coordinate, 2: a bin >= 2^32, 4: a label outside
    [0, n_labels], 8: an object outside [0, n_objects]) and the largest bin of x, y, z; see spg_prune_bounds."""
    _need_cuda(xyz, labels, objects, ws)
    assert xyz.dtype == torch.float32 and xyz.is_contiguous()
    for t in (labels, objects):
        assert t is None or (t.dtype == torch.int64 and t.is_contiguous())
    words = torch.empty(4, dtype=torch.int64, device=xyz.device)
    _lib.call("spg_prune_bounds", xyz, xyz.shape[0], int(chunk_rows), float(voxel_size), labels, int(n_labels),
              objects, int(n_objects), ws, ws.numel(), words, _lib.current_stream())
    return words


def prune_voxels(xyz, chunk_rows, voxel_size, max_bins, ws):
    """int64 [1] on the device: the number of voxels; the sorted points and the voxels' runs stay in `ws`.  See
    spg_prune_voxels."""
    _need_cuda(xyz, ws)
    n_voxels = torch.empty(1, dtype=torch.int64, device=xyz.device)
    _lib.call("spg_prune_voxels", xyz, xyz.shape[0], int(chunk_rows), float(voxel_size), int(max_bins[0]),
              int(max_bins[1]), int(max_bins[2]), ws, ws.numel(), n_voxels, _lib.current_stream())
    return n_voxels


def prune_reduce(xyz, rgb, labels, n_labels, objects, n_objects, chunk_rows, ws, m):
    """(xyz [m, 3] float32, rgb [m, 3] uint8, labels [m, n_labels + 1] int64, objects [m, n_objects + 1] int64) of
    the m voxels that prune_voxels left in `ws`; see spg_prune_reduce."""
    _need_cuda(xyz, rgb, labels, objects, ws)
    assert rgb.dtype == torch.uint8 and rgb.is_contiguous()
    dev = xyz.device
    xyz_out = torch.empty((m, 3), dtype=torch.float32, device=dev)
    rgb_out = torch.empty((m, 3), dtype=torch.uint8, device=dev)
    labels_out = torch.empty((m, n_labels + 1), dtype=torch.int64, device=dev)
    objects_out = torch.empty((m, n_objects + 1), dtype=torch.int64, device=dev)
    _lib.call("spg_prune_reduce", xyz, rgb, labels, int(n_labels), objects, int(n_objects), xyz.shape[0],
              int(chunk_rows), ws, ws.numel(), int(m), xyz_out, rgb_out, labels_out, objects_out,
              _lib.current_stream())
    return xyz_out, rgb_out, labels_out, objects_out


# ------------------------------------------------------------- Delaunay triangulation (csrc/delaunay.cu)
class DelaunayStore(object):
    """The workspace of one device triangulation: n points, a store of `cap` tetrahedra; see spg_dt_*."""

    def __init__(self, n, cap, device):
        self.n, self.cap, self.device = int(n), int(cap), device
        self.ws = _workspace("spg_dt_workspace", device, self.n, self.cap)
        self.out = torch.zeros(8, dtype=torch.int64)

    def _call(self, name, *args):
        _lib.call(name, self.n, self.cap, self.ws, self.ws.numel(), *args, _lib.current_stream())

    def setup(self, xyz):
        """(status, unique points); status 1: a non-finite coordinate."""
        _need_cuda(xyz)
        assert xyz.dtype == torch.float32 and xyz.is_contiguous() and xyz.shape == (self.n, 3)
        _lib.call("spg_dt_setup", xyz, self.n, self.cap, self.ws, self.ws.numel(), self.out, _lib.current_stream())
        return int(self.out[0]), int(self.out[1])

    def init(self):
        """status: 2 fewer than 4 affinely independent points, 4 a walk that did not end."""
        self._call("spg_dt_init", self.out)
        return int(self.out[0])

    def cavities(self, big_point=-1):
        """(nominees, winners, new tetrahedra, overflowing nominees, smallest overflowing, free slots, top,
        largest cavity)."""
        self._call("spg_dt_cavities", int(big_point), self.out)
        return tuple(int(v) for v in self.out)

    def commit(self):
        """(short of slots, status): nothing is written when the store is short."""
        self._call("spg_dt_commit", self.out)
        return int(self.out[0]), int(self.out[1])

    def grow(self, cap):
        """Moves the state into a workspace for `cap` tetrahedra."""
        nbytes = torch.zeros(1, dtype=torch.int64)
        _lib.call("spg_dt_workspace", self.n, int(cap), nbytes)
        ws = torch.empty(int(nbytes[0]), dtype=torch.uint8, device=self.device)
        self._call("spg_dt_grow", int(cap), ws, ws.numel())
        self.ws, self.cap = ws, int(cap)

    def output(self):
        """int32 [T, 4] on the device: the finite tetrahedra, canonical (consumes the adjacency)."""
        count = torch.zeros(1, dtype=torch.int64)
        self._call("spg_dt_output", count, None)
        simplices = torch.empty((int(count[0]), 4), dtype=torch.int32, device=self.device)
        if simplices.shape[0]:
            self._call("spg_dt_output", count, simplices)
        return simplices


# ------------------------------------------------------------- learned partition's structure (csrc/structure.cu)
def _status(dev):
    return torch.empty(1, dtype=torch.int32, device=dev)


def st_vor_count(xyz, simplices, voronoi):
    """(block_counts int64 [blocks + 1], status int32 [1]; 2: an id outside [0, n)) on the device;
    block_counts[-1] is the number of kept candidates.  voronoi: the float32 threshold.  See spg_st_vor_count."""
    _need_cuda(xyz, simplices)
    assert simplices.dtype in (torch.int32, torch.int64) and simplices.is_contiguous()
    dev, t = xyz.device, simplices.shape[0]
    counts = torch.empty(int(_lib.lib().spg_st_vor_blocks(int(t))) + 1, dtype=torch.int64, device=dev)
    status = _status(dev)
    _lib.call("spg_st_vor_count", xyz, xyz.shape[0], simplices, int(simplices.dtype == torch.int64), int(t),
              float(voronoi), counts, status, _lib.current_stream())
    return counts, status


def st_vor_build(xyz, simplices, voronoi, counts, knn_target, k1, n_kept):
    """(distances float32 [n_kept], source, target int64 [n_kept + n k1], n_edges int64 [1], status int32 [1]) on
    the device: the first n_edges of source / target are the deduplicated union.  See spg_st_vor_build."""
    _need_cuda(xyz, simplices, counts, knn_target)
    assert knn_target.dtype == torch.int64 and knn_target.is_contiguous()
    dev, n, t = xyz.device, xyz.shape[0], simplices.shape[0]
    ws = _workspace("spg_st_vor_workspace", dev, n, t, n * k1, n_kept)
    distances = torch.empty(n_kept, dtype=torch.float32, device=dev)
    source = torch.empty(n_kept + n * k1, dtype=torch.int64, device=dev)
    target = torch.empty(n_kept + n * k1, dtype=torch.int64, device=dev)
    n_edges = torch.empty(1, dtype=torch.int64, device=dev)
    status = _status(dev)
    _lib.call("spg_st_vor_build", xyz, n, simplices, int(simplices.dtype == torch.int64), int(t), float(voronoi),
              counts, knn_target, int(k1), int(n_kept), ws, ws.numel(), distances, source, target, n_edges, status,
              _lib.current_stream())
    return distances, source, target, n_edges, status


def st_cc(src, tgt, active, n_ver):
    """(in_component, offsets [n_ver + 1], members, n_comp [1], all int64, status int32 [1]) on the device; see
    spg_st_cc.  active: uint8 [E], an edge is active where the byte read as a signed char is > 0."""
    _need_cuda(src, tgt, active)
    assert src.dtype == tgt.dtype == torch.int64 and active.dtype == torch.uint8
    dev = src.device
    ws = _workspace("spg_st_cc_workspace", dev, n_ver)
    in_comp = torch.empty(n_ver, dtype=torch.int64, device=dev)
    offsets = torch.empty(n_ver + 1, dtype=torch.int64, device=dev)
    members = torch.empty(n_ver, dtype=torch.int64, device=dev)
    n_comp = torch.empty(1, dtype=torch.int64, device=dev)
    status = _status(dev)
    _lib.call("spg_st_cc", src, tgt, active, int(n_ver), src.shape[0], ws, ws.numel(), in_comp, offsets, members,
              n_comp, status, _lib.current_stream())
    return in_comp, offsets, members, n_comp, status


def st_argmax(a, col0, add, zero_empty=False, want_weight=False):
    """(out int64 [n], weight float32 [n] or None): add + the first argmax of a[:, col0:]; see spg_st_argmax."""
    _need_cuda(a)
    assert a.dtype == torch.int64 and a.dim() == 2 and a.is_contiguous()
    n, cols = a.shape
    out = torch.empty(n, dtype=torch.int64, device=a.device)
    weight = torch.empty(n, dtype=torch.float32, device=a.device) if want_weight else None
    _lib.call("spg_st_argmax", a, int(n), int(cols), int(col0), int(add), int(bool(zero_empty)), out, weight,
              _lib.current_stream())
    return out, weight


ST_DIFFERENT, ST_INPAINT, ST_EQUAL = 0, 1, 2


def st_transitions(lab, src, tgt, mode):
    """(uint8 [E], status int32 [1]; 2: an id outside [0, n)): mode ST_DIFFERENT lab[s] != lab[t], ST_INPAINT
    graph_processing.py:155-156, ST_EQUAL lab[s] == lab[t]; see spg_st_transitions."""
    _need_cuda(lab, src, tgt)
    assert lab.dtype == src.dtype == tgt.dtype == torch.int64
    out = torch.empty(src.shape[0], dtype=torch.uint8, device=src.device)
    status = _status(src.device)
    _lib.call("spg_st_transitions", lab, lab.shape[0], src, tgt, src.shape[0], int(mode), out, status,
              _lib.current_stream())
    return out, status


def st_select(flags, want):
    """(index int64 [n], count int64 [1]) on the device: the first count entries of index are the ascending i with
    (flags[i] != 0) == want; see spg_st_select."""
    _need_cuda(flags)
    assert flags.dtype == torch.uint8 and flags.is_contiguous()
    dev, n = flags.device, flags.shape[0]
    ws = _workspace("spg_st_select_workspace", dev, n)
    index = torch.empty(n, dtype=torch.int64, device=dev)
    count = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.call("spg_st_select", flags, int(n), int(bool(want)), ws, ws.numel(), index, count, _lib.current_stream())
    return index, count


def st_gather_rows(src, index, m):
    """(src[index[:m]], status int32 [1]) on the device: whole rows of a contiguous tensor."""
    _need_cuda(src, index)
    assert src.is_contiguous() and index.dtype == torch.int64
    out = torch.empty((m,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    status = _status(src.device)
    row_bytes = src[0].numel() * src.element_size() if src.shape[0] else 1
    _lib.call("spg_st_gather_rows", src, src.shape[0], int(row_bytes), index, int(m), out, status,
              _lib.current_stream())
    return out, status


def st_points(xyz, bounds, plane=None, elevation=None, xyn=None, low=None, geof=None):
    """Fills the given outputs (elevation float32 [n], xyn float32 [n, 2], low uint8 [n], geof float32 [n, 4]:
    column 3 doubled in place); plane = (c0, c1, b) or None.  bounds: knn_bounds(xyz).  See spg_st_points."""
    _need_cuda(xyz, bounds)
    c0, c1, b = (0.0, 0.0, 0.0) if plane is None else plane
    _lib.call("spg_st_points", xyz, xyz.shape[0], bounds, int(plane is not None), float(c0), float(c1), float(b),
              elevation, xyn, low, geof, _lib.current_stream())


# ------------------------------------------------------------- superpoint graph batch builder

def batch_select(src, tgt, adjacency, sizes, perm, centres, order, minpts, cut, out=None):
    """Sub-graph selection of one resident graph (see spg_batch_select).  adjacency: the spg_graph_build views
    (EccGraph.to(device)) of its target-sorted edges.  Returns (new_index int32 [n], edge_pos int32 [E + 1],
    out int32 [2 + n] = kept vertices, kept edges, kept original ids); `out` may be given (a contiguous int32
    [2 + n] slice of a larger buffer)."""
    _need_cuda(src, tgt, sizes, perm, centres, out)
    n, E = sizes.numel(), src.numel()
    i32 = dict(dtype=torch.int32, device=sizes.device)
    new_index, edge_pos = torch.empty(n, **i32), torch.empty(E + 1, **i32)
    if out is None:
        out = torch.empty(2 + n, **i32)
    assert out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 + n
    ws = _workspace("spg_batch_select_workspace", sizes.device, n, E)
    _lib.call("spg_batch_select", src, tgt, n, E, adjacency["tgt_rowptr"], adjacency["idxn"],
              adjacency["src_rowptr"], adjacency["src_perm"], adjacency["edge_tgt"], sizes, perm, centres,
              0 if centres is None else centres.numel(), int(order), int(minpts), int(cut), new_index, edge_pos, out,
              ws, ws.numel(), _lib.current_stream())
    return new_index, edge_pos, out


def batch_edges(src, tgt, new_index, edge_pos, kept, n_kept, n_kept_edges, vertex_offset, edge_feats, targets,
                idxn_out, tgt_out, degs_out, feats_out, targets_out):
    """One graph's slice of the collated batch (see spg_batch_edges); every output is that slice."""
    _need_cuda(src, tgt, new_index, edge_pos, kept, edge_feats, targets, idxn_out, tgt_out, degs_out, feats_out,
               targets_out)
    assert edge_feats.dtype == torch.float32 and targets.dtype == torch.int64
    ws = _workspace("spg_batch_edges_workspace", src.device, n_kept, n_kept_edges)
    _lib.call("spg_batch_edges", src, tgt, src.numel(), new_index, edge_pos, kept, int(n_kept), int(n_kept_edges),
              int(vertex_offset), edge_feats, edge_feats.shape[1], targets, targets.shape[1], idxn_out, tgt_out,
              degs_out, feats_out, targets_out, ws, ws.numel(), _lib.current_stream())


def _seed64(seed):
    """A seed as the int64 with the same 64 bits (the C-ABI takes the key as int64_t)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s - (1 << 64) if s >= (1 << 63) else s


def batch_draw(n, seed, graph_pos, permute, n_centres, device):
    """(perm int32 [n] or None, centres int32 [n_centres] or None) on the device: the graph draws of position
    `graph_pos` of a batch under `seed` (see spg_batch_draw)."""
    i32 = dict(dtype=torch.int32, device=device)
    perm = torch.empty(n, **i32) if permute else None
    centres = torch.empty(n_centres, **i32) if n_centres > 0 else None
    if perm is None and centres is None:
        return None, None
    ws = _workspace("spg_batch_draw_workspace", device, n)
    _lib.call("spg_batch_draw", int(n), _seed64(seed), int(graph_pos), int(bool(permute)), int(n_centres), perm,
              centres, ws, ws.numel(), _lib.current_stream())
    return perm, centres


def batch_cloud_flags(selected, graph_pos, sp_index, minpts, flags, valid, first_row, count, key):
    """One graph's slice of the batch's cloud table from batch_select's `selected` (see spg_batch_cloud_flags);
    sp_index = (first row int64 [ids], count int32 [ids]) of the file in the superpoint store, or None."""
    _need_cuda(selected, flags, valid, first_row, count, key)
    rows, counts = sp_index if sp_index is not None else (None, None)
    n_ids = 0 if counts is None else counts.numel()
    _lib.call("spg_batch_cloud_flags", selected, flags.numel(), int(graph_pos), rows, counts, int(n_ids), int(minpts),
              flags, valid, first_row, count, key, _lib.current_stream())


def batch_clouds(valid, first_row, count, key):
    """(start int64 [n], count int32 [n], key int64 [n]) whose first sum(valid) entries are the valid positions'
    values in order (see spg_batch_clouds)."""
    _need_cuda(valid, first_row, count, key)
    n, dev = valid.numel(), valid.device
    start_out, key_out = torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int64, device=dev)
    count_out = torch.empty(n, dtype=torch.int32, device=dev)
    ws = _workspace("spg_batch_clouds_workspace", dev, n)
    _lib.call("spg_batch_clouds", valid, first_row, count, key, n, ws, ws.numel(), start_out, count_out, key_out,
              _lib.current_stream())
    return start_out, count_out, key_out


def batch_cloud_draw(key, count, n_clouds, n_points, n_attribs, seed, train, test_seed_offset=0, scale=0.0, rotate=0,
                     mirror_prob=0.0, jitter=False):
    """(sample_idx int32 [n, L], xform float64 [n, 9] or None, jitter float32 [n, L, F] or None) on the device: the
    cloud draws of the first n_clouds entries of key / count (see spg_batch_cloud_draw).  Evaluation (train False)
    draws neither matrices nor jitter."""
    _need_cuda(key, count)
    assert key.dtype == torch.int64 and count.dtype == torch.int32
    dev = key.device
    idx = torch.empty((n_clouds, n_points), dtype=torch.int32, device=dev)
    xform = torch.empty((n_clouds, 9), dtype=torch.float64, device=dev) if train else None
    noise = (torch.empty((n_clouds, n_points, n_attribs), dtype=torch.float32, device=dev)
             if train and jitter else None)
    _lib.call("spg_batch_cloud_draw", key, count, int(n_clouds), int(n_points), int(n_attribs), _seed64(seed),
              int(bool(train)), int(test_seed_offset), float(scale), int(rotate), float(mirror_prob), idx, xform,
              noise, _lib.current_stream())
    return idx, xform, noise
