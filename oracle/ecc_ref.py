"""ORACLE (test infrastructure, never imported by the product path).

CPU restatement of the reference's edge-conditioned convolution and its host-side graph
bookkeeping.  Pinned against the reference itself: tests/golden/make_golden.py imports
the reference checkout (SPG_REFERENCE) and stores its outputs, tests/test_oracle_golden.py checks
this file against them.

Each function cites the reference lines it restates (paths relative to the reference root).
"""
import numpy as np
import torch


# --------------------------------------------------------------------------- host bookkeeping
def edge_shards(degs, edge_mem_limit):
    """learning/ecc/utils.py:56-69 — blocks of output nodes holding ~edge_mem_limit edges each.
    Returns [(n_nodes, n_edges), ...]."""
    d = np.asarray(degs)
    cs = np.cumsum(d)
    bucket = cs // edge_mem_limit
    out, start = [], 0
    n = len(d)
    while start < n:
        stop = start
        while stop < n and bucket[stop] == bucket[start]:
            stop += 1
        out.append((stop - start, int(d[start:stop].sum())))
        start = stop
    return out


def graph_conv_info(edge_lists, n_vertices, edge_feats):
    """learning/ecc/GraphConvInfo.py:33-69 without igraph.

    edge_lists[g]: int array [E_g, 2] of (source, target); n_vertices[g]: vertex count;
    edge_feats[g]: [E_g, Fe].  Returns (idxn int64[E], degrees int64[N], edgefeats [E,Fe],
    edge_indexes int64[2,E]) with edges of every graph sorted by target using numpy's default
    argsort, exactly as line :50 does."""
    p = 0
    idxn, degs, feats, eidx = [], [], [], []
    for E, nv, f in zip(edge_lists, n_vertices, edge_feats):
        E = np.asarray(E)
        order = E[:, 1].argsort()                       # :50
        idxn.append(p + E[order, 0])                    # :52
        feats.append(np.asarray(f)[order])              # :53-55 (attribute values in sorted order)
        degs.append(np.bincount(E[:, 1], minlength=nv))  # :56 in-degree incl. loops
        eidx.append(p + E[order])                       # :57
        p += nv                                         # :58
    return (np.concatenate(idxn).astype(np.int64), np.concatenate(degs).astype(np.int64),
            np.concatenate(feats), np.concatenate(eidx).T.astype(np.int64))


# ------------------------------------------------------------------------------------- forward
def graph_conv_forward_loop(x, w, idxn, idxe, degs):
    """learning/ecc/GraphConvModule.py:59-94, CPU branch: gather, per-edge product, then a Python
    loop taking torch.mean over each node's slice; zero rows for zero-degree nodes."""
    sel = x.index_select(0, idxn)                                   # :66
    ww = w if idxe is None else w.index_select(0, idxe)             # :68-71
    if w.dim() == 3:
        prod = torch.bmm(sel.unsqueeze(1), ww).squeeze(1)           # :38
    else:
        prod = sel * ww                                             # :41
    out = x.new_zeros((len(degs), prod.shape[1]))
    k = 0
    for i, d in enumerate(degs.tolist()):                           # :82-88
        if d > 0:
            out[i] = prod[k:k + d].mean(0)
        k += d
    return out


def graph_conv_forward(x, w, idxn, idxe, degs):
    """Same result, vectorised and differentiable (follows the didactic
    GraphConvModulePureAutograd, GraphConvModule.py:228-247): segment sum / degree."""
    sel = x.index_select(0, idxn)
    ww = w if idxe is None else w.index_select(0, idxe)
    prod = torch.bmm(sel.unsqueeze(1), ww).squeeze(1) if w.dim() == 3 else sel * ww
    tgt = torch.repeat_interleave(torch.arange(len(degs)), degs)
    out = x.new_zeros((len(degs), prod.shape[1])).index_add_(0, tgt, prod)
    return out / degs.clamp(min=1).to(x.dtype).unsqueeze(1)


def graph_conv_backward(x, w, idxn, idxe, degs, grad_out):
    """learning/ecc/GraphConvModule.py:96-152: grad_products = grad_out[tgt]/deg (:110-121),
    grad_weights = x[idxn] (outer|elementwise) grad_products (:124-133, index_add_ under idxe),
    grad_input = index_add_(idxn, grad_products (@ W^T | * w)) (:136-146)."""
    tgt = torch.repeat_interleave(torch.arange(len(degs)), degs)
    gp = grad_out.index_select(0, tgt) / degs.index_select(0, tgt).to(x.dtype).unsqueeze(1)
    sel = x.index_select(0, idxn)
    ww = w if idxe is None else w.index_select(0, idxe)
    if w.dim() == 3:
        gw_e = torch.bmm(sel.unsqueeze(2), gp.unsqueeze(1))
        gx_e = torch.bmm(gp.unsqueeze(1), ww.transpose(1, 2)).squeeze(1)
    else:
        gw_e = sel * gp
        gx_e = gp * ww
    if idxe is None:
        gw = gw_e
    else:
        gw = torch.zeros_like(w).index_add_(0, idxe, gw_e)
    gx = torch.zeros_like(x).index_add_(0, idxn, gx_e)
    return gx, gw


class GraphConvLoop(torch.autograd.Function):
    """The reference's CPU code path with its per-node Python loops in forward (:82-88) and
    backward (:114-121); used as the faithful CPU baseline ("port") in bench.py."""

    @staticmethod
    def forward(ctx, x, w, idxn, degs):
        ctx.save_for_backward(x, w)
        ctx.idxn, ctx.degs = idxn, degs
        return graph_conv_forward_loop(x, w, idxn, None, degs)

    @staticmethod
    def backward(ctx, grad_out):
        x, w = ctx.saved_tensors
        idxn, degs = ctx.idxn, ctx.degs
        gp = x.new_empty((idxn.numel(), grad_out.shape[1]))
        k = 0
        for i, d in enumerate(degs.tolist()):
            if d > 0:
                gp[k:k + d] = grad_out[i] / d
                k += d
        sel = x.index_select(0, idxn)
        if w.dim() == 3:
            gw = torch.bmm(sel.unsqueeze(2), gp.unsqueeze(1))
            gx_e = torch.bmm(gp.unsqueeze(1), w.transpose(1, 2)).squeeze(1)
        else:
            gw = sel * gp
            gx_e = gp * w
        gx = torch.zeros_like(x).index_add_(0, idxn, gx_e)
        return gx, gw, None, None
