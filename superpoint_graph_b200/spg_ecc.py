"""Edge-conditioned convolution with the reference's `learning/ecc` API on the sm_90a kernels.

Mirrors (names, argument order, defaults, error behaviour):
  GraphConvInfo      ref: learning/ecc/GraphConvInfo.py:16-86
  GraphConvFunction  ref: learning/ecc/GraphConvModule.py:19-152
  GraphConvModule    ref: learning/ecc/GraphConvModule.py:156-193
  get_edge_shards    ref: learning/ecc/utils.py:56-69

The kernels stream over a CSR and need no sharding, so `edge_mem_limit` is accepted and ignored
(the reference's own test asserts shard invariance: learning/ecc/test_GraphConvModule.py:59-75).
"""
from collections import defaultdict

import numpy as np
import torch
import torch.nn as nn

from . import ops


class GraphConvInfo(object):
    """Vectorised structure of a batch of graphs (disjoint union).  Host-side, numpy only.

    `graphs` are igraph-like objects (get_edgelist(), es[...] / es.attributes(), indegree(),
    vcount()); integer outputs are produced by the same numpy calls as the reference so that
    they are bit-identical (default-kind argsort on the target column included)."""

    def __init__(self, *args, **kwargs):
        self._idxn = None
        self._idxe = None
        self._degrees = None
        self._degrees_gpu = None
        self._edgefeats = None
        self._edge_indexes = None
        self._graph = None  # ops.EccGraph, built lazily
        if len(args) > 0 or len(kwargs) > 0:
            self.set_batch(*args, **kwargs)

    def set_batch(self, graphs, edge_feat_func):
        """Disjoint union of `graphs` in the target-sorted edge order of the reference
        (ref: learning/ecc/GraphConvInfo.py:33-69), built from arrays: one vertex offset per graph,
        one per-graph argsort of the target column (numpy's default kind on the same int64 column as the
        reference, hence the same — not merely an equivalent — permutation), in-degrees by bincount."""
        graphs = list(graphs) if isinstance(graphs, (list, tuple)) else [graphs]
        edges = [np.asarray(G.get_edgelist(), dtype=np.int64).reshape(-1, 2) for G in graphs]
        sizes = np.asarray([G.vcount() for G in graphs], dtype=np.int64)
        offsets = np.cumsum(sizes) - sizes
        orders = [E[:, 1].argsort() for E in edges]
        pairs = [off + E[o] for E, o, off in zip(edges, orders, offsets)]  # [e_g, 2] = (source, target)
        pairs = np.concatenate(pairs) if pairs else np.zeros((0, 2), dtype=np.int64)
        total = int(sizes.sum())
        # every edge attribute, gathered per graph in that graph's sorted order (lists, as igraph yields)
        names = []
        for G in graphs:
            names += [a for a in G.es.attributes() if a not in names]
        edgeattrs = defaultdict(list)
        for G, o in zip(graphs, orders):
            picked = G.es[o.tolist()]
            for a in G.es.attributes():
                edgeattrs[a] += picked.get_attribute_values(a)
        self._edgefeats, self._idxe = edge_feat_func(edgeattrs)
        self._idxn = torch.from_numpy(np.ascontiguousarray(pairs[:, 0]))
        if self._idxe is not None:
            assert self._idxe.numel() == self._idxn.numel()
        self._degrees = torch.from_numpy(np.bincount(pairs[:, 1], minlength=total).astype(np.int64))
        self._degrees_gpu = None
        self._edge_indexes = torch.from_numpy(np.ascontiguousarray(pairs.T))
        self._graph = None

    @classmethod
    def from_arrays(cls, idxn, degrees, edgefeats, idxe=None):
        """Builds the info object from already target-sorted arrays (synthetic data, tests)."""
        gi = cls()
        gi._idxn = torch.as_tensor(idxn, dtype=torch.long)
        gi._degrees = torch.as_tensor(degrees, dtype=torch.long)
        gi._edgefeats = torch.as_tensor(edgefeats)
        gi._idxe = None if idxe is None else torch.as_tensor(idxe, dtype=torch.long)
        tgt = torch.repeat_interleave(torch.arange(gi._degrees.numel()), gi._degrees)
        gi._edge_indexes = torch.stack([gi._idxn, tgt])
        return gi

    def graph(self):
        """The CSR bundle the kernels read (built once per batch from idxn/degs: on the device by cuda(),
        else on first use from the host arrays)."""
        if self._graph is None:
            self._graph = ops.EccGraph(self._idxn, self._idxe, self._degrees,
                                       n_in=int(self._degrees.numel()))
        return self._graph

    def cuda(self):
        """Uploads the buffers (GraphConvInfo.py:71-77) and builds the kernels' CSR views on the device from
        the uploaded (idxn, degs) pair (spg_graph_build) unless a host-built graph exists already."""
        self._idxn = self._idxn.cuda()
        if self._idxe is not None:
            self._idxe = self._idxe.cuda()
        self._degrees_gpu = self._degrees.cuda()
        self._edgefeats = self._edgefeats.cuda()
        self._edge_indexes = self._edge_indexes.cuda()
        if self._graph is None:
            self._graph = ops.EccGraph.from_device(self._idxn, self._degrees_gpu, n_in=int(self._degrees.numel()),
                                                   idxe=self._idxe, check=True)
        else:
            self._graph.to(self._idxn.device)

    def get_buffers(self):
        return self._idxn, self._idxe, self._degrees, self._degrees_gpu, self._edgefeats

    def get_pyg_buffers(self):
        return self._edge_indexes


def _graph_for(idxn, idxe, degs, degs_gpu, n_in):
    """EccGraph for a raw (idxn, idxe, degs, degs_gpu) argument list, cached on the degs tensor object and
    keyed on the identity AND version of the index tensors (an in-place edit invalidates it).  CUDA
    arguments are turned into the CSR views on the device; host arguments by the numpy builder."""
    cache = getattr(degs, "_spg_graph", None)
    key = (idxn.data_ptr(), idxn._version, None if idxe is None else (idxe.data_ptr(), idxe._version),
           degs._version, int(idxn.numel()), n_in)
    if cache is not None and cache[0] == key:
        return cache[1]
    if idxn.is_cuda and degs_gpu is not None and degs_gpu.is_cuda:
        g = ops.EccGraph.from_device(idxn.long().contiguous(), degs_gpu.long().contiguous(), n_in=n_in,
                                     idxe=idxe, check=True)
    else:
        g = ops.EccGraph(idxn, idxe, degs, n_in=n_in)
    try:
        degs._spg_graph = (key, g)
    except Exception:
        pass
    return g


class GraphConvFunction(torch.autograd.Function):
    """out[i] = mean over in-edges e of (input[idxn[e]] (*|@) weights[e]); zero rows for
    zero-degree nodes.  2-D weights: element-wise product; 3-D weights: vector-matrix product."""

    @staticmethod
    def forward(ctx, input, weights, in_channels, out_channels, idxn, idxe, degs, degs_gpu,
                edge_mem_limit=1e20):
        full = weights.dim() == 3
        assert full or (in_channels == out_channels and weights.size(1) == in_channels)
        graph = idxn if isinstance(idxn, ops.EccGraph) else _graph_for(idxn, idxe, degs, degs_gpu,
                                                                       int(input.shape[0]))
        ctx.save_for_backward(input, weights)
        ctx._graph = graph
        ctx._in_channels, ctx._out_channels = in_channels, out_channels
        return ops.ecc_fwd(input, weights, graph, out_channels)

    @staticmethod
    def backward(ctx, grad_output):
        input, weights = ctx.saved_tensors
        g = grad_output.contiguous()
        graph = ctx._graph
        grad_input = grad_weights = None
        if ctx.needs_input_grad[1]:
            grad_weights = ops.ecc_bwd_w(input, g, graph, tuple(weights.shape), n_iter=1)
        if ctx.needs_input_grad[0]:
            grad_input = ops.ecc_bwd_x(weights, g, graph, ctx._in_channels)
        return grad_input, grad_weights, None, None, None, None, None, None, None


class GraphConvModule(nn.Module):
    """Graph convolution whose filters come from `filter_net(edge features)`."""

    def __init__(self, in_channels, out_channels, filter_net, gc_info=None, edge_mem_limit=1e20):
        super(GraphConvModule, self).__init__()
        self._in_channels = in_channels
        self._out_channels = out_channels
        self._fnet = filter_net
        self._edge_mem_limit = edge_mem_limit
        self.set_info(gc_info)

    def set_info(self, gc_info):
        self._gci = gc_info

    def forward(self, input):
        from .dense import run_sequential

        idxn, idxe, degs, degs_gpu, edgefeats = self._gci.get_buffers()
        weights = run_sequential(self._fnet, edgefeats, self.training)
        assert input.dim() == 2 and weights.dim() == 2 and (
            weights.size(1) == self._in_channels * self._out_channels or
            (self._in_channels == self._out_channels and weights.size(1) == self._in_channels))
        if weights.size(1) == self._in_channels * self._out_channels:
            weights = weights.view(-1, self._in_channels, self._out_channels)
        return GraphConvFunction.apply(input, weights, self._in_channels, self._out_channels,
                                       self._gci.graph(), idxe, degs, degs_gpu,
                                       self._edge_mem_limit)


def get_edge_shards(degs, edge_mem_limit):
    """Splits the node range into blocks of about `edge_mem_limit` edges; returns
    [(num_nodes, num_edges), ...].  Kept for API parity; the kernels ignore sharding."""
    d = degs if isinstance(degs, np.ndarray) else degs.numpy()
    cs = np.cumsum(d)
    block = cs // edge_mem_limit
    _, first, count = np.unique(block, return_index=True, return_counts=True)
    shards = []
    for b in range(len(first)):
        last_edge = cs[-1] if b == len(first) - 1 else cs[first[b + 1] - 1]
        shards.append((int(count[b]), int(last_edge - cs[first[b]] + d[first[b]])))
    return shards
