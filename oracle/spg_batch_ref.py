"""Numpy restatement of the superpoint graph's batch builder (ref: learning/spg.py:114-143 `random_neighborhoods`,
`k_big_enough`, the permutation of `loader`; :178-193 `eccpc_collate`; learning/ecc/GraphConvInfo.py:33-69).

The draws are inputs instead of Python's global `random`: per graph, perm (perm[i] = new id of vertex i) or None,
centres (new ids) or None, and the hard cutoff k (0: none).  The neighbourhood union of igraph's `neighborhood`
is a level-synchronous multi-source breadth-first search ignoring edge directions.  Test infrastructure only.
"""
import numpy as np


def sample_graph(n, edges, s, perm, centres, order, minpts, k):
    """(kept original ids in sub-graph order, sub-graph edges [e, 2] in the file's edge order)."""
    edges = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    perm = np.arange(n) if perm is None else np.asarray(perm, dtype=np.int64)
    inv = np.empty(n, dtype=np.int64)
    inv[perm] = np.arange(n)
    if centres is None:
        kept = np.ones(n, dtype=bool)
    else:
        kept = np.zeros(n, dtype=bool)
        kept[inv[np.asarray(centres, dtype=np.int64)]] = True
        frontier = kept.copy()
        for _ in range(order):
            nxt = np.zeros(n, dtype=bool)
            nxt[edges[frontier[edges[:, 0]], 1]] = True
            nxt[edges[frontier[edges[:, 1]], 0]] = True
            frontier = nxt & ~kept
            kept |= nxt
    order_ids = inv[kept[inv]]  # kept original ids by increasing new id
    if k > 0:
        valid = np.asarray(s)[order_ids] >= minpts
        order_ids = order_ids[:np.argwhere(np.cumsum(valid) <= k)[-1][0] + 1]
    remap = -np.ones(n, dtype=np.int64)
    remap[order_ids] = np.arange(order_ids.shape[0])
    sel = (remap[edges[:, 0]] >= 0) & (remap[edges[:, 1]] >= 0)
    return order_ids, remap[edges[sel]], np.nonzero(sel)[0]


def collate(graphs, kind="stable"):
    """eccpc_collate's graph part over the graphs with edges: graphs = [(targets rows [n, T], sub-graph edges
    [e, 2], edge-feature rows [e, F])].  Returns (targets, idxn, degs, edgefeats, edge_index [2, E])."""
    idxn, tgts, degs, feats, p = [], [], [], [], 0
    for t, E, f in graphs:
        idx = E[:, 1].argsort(kind=kind)
        idxn.append(p + E[idx, 0])
        tgts.append(p + E[idx, 1])
        feats.append(np.asarray(f)[idx])
        degs.append(np.bincount(E[:, 1], minlength=t.shape[0]))
        p += t.shape[0]
    targets = np.concatenate([g[0] for g in graphs]).astype(np.int64)
    idxn, tgts = np.concatenate(idxn), np.concatenate(tgts)
    return targets, idxn, np.concatenate(degs).astype(np.int64), np.concatenate(feats), np.stack([idxn, tgts])
