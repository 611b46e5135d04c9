"""Vectorised numpy restatement of the superpoint graph (ref: partition/graphs.py:75-210 `compute_sp_graph`).
Test infrastructure only.  Sort-based, with no per-component Python loop, so it runs on 10^5-10^6 points.

Superpoints: the points sorted by (component, x, y, z) (-0 equal to +0, as np.unique(axis=0) compares them), the
unique rows marked.  The centroid is numpy's np.mean of the unique rows: a sequential float32 sum in sorted order from
+0, divided by the unique-row count u (the row itself when u == 1).  u == 2: the length is numpy's fp32
sqrt(sum(var)).  u >= 3: the float64 covariance (ddof 1) of the unique rows, np.linalg.eigh, eigenvalues
descending; length = ev0, surface = sqrt(ev0 ev1 + 1e-10), volume = sqrt(ev0 ev1 ev2 + 1e-10), rounded once to float32.

Superedges: the 6 vertex pairs of every tetrahedron whose endpoints lie in different components, both directions,
deduplicated; with d_max > 0 those with fp32 sqrt((dx dx + dy dy) + dz dz) < float32(d_max) kept; grouped by the
exact (source component, target component) key in ascending order.  Delta statistics in float64 of the exact
differences, rounded once (a block of one pair: its fp32 delta, std 0, its fp32 norm); ratios as the reference.
"""
import numpy as np

F32 = np.float32
PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


def _fkey(x):
    """Order-preserving uint64 keys of float32 values, -0 mapped to +0."""
    u = (np.asarray(x, F32) + F32(0)).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)


def _seq_sum(vals, start, count):
    """Per segment [start, start + count) of vals [m, c] (float32): numpy's sequential float32 sum from +0."""
    acc = np.zeros((start.size, vals.shape[1]), F32)
    order = np.argsort(-count, kind="stable")
    cnt = count[order]
    for j in range(int(cnt.max()) if cnt.size else 0):
        a = int(np.count_nonzero(cnt > j))  # the segments with count > j: a prefix of `order`
        act = order[:a]
        acc[act] = acc[act] + vals[start[act] + j]
    return acc


def sort_points(xyz, in_component):
    """(order, comp_sorted, unique flags) of the points sorted by (component, x, y, z)."""
    xyz = np.asarray(xyz, F32)
    comp = np.asarray(in_component).astype(np.int64)
    k = [_fkey(xyz[:, c]) for c in range(3)]
    order = np.lexsort((k[2], k[1], k[0], comp))
    cs = comp[order]
    ks = [kk[order] for kk in k]
    first = np.ones(len(order), bool)
    first[1:] = (cs[1:] != cs[:-1]) | (ks[0][1:] != ks[0][:-1]) | (ks[1][1:] != ks[1][:-1]) | (ks[2][1:] != ks[2][:-1])
    return order, cs, first


def superpoints(xyz, in_component, labels, n_labels):
    """dict of sp_centroids [n_com, 3], sp_length / sp_surface / sp_volume [n_com, 1] (float32), sp_point_count
    [n_com, 1] and sp_labels [n_com, n_labels + 1] (int64, [] without labels), u [n_com] (unique rows)."""
    xyz = np.asarray(xyz, F32)
    comp = np.asarray(in_component).astype(np.int64)
    n_com = int(comp.max()) + 1
    order, cs, first = sort_points(xyz, comp)
    m = np.bincount(comp, minlength=n_com)
    if (m == 0).any():
        raise ValueError("component %d holds no point" % int(np.argmin(m)))
    uc = cs[first]
    rows = xyz[order][first]
    u = np.bincount(uc, minlength=n_com)
    ustart = np.concatenate([[0], np.cumsum(u)[:-1]])
    acc = _seq_sum(rows, ustart, u)
    cen = (acc.astype(np.float64) / u[:, None]).astype(F32)  # np.mean divides by the integer count in float64
    one = u == 1
    cen[one] = rows[ustart[one]]  # graphs.py:157 assigns the unique row itself
    length = np.zeros(n_com, F32)
    surface = np.zeros(n_com, F32)
    volume = np.zeros(n_com, F32)
    # u == 2: np.var's fp32 sequence, the centroid being its mean
    two = np.nonzero(u == 2)[0]
    if two.size:
        a, b = rows[ustart[two]], rows[ustart[two] + 1]
        xa, xb = a - cen[two], b - cen[two]
        var = ((F32(0) + xa * xa) + xb * xb) / F32(2)
        s = ((F32(0) + var[:, 0]) + var[:, 1]) + var[:, 2]
        length[two] = np.sqrt(s)
    big = np.nonzero(u >= 3)[0]
    if big.size:
        r64 = rows.astype(np.float64)
        mean = np.stack([np.bincount(uc, weights=r64[:, c], minlength=n_com) for c in range(3)], 1) / u[:, None]
        d = r64 - mean[uc]
        C = np.empty((n_com, 3, 3))
        for i in range(3):
            for j in range(i, 3):
                C[:, i, j] = C[:, j, i] = np.bincount(uc, weights=d[:, i] * d[:, j], minlength=n_com)
        C = C[big] / (u[big] - 1)[:, None, None]
        ev = np.linalg.eigvalsh(C)[:, ::-1]
        length[big] = ev[:, 0]
        surface[big] = np.sqrt(ev[:, 0] * ev[:, 1] + 1e-10)
        volume[big] = np.sqrt(ev[:, 0] * ev[:, 1] * ev[:, 2] + 1e-10)
    out = {"sp_centroids": cen, "sp_length": length[:, None], "sp_surface": surface[:, None],
           "sp_volume": volume[:, None], "sp_point_count": m.astype(np.int64)[:, None], "u": u}
    out["sp_labels"] = sp_labels(comp, n_com, labels, n_labels)
    return out


def sp_labels(comp, n_com, labels, n_labels):
    """graphs.py:79-80,148-153: histogram of the values 0..n_labels, or the sum of the label rows."""
    if len(labels) <= 1:
        return []
    lab = np.asarray(labels)
    if lab.ndim > 1 and lab.shape[1] > 1:
        out = np.zeros((n_com, lab.shape[1]), np.int64)
        np.add.at(out, comp, lab.astype(np.int64))
        return out
    v = lab.reshape(-1).astype(np.int64)
    ok = (v >= 0) & (v <= n_labels)
    return np.bincount(comp[ok] * (n_labels + 1) + v[ok], minlength=n_com * (n_labels + 1)).reshape(
        n_com, n_labels + 1).astype(np.int64)


def vertex_pairs(xyz, in_component, simplices, d_max):
    """(a, b) int64: the deduplicated directed pairs across components, sorted by (a, b), after the d_max cut."""
    xyz = np.asarray(xyz, F32)
    comp = np.asarray(in_component).astype(np.int64)
    s = np.asarray(simplices).astype(np.int64)
    n = xyz.shape[0]
    a = np.concatenate([s[:, i] for i, j in PAIRS])
    b = np.concatenate([s[:, j] for i, j in PAIRS])
    keep = comp[a] != comp[b]
    a, b = a[keep], b[keep]
    key = np.unique(np.concatenate([a * n + b, b * n + a]))
    a, b = key // n, key % n
    if d_max > 0:
        d = xyz[a] - xyz[b]
        dist = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        keep = dist < F32(d_max)
        a, b = a[keep], b[keep]
    return a, b


def superedges(xyz, in_component, simplices, d_max, sp):
    """dict of source, target [n_sedg, 1] (int64) and the se_* features, plus `pairs` [n_sedg] (block sizes)."""
    xyz = np.asarray(xyz, F32)
    comp = np.asarray(in_component).astype(np.int64)
    n_com = sp["sp_centroids"].shape[0]
    a, b = vertex_pairs(xyz, comp, simplices, d_max)
    key = comp[a] * n_com + comp[b]
    order = np.argsort(key, kind="stable")
    a, b, key = a[order], b[order], key[order]
    ukey, start, cnt = np.unique(key, return_index=True, return_counts=True)
    src, tgt = ukey // n_com, ukey % n_com
    blk = np.repeat(np.arange(ukey.size), cnt)
    d = xyz[a].astype(np.float64) - xyz[b].astype(np.float64)
    norm = np.sqrt((d * d).sum(1))
    sums = lambda v: np.add.reduceat(v, start, axis=0) if v.size else np.zeros((0,) + v.shape[1:])
    mean = sums(d) / cnt[:, None]
    std = np.sqrt(sums((d - mean[blk]) ** 2) / cnt[:, None])
    nrm = sums(norm) / cnt
    mean, std, nrm = mean.astype(F32), std.astype(F32), nrm.astype(F32)
    one = cnt == 1
    d32 = xyz[a[start[one]]] - xyz[b[start[one]]]
    mean[one] = d32
    std[one] = 0
    nrm[one] = np.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
    cen, pc = sp["sp_centroids"], sp["sp_point_count"][:, 0]
    ratio = lambda k: (sp[k][src, 0] / (sp[k][tgt, 0] + F32(1e-6))).astype(F32)[:, None]
    return {"source": src[:, None], "target": tgt[:, None], "se_delta_mean": mean, "se_delta_std": std,
            "se_delta_norm": nrm[:, None], "se_delta_centroid": cen[src] - cen[tgt],
            "se_length_ratio": ratio("sp_length"), "se_surface_ratio": ratio("sp_surface"),
            "se_volume_ratio": ratio("sp_volume"),
            "se_point_count_ratio": (pc[src].astype(np.float64) / (pc[tgt].astype(np.float64) + 1e-6)).astype(
                F32)[:, None], "pairs": cnt}


def compute_sp_graph(xyz, d_max, in_component, labels, n_labels, simplices):
    """graphs.py:75-210 with exact superedge keys; the superpoint and superedge dicts merged, is_nn False."""
    sp = superpoints(xyz, in_component, labels, n_labels)
    g = {"is_nn": False}
    g.update(sp)
    g.update(superedges(xyz, in_component, simplices, d_max, sp))
    return g
