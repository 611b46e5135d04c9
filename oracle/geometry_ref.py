"""Float64 numpy restatement of the k-NN graphs and geometric features of the partition pipelines
(ref: partition/graphs.py:11-70 `compute_graph_nn`, `compute_graph_nn_2`; partition/ply_c/ply_c.cpp:384-462
`compute_geof`).  Test infrastructure only; brute force, so meant for clouds of up to a few 10^4 points or for a
sample of rows.

Ranking: d2 = (dx dx + dy dy) + dz dz in float64 from the float32 coordinates (the expression sklearn's kd-tree
compares; its reported distances are numpy's sqrt of it), ties by the smaller index, the vertex itself first and
dropped.  compute_geof: fp64 mean and covariance / (k + 1), np.linalg.eigh, eigenvalues descending and clamped at
0, the reference's four formulas; NaN in all four where the largest eigenvalue is 0.
"""
import numpy as np


def sqdist(q, xyz):
    """d2 [m, n] between the rows q [m, 3] and xyz [n, 3] (float32 in, float64 out), the reference's expression."""
    q = np.asarray(q, np.float32).astype(np.float64)
    x = np.asarray(xyz, np.float32).astype(np.float64)
    dx = q[:, 0:1] - x[None, :, 0]
    dy = q[:, 1:2] - x[None, :, 1]
    dz = q[:, 2:3] - x[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def knn(xyz, k, rows=None, extra=1, chunk=128):
    """(ids int64 [m, k], d2 float64 [m, k + extra]) for the rows (all by default): the k nearest other vertices
    by (d2, index); d2 also holds the next `extra` candidates' values (inf where there are none)."""
    xyz = np.asarray(xyz, np.float32)
    n = xyz.shape[0]
    rows = np.arange(n) if rows is None else np.asarray(rows)
    kk = min(k + extra, n - 1)
    ids = np.empty((rows.size, k), np.int64)
    d2 = np.full((rows.size, k + extra), np.inf)
    for r0 in range(0, rows.size, chunk):
        r = rows[r0:r0 + chunk]
        D = sqdist(xyz[r], xyz)
        D[np.arange(r.size), r] = np.inf  # the vertex itself comes first and is dropped
        thr = np.partition(D, kk - 1, axis=1)[:, kk - 1]
        for i in range(r.size):
            cand = np.nonzero(D[i] <= thr[i])[0]
            order = np.lexsort((cand, D[i, cand]))[:kk]
            ids[r0 + i] = cand[order[:k]]
            d2[r0 + i, :kk] = D[i, cand[order]]
    return ids, d2


def compute_graph_nn(xyz, k_nn):
    """graphs.py:11-24 with the reference's dtypes (uint32 ids, float32 distances)."""
    n = np.asarray(xyz).shape[0]
    ids, d2 = knn(xyz, k_nn, extra=0)
    return {"is_nn": True, "source": np.repeat(np.arange(n), k_nn).astype("uint32"),
            "target": ids.reshape(-1).astype("uint32"),
            "distances": np.sqrt(d2[:, :k_nn]).reshape(-1).astype("float32")}


def compute_graph_nn_2(xyz, k_nn1, k_nn2):
    """graphs.py:26-70 without the voronoi branch: (graph of the first k_nn1 neighbours, target2 uint32)."""
    assert k_nn1 <= k_nn2, "knn1 must be smaller than knn2"
    n = np.asarray(xyz).shape[0]
    ids, d2 = knn(xyz, k_nn2, extra=0)
    graph = {"is_nn": True, "source": np.repeat(np.arange(n), k_nn1).astype("uint32"),
             "target": ids[:, :k_nn1].reshape(-1).astype("uint32"),
             "distances": np.sqrt(d2[:, :k_nn1]).reshape(-1).astype("float32")}
    return graph, ids.reshape(-1).astype("uint32")


def covariance(xyz, target, k_nn):
    """float64 [n, 3, 3]: the covariance / (k + 1) of every vertex and its k_nn neighbours, centred on the vertex
    first (translation changes nothing in exact arithmetic; coincident points give exactly 0)."""
    x = np.asarray(xyz, np.float32).astype(np.float64)
    n = x.shape[0]
    t = np.asarray(target).reshape(-1)[:n * k_nn].astype(np.int64).reshape(n, k_nn)
    P = np.concatenate([np.zeros((n, 1, 3)), x[t] - x[:, None, :]], 1)
    C = P - P.mean(1, keepdims=True)
    return np.einsum("nki,nkj->nij", C, C) / (k_nn + 1)


def compute_geof(xyz, target, k_nn, return_eigenvalues=False):
    """ply_c.cpp:384-462 in float64: float32 [n, 4] (linearity, planarity, scattering, verticality); with
    return_eigenvalues also the clamped eigenvalues [n, 3], descending."""
    w, V = np.linalg.eigh(covariance(xyz, target, k_nn))
    w, V = w[:, ::-1], V[:, :, ::-1]  # descending; column c of V is the vector of w[:, c]
    lam = np.maximum(w, 0.0)
    s = np.sqrt(lam)
    with np.errstate(divide="ignore", invalid="ignore"):
        lin = (s[:, 0] - s[:, 1]) / s[:, 0]
        pla = (s[:, 1] - s[:, 2]) / s[:, 0]
        sca = s[:, 2] / s[:, 0]
        unary = (lam[:, None, :] * np.abs(V)).sum(2)  # unary[r] = sum_c lambda_c |v_c[r]|
        vert = unary[:, 2] / np.sqrt((unary * unary).sum(1))
    out = np.stack([lin, pla, sca, vert], 1).astype(np.float32)
    return (out, lam) if return_eigenvalues else out
