"""k-NN graphs and geometric features of a point cloud (superpoint_graph_b200.spg_geometry, csrc/geometry.cu).

CPU: the float64 oracle (oracle/geometry_ref.py) against the reference's own graphs (geometry.npz, from the unmodified
partition/graphs.py): distances bit for bit, ids wherever untied; the oracle's compute_geof on analytic
neighbourhoods; host validation.
GPU: every golden cloud and parameter pair; seeded clouds of 10^5-10^6 points against the reference's distance
expression and scipy's cKDTree; compute_geof against the float64 oracle; edge cases; local_geometry fed to the
learned partition's batch builder.
"""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import geometry_ref as gref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geometry.npz")
_Z = np.load(GOLDEN, allow_pickle=False)
G = {k: _Z[k] for k in _Z.files}
META = json.loads(str(G["meta"]))
CLOUDS = [c["name"] for c in META["clouds"]]
PAIRS = [tuple(p) for p in META["pairs"]]
CASES = [(c, p) for c in CLOUDS for p in PAIRS]


def _gold(cloud, pair, key):
    return G["%s.%d_%d.%s" % (cloud, pair[0], pair[1], key)]


def _d2_rows(xyz, ids):
    """The reference's d2 from every vertex to its listed ids [n, k]."""
    x = xyz.astype(np.float64)
    d = x[:, None, :] - x[ids]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def check_ids(xyz, got, want, next_d2):
    """Tie-aware id check of got [n, k] against want [n, k]: every got id carries the distance of its position in
    want, with no repeats and never the vertex itself; wherever the d2 of a position is untied (with its neighbours
    in the row and with the next candidate next_d2 [n]) the ids are equal."""
    n, k = got.shape
    got, want = got.astype(np.int64), want.astype(np.int64)
    assert ((got >= 0) & (got < n)).all()
    dg, dw = _d2_rows(xyz, got), _d2_rows(xyz, want)
    assert np.array_equal(dg, dw), "ids with other distances in %d rows" % int((dg != dw).any(1).sum())
    s = np.sort(got, 1)
    assert (s[:, 1:] != s[:, :-1]).all(), "repeated id"
    assert (got != np.arange(n)[:, None]).all(), "a vertex in its own list"
    ext = np.concatenate([np.full((n, 1), -1.0), dw, next_d2.reshape(n, 1)], 1)
    untied = (ext[:, 1:-1] != ext[:, :-2]) & (ext[:, 1:-1] != ext[:, 2:])
    assert np.array_equal(got[untied], want[untied])
    return int(untied.sum())


# ---------------------------------------------------------------------------------------------------- CPU
def test_golden_records_versions_and_clouds():
    assert META["sklearn"] and META["numpy"] and META["scipy"]
    assert set(CLOUDS) == {"room", "lidar", "lattice", "line", "blob", "offset"}
    assert set(PAIRS) == {(10, 45), (5, 20)}
    assert os.path.getsize(GOLDEN) < 1 << 20
    # the lattice has exact ties and the blob more than k + 2 coincident points
    lat = G["lattice.10_45.distances"].reshape(-1, 10)
    assert (lat[:, 1:] == lat[:, :-1]).any()
    assert (G["blob.10_45.distances"] == 0).sum() >= 60 * 10


@pytest.mark.parametrize("cloud,pair", CASES)
def test_oracle_reproduces_golden(cloud, pair):
    k1, k2 = pair
    xyz = G[cloud + ".xyz"]
    n = xyz.shape[0]
    graph, target2 = gref.compute_graph_nn_2(xyz, k1, k2)
    _, d2 = gref.knn(xyz, k2, extra=1)
    assert np.array_equal(graph["source"], _gold(cloud, pair, "source").astype(np.uint32))
    assert np.array_equal(graph["distances"].view(np.uint32), _gold(cloud, pair, "distances").view(np.uint32))
    nn = gref.compute_graph_nn(xyz, k1)
    assert np.array_equal(nn["distances"].view(np.uint32), _gold(cloud, pair, "nn.distances").view(np.uint32))
    check_ids(xyz, target2.reshape(n, k2), _gold(cloud, pair, "target2").reshape(n, k2), d2[:, k2])
    check_ids(xyz, graph["target"].reshape(n, k1), _gold(cloud, pair, "target").reshape(n, k1), d2[:, k1])
    check_ids(xyz, nn["target"].reshape(n, k1), _gold(cloud, pair, "nn.target").reshape(n, k1), d2[:, k1])


def _geof_of(points, k):
    """compute_geof of vertex 0 of `points` with every other point as its neighbours."""
    pts = np.asarray(points, np.float32)
    n = pts.shape[0]
    assert n == k + 1
    target = np.array([[j for j in range(n) if j != i] for i in range(n)])
    return gref.compute_geof(pts, target, k)[0]


def test_oracle_geof_analytic():
    t = np.linspace(-1, 1, 11)
    # a line: linearity 1, planarity and scattering 0; vertical line verticality 1, horizontal 0
    f = _geof_of(np.c_[t * 0, t * 0, t][np.r_[5, 0:5, 6:11]], 10)
    assert abs(f[0] - 1) < 1e-6 and abs(f[1]) < 1e-6 and abs(f[2]) < 1e-6 and abs(f[3] - 1) < 1e-6
    f = _geof_of(np.c_[t, 0.5 * t, t * 0][np.r_[5, 0:5, 6:11]], 10)
    assert abs(f[0] - 1) < 1e-6 and abs(f[3]) < 1e-6
    # a horizontal disc (isotropic in its plane): planarity 1, verticality 0
    a = np.arange(12) * (2 * np.pi / 12)
    f = _geof_of(np.r_[[[0, 0, 0]], np.c_[np.cos(a), np.sin(a), 0 * a]], 12)
    assert abs(f[1] - 1) < 1e-6 and abs(f[0]) < 1e-6 and abs(f[2]) < 1e-6 and abs(f[3]) < 1e-6
    # a wall elongated in z: verticality high
    f = _geof_of(np.r_[[[0, 0, 0]], np.c_[0.3 * np.cos(a), 0 * a, 2 * np.sin(a)]], 12)
    assert f[3] > 0.99
    # an isotropic blob (the six octahedron vertices): scattering 1
    oct_ = np.r_[np.eye(3), -np.eye(3)]
    f = _geof_of(np.r_[[[0, 0, 0]], oct_], 6)
    assert abs(f[2] - 1) < 1e-6 and abs(f[0]) < 1e-6 and abs(f[1]) < 1e-6
    # k + 1 coincident points: NaN in all four columns
    f = _geof_of(np.full((21, 3), 7.25), 20)
    assert np.isnan(f).all()


def test_host_validation():
    from superpoint_graph_b200.spg_geometry import compute_geof, compute_graph_nn, compute_graph_nn_2
    from superpoint_graph_b200 import ops
    xyz = G["room.xyz"]
    with pytest.raises(AssertionError, match="knn1 must be smaller than knn2"):
        compute_graph_nn_2(xyz, 20, 10)
    with pytest.raises(NotImplementedError):
        compute_graph_nn_2(xyz, 10, 45, voronoi=0.5)
    with pytest.raises(ValueError, match="n_neighbors"):
        compute_graph_nn(xyz[:10], 10)
    with pytest.raises(ValueError, match="n_neighbors"):
        compute_graph_nn_2(xyz[:45], 10, 45)
    with pytest.raises(TypeError):
        compute_graph_nn(xyz.astype(np.float64), 10)
    with pytest.raises(TypeError):
        compute_graph_nn_2(torch.from_numpy(xyz).double(), 10, 45)
    with pytest.raises(ValueError):
        compute_graph_nn(xyz[:, :2].copy(), 10)
    with pytest.raises(ValueError):
        compute_graph_nn(xyz, 0)
    cap = ops.knn_max_k()
    assert cap >= 64
    with pytest.raises(ValueError, match="cap of %d" % cap):
        compute_graph_nn(xyz, cap + 1)
    with pytest.raises(ValueError, match="cap of %d" % cap):
        compute_graph_nn_2(xyz, 10, cap + 1)
    huge = np.broadcast_to(np.zeros(3, np.float32), (2 ** 31, 3))
    with pytest.raises(ValueError, match="2\\^31"):
        compute_graph_nn(huge, 10)
    n = xyz.shape[0]
    with pytest.raises(ValueError):
        compute_geof(xyz, np.zeros(n * 45 - 1, np.uint32), 45)
    with pytest.raises(TypeError):
        compute_geof(xyz, np.zeros(n * 45, np.float32), 45)
    with pytest.raises(TypeError):
        compute_geof(xyz.astype(np.float64), np.zeros(n * 45, np.uint32), 45)


# ---------------------------------------------------------------------------------------------------- GPU
def _np(t):
    return t.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("cloud,pair", CASES)
def test_device_graphs_match_golden(cloud, pair):
    from superpoint_graph_b200.spg_geometry import compute_graph_nn, compute_graph_nn_2
    k1, k2 = pair
    xyz = G[cloud + ".xyz"]
    n = xyz.shape[0]
    _, d2 = gref.knn(xyz, k2, extra=1)
    graph, target2 = compute_graph_nn_2(xyz, k1, k2)
    assert graph["is_nn"] is True
    assert target2.is_cuda and target2.dtype == torch.int64 and graph["distances"].dtype == torch.float32
    assert np.array_equal(_np(graph["source"]), _gold(cloud, pair, "source").astype(np.int64))
    assert np.array_equal(_np(graph["distances"]).view(np.uint32), _gold(cloud, pair, "distances").view(np.uint32))
    check_ids(xyz, _np(target2).reshape(n, k2), _gold(cloud, pair, "target2").reshape(n, k2), d2[:, k2])
    check_ids(xyz, _np(graph["target"]).reshape(n, k1), _gold(cloud, pair, "target").reshape(n, k1), d2[:, k1])
    nn = compute_graph_nn(torch.from_numpy(xyz).cuda(), k1)
    assert np.array_equal(_np(nn["source"]), _gold(cloud, pair, "source").astype(np.int64))
    assert np.array_equal(_np(nn["distances"]).view(np.uint32), _gold(cloud, pair, "nn.distances").view(np.uint32))
    check_ids(xyz, _np(nn["target"]).reshape(n, k1), _gold(cloud, pair, "nn.target").reshape(n, k1), d2[:, k1])


def room_cloud(n, seed):
    """Seeded room-like surfaces: floor, ceiling, four walls, tables and cylinders (float32)."""
    rng = np.random.default_rng(seed)
    W, D, H = 12.0, 8.0, 3.0
    parts = []
    m = n // 8
    parts.append(np.c_[rng.uniform(0, W, m), rng.uniform(0, D, m), np.zeros(m)])
    parts.append(np.c_[rng.uniform(0, W, m), rng.uniform(0, D, m), np.full(m, H)])
    parts.append(np.c_[rng.uniform(0, W, m), np.zeros(m), rng.uniform(0, H, m)])
    parts.append(np.c_[rng.uniform(0, W, m), np.full(m, D), rng.uniform(0, H, m)])
    parts.append(np.c_[np.zeros(m), rng.uniform(0, D, m), rng.uniform(0, H, m)])
    parts.append(np.c_[np.full(m, W), rng.uniform(0, D, m), rng.uniform(0, H, m)])
    parts.append(np.c_[rng.uniform(2, 5, m), rng.uniform(2, 4, m), np.full(m, 0.75)])
    r = n - 7 * m
    a = rng.uniform(0, 2 * np.pi, r)
    parts.append(np.c_[9 + 0.3 * np.cos(a), 5 + 0.3 * np.sin(a), rng.uniform(0, 2, r)])
    xyz = np.concatenate(parts) + rng.normal(0, 0.002, (n, 3))
    return xyz[rng.permutation(n)].astype(np.float32)


def falloff_cloud(n, seed):
    """Seeded LiDAR-like scan: a ground plane and building faces whose density falls off as 1 / range^2."""
    rng = np.random.default_rng(seed)
    m = (2 * n) // 3
    rg = np.exp(rng.uniform(np.log(1.0), np.log(80.0), m))
    a = rng.uniform(0, 2 * np.pi, m)
    ground = np.c_[rg * np.cos(a), rg * np.sin(a), rng.normal(0, 0.02, m)]
    w = n - m
    d = np.exp(rng.uniform(np.log(5.0), np.log(60.0), w))
    side = rng.integers(0, 2, w) * 2 - 1
    faces = np.c_[d * side, np.full(w, 15.0) * side, rng.uniform(0, 10, w)]
    return np.concatenate([ground, faces])[rng.permutation(n)].astype(np.float32)


def _kdtree_check(xyz, ids, k):
    """ids [n, k] against scipy's cKDTree wherever the k-th and (k+1)-th neighbours are clearly apart."""
    from scipy.spatial import cKDTree
    n = xyz.shape[0]
    dd, ii = cKDTree(xyz.astype(np.float64)).query(xyz.astype(np.float64), k + 2)
    selfcol = ii == np.arange(n)[:, None]
    ok = selfcol[:, 0] & ~selfcol[:, 1:].any(1)
    nd, ni = dd[:, 1:], ii[:, 1:]
    ok &= nd[:, k] - nd[:, k - 1] > 1e-9 * np.maximum(nd[:, k], 1e-30)
    assert ok.mean() > 0.99
    want = np.sort(ni[ok, :k], 1)
    got = np.sort(ids[ok], 1)
    assert np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,pair", [("room", 1000000, (10, 45)), ("falloff", 300000, (5, 20)),
                                         ("falloff", 300000, (10, 45))])
def test_large_clouds_exact(kind, n, pair):
    from superpoint_graph_b200.spg_geometry import compute_graph_nn_2
    k1, k2 = pair
    xyz = room_cloud(n, 1) if kind == "room" else falloff_cloud(n, 2)
    graph, target2 = compute_graph_nn_2(xyz, k1, k2)
    t2 = _np(target2).reshape(n, k2)
    dist = _np(graph["distances"]).reshape(n, k1)
    d2 = _d2_rows(xyz, t2)
    assert (d2[:, 1:] >= d2[:, :-1]).all()
    assert np.array_equal(dist.view(np.uint32), np.sqrt(d2[:, :k1]).astype(np.float32).view(np.uint32))
    assert np.array_equal(_np(graph["target"]).reshape(n, k1), t2[:, :k1])
    _kdtree_check(xyz, t2, k2)
    g2, tt2 = compute_graph_nn_2(xyz, k1, k2)
    assert torch.equal(tt2, target2) and torch.equal(g2["target"], graph["target"])
    assert torch.equal(g2["distances"].view(torch.int32), graph["distances"].view(torch.int32))


def _geof_check(xyz, target, k, got):
    want, lam = gref.compute_geof(xyz, target, k, return_eigenvalues=True)
    nan_w = np.isnan(want).any(1)
    assert np.array_equal(np.isnan(got).all(1), nan_w) and np.array_equal(np.isnan(got).any(1), nan_w)
    g, w, lam = got[~nan_w], want[~nan_w], lam[~nan_w]
    err = np.abs(g[:, :3].astype(np.float64) - w[:, :3])
    assert err.max() <= 1e-6, "linearity/planarity/scattering error %.3g" % err.max()
    gaps = np.minimum(lam[:, 0] - lam[:, 1], lam[:, 1] - lam[:, 2]) / lam[:, 0]
    sep = gaps >= 1e-3
    verr = np.abs(g[sep, 3].astype(np.float64) - w[sep, 3])
    assert verr.max() <= 1e-5, "verticality error %.3g" % verr.max()
    assert np.isfinite(g).all() and (g >= 0).all() and (g <= 1).all()
    return sep.mean()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,k", [("room", 200000, 45), ("falloff", 200000, 20)])
def test_geof_matches_float64_oracle(kind, n, k):
    from superpoint_graph_b200.spg_geometry import compute_geof, compute_graph_nn_2
    xyz = room_cloud(n, 3) if kind == "room" else falloff_cloud(n, 4)
    _, target2 = compute_graph_nn_2(xyz, 5, k)
    got = _np(compute_geof(xyz, target2, k))
    assert got.shape == (n, 4) and got.dtype == np.float32
    assert _geof_check(xyz, _np(target2), k, got) > 0.9
    again = _np(compute_geof(torch.from_numpy(xyz).cuda(), target2, k))
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    # numpy uint32 target, as the reference passes it
    host = _np(compute_geof(xyz, _np(target2).astype(np.uint32), k))
    assert np.array_equal(got.view(np.uint32), host.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("cloud", ["blob", "offset", "line", "lattice"])
def test_geof_golden_clouds(cloud):
    from superpoint_graph_b200.spg_geometry import compute_geof
    xyz = G[cloud + ".xyz"]
    target2 = _gold(cloud, (10, 45), "target2").astype(np.int64)
    got = _np(compute_geof(xyz, target2, 45))
    want = gref.compute_geof(xyz, target2, 45)
    nan_w = np.isnan(want).any(1)
    assert np.array_equal(np.isnan(got).any(1), nan_w) and np.array_equal(np.isnan(got).all(1), nan_w)
    assert np.abs(got[~nan_w, :3].astype(np.float64) - want[~nan_w, :3]).max() <= 1e-6
    assert (got[~nan_w] >= 0).all() and (got[~nan_w] <= 1).all()
    if cloud == "blob":  # rows whose 46 points all coincide
        assert nan_w.sum() >= 1


@pytest.mark.gpu
def test_edge_cases():
    from superpoint_graph_b200.spg_geometry import compute_geof, compute_graph_nn, compute_graph_nn_2
    rng = np.random.default_rng(5)
    # n = k + 1: every other vertex, by (d2, index)
    xyz = rng.normal(size=(46, 3)).astype(np.float32)
    graph, target2 = compute_graph_nn_2(xyz, 10, 45)
    ids, d2 = gref.knn(xyz, 45, extra=0)
    assert np.array_equal(_np(target2).reshape(46, 45), ids)
    # all points coincident: distances 0, the other ids in increasing order, NaN features
    xyz = np.full((50, 3), 3.5, np.float32)
    g = compute_graph_nn(xyz, 45)
    assert not _np(g["distances"]).any()
    want = np.array([[j for j in range(50) if j != i][:45] for i in range(50)])
    assert np.array_equal(_np(g["target"]).reshape(50, 45), want)
    assert torch.isnan(compute_geof(xyz, g["target"], 45)).all()
    # 10^4 m offset: the same distances as the reference's expression, ids as the oracle's
    base = room_cloud(20000, 6)
    off = (base + np.float32(1e4)).astype(np.float32)
    graph, target2 = compute_graph_nn_2(off, 10, 45)
    ids, d2 = gref.knn(off, 45, rows=np.arange(0, 20000, 10), extra=1)
    t2 = _np(target2).reshape(-1, 45)
    check_ids(off, t2, t2, np.full(20000, np.inf))  # no repeats, not self
    got_d2 = _d2_rows(off, t2)[::10]
    assert np.array_equal(got_d2, d2[:, :45])
    # CUDA and numpy inputs give the same bits
    gc, tc = compute_graph_nn_2(torch.from_numpy(off).cuda(), 10, 45)
    assert torch.equal(tc, target2) and torch.equal(gc["distances"].view(torch.int32),
                                                     graph["distances"].view(torch.int32))


@pytest.mark.gpu
def test_stray_points_far_from_the_cloud():
    """A room of 10^6 points plus a few stray points 10^2-10^3 m away: every stray point's neighbours are the oracle's,
    the sampled rows too, and the stray points cost no more than a bounded sweep of the cell table."""
    import time
    from superpoint_graph_b200.spg_geometry import compute_graph_nn_2
    base = room_cloud(1000000, 13)
    stray = np.array([[112.0, 4.0, 1.5], [-300.0, 250.0, 2.0], [6.0, 1000.0, 0.5], [5.0, 3.0, 800.0],
                      [-700.0, -700.0, -700.0]], np.float32)
    xyz = np.concatenate([base, stray]).astype(np.float32)
    n = xyz.shape[0]

    def timed(cloud):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = compute_graph_nn_2(cloud, 10, 45)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    timed(base)
    t_base, _ = timed(base)
    timed(xyz)
    t_stray, (graph, target2) = timed(xyz)
    rows = np.r_[np.arange(n - len(stray), n), np.random.default_rng(14).choice(n - len(stray), 120, replace=False)]
    ids, d2 = gref.knn(xyz, 45, rows=rows, extra=1, chunk=8)
    t2 = _np(target2).reshape(n, 45)[rows]
    dist = _np(graph["distances"]).reshape(n, 10)[rows]
    x = xyz.astype(np.float64)
    d = x[rows][:, None, :] - x[t2]
    got_d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert np.array_equal(got_d2, d2[:, :45])
    assert np.array_equal(dist.view(np.uint32), np.sqrt(d2[:, :10]).astype(np.float32).view(np.uint32))
    ext = np.concatenate([np.full((rows.size, 1), -1.0), d2], 1)
    untied = (ext[:, 1:-1] != ext[:, :-2]) & (ext[:, 1:-1] != ext[:, 2:])
    assert np.array_equal(t2[untied], ids[untied])
    # without the sweep, the 1 km stray points alone needed ~10^9 cell-column visits
    assert t_stray < t_base + 0.5, "stray points cost %.3f s over %.3f s" % (t_stray - t_base, t_base)


@pytest.mark.gpu
def test_device_validation():
    from superpoint_graph_b200.spg_geometry import compute_geof, compute_graph_nn
    xyz = G["room.xyz"].copy()
    xyz[17, 1] = np.nan
    with pytest.raises(ValueError, match="NaN or infinity"):
        compute_graph_nn(xyz, 10)
    xyz[17, 1] = np.inf
    with pytest.raises(ValueError, match="NaN or infinity"):
        compute_graph_nn(torch.from_numpy(xyz).cuda(), 10)
    xyz = G["room.xyz"]
    n = xyz.shape[0]
    bad = _gold("room", (10, 45), "target2").astype(np.int64)
    bad[123] = n
    with pytest.raises(IndexError):
        compute_geof(xyz, torch.from_numpy(bad).cuda(), 45)
    bad[123] = -1
    with pytest.raises(IndexError):
        compute_geof(xyz, bad, 45)


@pytest.mark.gpu
def test_local_geometry_feeds_the_partition_loader():
    """target2 of (5, 20) as `local_geometry` of the learned partition's batch builder: the batch equals the one
    built from the reference's sklearn lists bit for bit."""
    from superpoint_graph_b200.spg_geometry import compute_graph_nn_2
    from superpoint_graph_b200.spg_partition_loader import PartitionStore, load_batch
    xyz = G["room.xyz"]
    n = xyz.shape[0]
    graph, target2 = compute_graph_nn_2(xyz, 5, 20)
    gold_lg = _gold("room", (5, 20), "target2").astype(np.int64).reshape(n, 20)
    lg = _np(target2).reshape(n, 20)
    assert np.array_equal(lg, gold_lg)  # the room cloud has no ties
    rng = np.random.default_rng(8)
    src, tgt = _np(graph["source"]), _np(graph["target"])
    obj = np.arange(n) // 40
    labels = np.zeros((n, 14), np.uint32)
    labels[np.arange(n), 1 + obj % 13] = 1
    rest = (rng.integers(0, 256, (n, 3)).astype(np.float32), src, tgt, (obj[src] != obj[tgt]).astype(np.uint8))
    tail = (labels, obj, rng.normal(size=n).astype(np.float32), rng.normal(size=(n, 2)).astype(np.float32))
    args = SimpleNamespace(ver_value="ptn", k_nn_local=20, use_rgb=1, global_feat="eXYrgb", pc_augm_rot=0,
                           pc_augm_jitter=0, max_ver_train=0)
    out = []
    for geometry in (lg, gold_lg):
        st = PartitionStore().add("geo/room.h5", xyz, *rest, geometry, *tail).finalize("cuda")
        out.append(load_batch(st, ["geo/room.h5"], False, args))
    a, b = out
    for x, y in zip((a[1], a[2], a[3], a[4], a[5], a[6][0], a[6][1], a[7]),
                    (b[1], b[2], b[3], b[4], b[5], b[6][0], b[6][1], b[7])):
        assert x.dtype == y.dtype and torch.equal(x.view(torch.uint8) if x.dtype.is_floating_point else x,
                                                  y.view(torch.uint8) if y.dtype.is_floating_point else y)
