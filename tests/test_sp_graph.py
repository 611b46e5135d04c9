"""The superpoint graph of a partition (superpoint_graph_b200.spg_sp_graph, csrc/sp_graph.cu).

CPU: the vectorised oracle (oracle/sp_graph_ref.py) against the reference's own graphs (sp_graph.npz, from the
unmodified partition/graphs.py): integers and centroids bit for bit, the other floats within tolerance; the golden's
coverage; host validation; the ABI symbols and kernel names.
GPU: every golden cloud x labels mode x d_max with the stored simplices; simplices=None; a seeded cloud of 2 10^5
points against the oracle; two runs bit-identical; the error cases; to_numpy's dtypes.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import sp_graph_ref as sref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sp_graph.npz")
_Z = np.load(GOLDEN, allow_pickle=False)
G = {k: _Z[k] for k in _Z.files}
META = json.loads(str(G["meta"]))
N_LABELS = META["n_labels"]
CLOUDS = [c["name"] for c in META["clouds"]]
MODES = META["label_modes"]
CASES = [(c, m, d) for c in CLOUDS for m in MODES for d in (0.0, META["d_max"][c])]
EXACT = ("source", "target", "sp_point_count", "sp_centroids", "se_delta_centroid", "se_point_count_ratio")


def _cloud(name):
    return G[name + ".xyz"], G[name + ".in_component"], G[name + ".simplices"].astype(np.int32)


def _labels(name, mode):
    return [] if mode == "none" else G["%s.labels.%s" % (name, mode)]


def _gold(name, d_max, key):
    return G["%s.%g.%s" % (name, d_max, key)]


def _components(comp):
    order = np.argsort(comp, kind="stable")
    return np.split(order, np.cumsum(np.bincount(comp))[:-1])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------- CPU
def test_golden_records_versions_and_covers_every_case():
    assert META["numpy"] and META["scipy"]
    assert os.path.getsize(GOLDEN) < 1 << 20
    assert set(MODES) == {"none", "1d", "hist"}
    assert any(np.abs(G[c + ".xyz"]).min() > 5e3 for c in CLOUDS)  # the cloud offset by 10^4 m
    seen = {"u1": 0, "u2": 0, "dup": 0, "collinear": 0, "single_pair": 0, "cut": 0}
    for c in CLOUDS:
        xyz, comp, s = _cloud(c)
        sp = sref.superpoints(xyz, comp, [], N_LABELS)
        u, m = sp["u"], sp["sp_point_count"][:, 0]
        seen["u1"] += int((u == 1).sum())
        seen["u2"] += int((u == 2).sum())
        seen["dup"] += int(((m > u) & (u >= 3)).sum())
        seen["collinear"] += int(((u >= 3) & (sp["sp_surface"][:, 0] < 1e-4)).sum())
        seen["single_pair"] += int((sref.superedges(xyz, comp, s, 0.0, sp)["pairs"] == 1).sum())
        d = META["d_max"][c]
        seen["cut"] += int(len(sref.vertex_pairs(xyz, comp, s, d)[0]) < len(sref.vertex_pairs(xyz, comp, s, 0.0)[0]))
        assert G[c + ".labels.1d"].ndim == 1 and (G[c + ".labels.1d"] > N_LABELS).any()
        assert G[c + ".labels.hist"].shape[1] == N_LABELS + 1
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("cloud,mode,d_max", CASES)
def test_oracle_reproduces_golden(cloud, mode, d_max):
    xyz, comp, s = _cloud(cloud)
    g = sref.compute_sp_graph(xyz, d_max, comp, _labels(cloud, mode), N_LABELS, s)
    for k in EXACT:
        want = _gold(cloud, d_max, k)
        assert np.array_equal(np.asarray(g[k]).astype(want.dtype), want), k
    if mode == "none":
        assert g["sp_labels"] == []
    else:
        assert np.array_equal(g["sp_labels"], G["%s.sp_labels.%s" % (cloud, mode)])
    u = g["u"]
    assert np.array_equal(_bits(g["sp_length"][u <= 2]), _bits(_gold(cloud, d_max, "sp_length")[u <= 2]))
    for k in ("sp_length", "sp_surface", "sp_volume"):
        np.testing.assert_allclose(g[k][u >= 3], _gold(cloud, d_max, k)[u >= 3], rtol=1e-5, atol=0)
    scale = np.abs(_delta_max(xyz, comp, s, d_max, g))
    for k in ("se_delta_mean", "se_delta_std", "se_delta_norm"):
        assert (np.abs(g[k] - _gold(cloud, d_max, k)) <= 1e-4 * scale[:, None]).all(), k


def _delta_max(xyz, comp, s, d_max, g):
    """Per superedge the largest |delta| component over its pairs (the scale of the delta statistics)."""
    a, b = sref.vertex_pairs(xyz, comp, s, d_max)
    n_com = g["sp_centroids"].shape[0]
    key = comp.astype(np.int64)[a] * n_com + comp.astype(np.int64)[b]
    order = np.argsort(key, kind="stable")
    d = np.abs(xyz[a[order]].astype(np.float64) - xyz[b[order]]).max(1)
    _, start = np.unique(key[order], return_index=True)
    return np.maximum.reduceat(d, start) if d.size else d


def test_host_validation():
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, s = _cloud("room")
    comps = _components(comp)
    with pytest.raises(TypeError, match="float32"):
        compute_sp_graph(xyz.astype(np.float64), 0, comp, comps, [], N_LABELS, s)
    with pytest.raises(TypeError, match="in_component"):
        compute_sp_graph(xyz, 0, comp.astype(np.float32), comps, [], N_LABELS, s)
    with pytest.raises(ValueError, match="in_component has shape"):
        compute_sp_graph(xyz, 0, comp[:-1], comps, [], N_LABELS, s)
    with pytest.raises(ValueError, match=r"n_labels \+ 1"):
        compute_sp_graph(xyz, 0, comp, comps, G["room.labels.hist"][:, :3], N_LABELS, s)
    with pytest.raises(TypeError, match="labels"):
        compute_sp_graph(xyz, 0, comp, comps, G["room.labels.1d"].astype(np.float32), N_LABELS, s)
    with pytest.raises(ValueError, match=r"\[n, 3\]"):
        compute_sp_graph(xyz[:, :2], 0, comp, comps, [], N_LABELS, s)
    with pytest.raises(ValueError, match="at least one point"):
        compute_sp_graph(xyz[:0], 0, comp[:0], [], [], N_LABELS, s)


def test_abi_symbols_and_kernel_names():
    from superpoint_graph_b200 import _lib
    names = ["spg_sp_scan", "spg_sp_points_workspace", "spg_sp_points", "spg_sp_edges_workspace",
             "spg_sp_edges_count", "spg_sp_edges_build", "spg_sp_edges_features"]
    protos = _lib.protos()
    lib = _lib.lib()
    for n in names:
        assert n in protos, n
        assert getattr(lib, n) is not None
    kn = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("sp_scan", "sp_sort_keys", "sp_points", "sp_tets", "sp_pairs", "sp_edges"):
        assert k in kn, k


# ------------------------------------------------------------------------------------------------- GPU
def _np(g):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in g.items()}


def _check_against(got, want, u, scale, rtol_sp, rtol_delta):
    for k in EXACT:
        assert np.array_equal(got[k].astype(np.asarray(want[k]).dtype), want[k]), k
    assert np.array_equal(_bits(got["sp_length"][u <= 2]), _bits(want["sp_length"][u <= 2]))
    for k in ("sp_length", "sp_surface", "sp_volume"):
        np.testing.assert_allclose(got[k][u >= 3], want[k][u >= 3], rtol=rtol_sp, atol=0, err_msg=k)
    for k in ("se_delta_mean", "se_delta_std", "se_delta_norm"):
        assert (np.abs(got[k] - want[k]) <= rtol_delta * scale[:, None]).all(), k


def _check_ratios(got):
    src, tgt = got["source"][:, 0], got["target"][:, 0]
    for k, f in (("se_length_ratio", "sp_length"), ("se_surface_ratio", "sp_surface"),
                 ("se_volume_ratio", "sp_volume")):
        want = got[f][src] / (got[f][tgt] + np.float32(1e-6))
        assert want.dtype == np.float32 and np.array_equal(_bits(got[k]), _bits(want)), k


@pytest.mark.gpu
@pytest.mark.parametrize("cloud,mode,d_max", CASES)
def test_golden_on_device(cloud, mode, d_max):
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, s = _cloud(cloud)
    labels = _labels(cloud, mode)
    g = compute_sp_graph(xyz, d_max, comp, _components(comp), labels, N_LABELS, simplices=s)
    for k, v in g.items():
        if k != "is_nn" and not (k == "sp_labels" and mode == "none"):
            assert torch.is_tensor(v) and v.is_cuda, k
    assert g["is_nn"] is False
    assert g["source"].dtype == torch.int64 and g["sp_point_count"].dtype == torch.int64
    assert g["sp_centroids"].dtype == torch.float32 and g["se_delta_mean"].dtype == torch.float32
    got = _np(g)
    ora = sref.compute_sp_graph(xyz, d_max, comp, labels, N_LABELS, s)
    u = ora["u"]
    scale = _delta_max(xyz, comp, s, d_max, ora)
    want = {k: _gold(cloud, d_max, k) for k in EXACT + ("sp_length", "sp_surface", "sp_volume", "se_delta_mean",
                                                        "se_delta_std", "se_delta_norm")}
    assert got["source"].shape == want["source"].shape  # the superedge count
    _check_against(got, want, u, scale, 1e-5, 1e-4)
    _check_against(got, ora, u, scale, 1e-6, 1e-6)
    _check_ratios(got)
    if mode == "none":
        assert got["sp_labels"] == []
    else:
        assert got["sp_labels"].dtype == np.int64
        assert np.array_equal(got["sp_labels"], G["%s.sp_labels.%s" % (cloud, mode)])


@pytest.mark.gpu
def test_simplices_none_is_scipy_delaunay():
    from scipy.spatial import Delaunay

    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, _ = _cloud("lidar")
    labels = G["lidar.labels.1d"]
    a = _np(compute_sp_graph(xyz, 1.0, comp, _components(comp), labels, N_LABELS))
    b = _np(compute_sp_graph(torch.from_numpy(xyz).cuda(), 1.0, torch.from_numpy(comp.astype(np.int64)).cuda(),
                             _components(comp), labels, N_LABELS, simplices=Delaunay(xyz).simplices))
    for k in a:
        if k != "is_nn":
            assert np.array_equal(a[k], b[k]), k


def _big_cloud(n, seed):
    rng = np.random.default_rng(seed)
    m = n // 4
    xyz = np.concatenate([np.c_[rng.uniform(0, 20, m), rng.uniform(0, 15, m), np.zeros(m)],
                          np.c_[rng.uniform(0, 20, m), np.zeros(m), rng.uniform(0, 4, m)],
                          np.c_[np.zeros(m), rng.uniform(0, 15, m), rng.uniform(0, 4, m)],
                          rng.uniform([2, 2, 0], [18, 13, 3], (n - 3 * m, 3))])
    xyz = (xyz + rng.normal(0, 0.005, xyz.shape)).astype(np.float32)  # exactly coplanar sets slow qhull down badly
    xyz[rng.choice(n, n // 100)] = xyz[rng.choice(n, n // 100)]  # duplicated points
    vox = np.floor(xyz / 1.0).astype(np.int64)
    _, comp = np.unique(vox, axis=0, return_inverse=True)
    return xyz, comp.reshape(-1).astype(np.uint32), rng.integers(0, 9, n).astype(np.uint8)


@pytest.mark.gpu
def test_large_cloud_against_oracle_and_bitwise_reproducible():
    from scipy.spatial import Delaunay

    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, labels = _big_cloud(200_000, 7)
    s = Delaunay(xyz).simplices
    for d_max in (0.0, 0.5):
        runs = [_np(compute_sp_graph(xyz, d_max, comp, _components(comp), labels, 8, simplices=s)) for _ in range(2)]
        for k in runs[0]:
            if k != "is_nn":
                assert np.array_equal(np.asarray(runs[0][k]).view(np.uint8), np.asarray(runs[1][k]).view(np.uint8)), k
        ora = sref.compute_sp_graph(xyz, d_max, comp, labels, 8, s)
        _check_against(runs[0], ora, ora["u"], _delta_max(xyz, comp, s, d_max, ora), 1e-6, 1e-6)
        _check_ratios(runs[0])
        assert np.array_equal(runs[0]["sp_labels"], ora["sp_labels"])


@pytest.mark.gpu
def test_error_cases_and_single_component():
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, s = _cloud("room")
    comps = _components(comp)
    bad = s.copy()
    bad[5, 2] = xyz.shape[0]
    with pytest.raises(IndexError, match="simplices"):
        compute_sp_graph(xyz, 0, comp, comps, [], N_LABELS, simplices=bad)
    gap = comp.copy()
    gap[gap == 3] = 4  # component 3 empty
    with pytest.raises(ValueError, match="holds no point"):
        compute_sp_graph(xyz, 0, gap, comps, [], N_LABELS, simplices=s)
    nan = xyz.copy()
    nan[10, 1] = np.nan
    with pytest.raises(ValueError, match="NaN or infinity"):
        compute_sp_graph(nan, 0, comp, comps, [], N_LABELS, simplices=s)
    one = np.zeros_like(comp)
    g = _np(compute_sp_graph(xyz, 0, one, [np.arange(len(comp))], G["room.labels.hist"], N_LABELS, simplices=s))
    assert g["source"].shape == (0, 1) and g["se_delta_mean"].shape == (0, 3)
    ora = sref.superpoints(xyz, one, G["room.labels.hist"], N_LABELS)
    for k in ("sp_centroids", "sp_point_count", "sp_labels"):
        assert np.array_equal(g[k], ora[k]), k


@pytest.mark.gpu
def test_to_numpy_has_write_spg_dtypes():
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph, to_numpy
    xyz, comp, s = _cloud("offset")
    g = to_numpy(compute_sp_graph(xyz, 0.3, comp, _components(comp), G["offset.labels.hist"], N_LABELS,
                                  simplices=s))
    want = {"source": np.uint32, "target": np.uint32, "sp_labels": np.uint32, "sp_point_count": np.uint64}
    for k, v in g.items():
        if k == "is_nn":
            continue
        assert isinstance(v, np.ndarray), k
        assert v.dtype == want.get(k, np.float32), k
    assert np.array_equal(g["source"], _gold("offset", 0.3, "source"))
    assert np.array_equal(g["sp_point_count"], _gold("offset", 0.3, "sp_point_count"))
    g = to_numpy(compute_sp_graph(xyz, 0.3, comp, _components(comp), [], N_LABELS, simplices=s))
    assert g["sp_labels"] == []
