"""The device Delaunay triangulation (superpoint_graph_b200/spg_delaunay.py, csrc/delaunay.cu) against its exact
oracle (oracle/delaunay_ref.py).

CPU: the oracle's certificate accepts scipy's triangulations of general-position clouds and rejects hand-broken
ones; the oracle's Bowyer-Watson equals scipy there and gives one answer on a permuted integer grid; host validation
of delaunay(); the ABI symbols and kernel names.
GPU: the device equals the oracle array for array on the golden sp_graph clouds, an integer grid, a cloud mixing
1e-30 and 1e3 coordinates and the 10^4-offset room; scipy as sets on general-position clouds; the certificate and
bitwise reproducibility on a 2 10^5-point room with exact planes; a store grown from a small capacity on two skew
lines; compute_sp_graph on device simplices against oracle/sp_graph_ref.py (test_sp_graph.py's bounds) and, in
general position, against compute_sp_graph on scipy's simplices; the workspace contract; prune -> ... -> delaunay -> superpoint graph on
device tensors.
"""
import os

import numpy as np
import pytest
import torch

from oracle import delaunay_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))


def _sets(s):
    return set(map(tuple, np.sort(np.asarray(s, dtype=np.int64), 1)))


def _oriented(xyz, s):
    """scipy's rows with their orientation made positive (flat rows stay flat)."""
    s = np.array(s, dtype=np.int64)
    for i, row in enumerate(s):
        if R.orient3d(*xyz[row]) < 0:
            s[i, [0, 1]] = s[i, [1, 0]]
    return s


def _uniform(n, seed):
    return np.random.default_rng(seed).uniform(0, 10, (n, 3)).astype(np.float32)


def _room(n, seed, noise=1e-3, exact_planes=False):
    rng = np.random.default_rng(seed)
    m = n // 5
    xyz = np.concatenate([np.c_[rng.uniform(0, 8, m), rng.uniform(0, 6, m), np.zeros(m)],
                          np.c_[rng.uniform(0, 8, m), np.full(m, 6.0), rng.uniform(0, 3, m)],
                          np.c_[np.zeros(m), rng.uniform(0, 6, m), rng.uniform(0, 3, m)],
                          np.c_[rng.uniform(0, 8, m), rng.uniform(0, 6, m), np.full(m, 3.0)],
                          rng.uniform([1, 1, 0], [7, 5, 2], (n - 4 * m, 3))])
    noisy = xyz + rng.normal(0, noise, xyz.shape)
    if exact_planes:  # the floor and one wall stay exactly planar
        noisy[:2 * m] = xyz[:2 * m]
    return noisy.astype(np.float32)


def _grid(k):
    return np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)


def _mixed(n, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, 3)) * np.where(rng.random((n, 3)) < 0.5, 1e-30, 1e3)
    return x.astype(np.float32)


def _skew_lines(m):
    t = np.linspace(-1, 1, m)
    a = np.c_[t, np.zeros(m), np.zeros(m)]
    b = np.c_[np.zeros(m), t, np.ones(m)]
    return np.concatenate([a, b]).astype(np.float32)


def _golden():
    d = np.load(os.path.join(HERE, "golden", "sp_graph.npz"))
    return {k: d[k + ".xyz"] for k in ("room", "lidar", "offset")}, d


# ------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("cloud", ["uniform", "room"])
def test_certificate_accepts_scipy_and_oracle_equals_it(cloud):
    from scipy.spatial import Delaunay
    xyz = _uniform(1500, 1) if cloud == "uniform" else _room(1500, 2)
    sc = Delaunay(xyz).simplices
    ok, why = R.certificate(xyz, _oriented(xyz, sc), return_reason=True)
    assert ok, why
    got = R.delaunay(xyz)
    assert _sets(got) == _sets(sc)
    assert R.certificate(xyz, got)


def test_certificate_rejects_broken_triangulations():
    xyz = _uniform(300, 3)
    good = R.delaunay(xyz)
    assert R.certificate(xyz, good)
    flipped = good.copy()
    flipped[0, [0, 1]] = flipped[0, [1, 0]]
    assert not R.certificate(xyz, flipped)
    assert not R.certificate(xyz, good[1:])
    # a non-Delaunay face: flip one interior face 2 -> 3 by hand
    faces = {}
    pair = None
    for t, row in enumerate(good):
        for i in range(4):
            key = tuple(sorted(np.delete(row, i)))
            if key in faces:
                pair = (faces[key], t, key)
                break
            faces[key] = t
        if pair:
            break
    t1, t2, f = pair
    a = [v for v in good[t1] if v not in f][0]
    b = [v for v in good[t2] if v not in f][0]
    new = [[a, b, f[0], f[1]], [a, b, f[1], f[2]], [a, b, f[2], f[0]]]
    rest = np.delete(good, [t1, t2], axis=0)
    flip = _oriented(xyz, np.concatenate([rest, new]))
    assert not R.certificate(xyz, flip)
    # a used duplicate
    dup = np.concatenate([xyz, xyz[:1]])
    used = good.copy()
    used[used == 0] = len(xyz)
    assert not R.certificate(dup, used)
    assert R.certificate(dup, good)


def test_perturbation_is_order_independent_on_a_grid():
    g = _grid(4)
    want = R.delaunay(g)
    assert R.certificate(g, want)
    for seed in range(3):
        p = np.random.default_rng(seed).permutation(len(g))
        got = R.delaunay(g[p])
        assert np.array_equal(R.canonical(p[got]), want)


def test_oracle_keeps_the_smallest_duplicate_and_zero_signs():
    xyz = _uniform(40, 4)
    xyz = np.concatenate([xyz, xyz[[3, 7]], [[-0.0, 1.0, 2.0], [0.0, 1.0, 2.0]]]).astype(np.float32)
    keep = R.unique_points(xyz)
    assert 40 not in keep and 41 not in keep and 42 in keep and 43 not in keep
    s = R.delaunay(xyz)
    assert set(np.unique(s)) == set(keep)
    assert R.certificate(xyz, s)


def test_host_validation():
    from superpoint_graph_b200.spg_delaunay import delaunay
    with pytest.raises(TypeError):
        delaunay(np.zeros((10, 3), np.float64))
    with pytest.raises(ValueError):
        delaunay(np.zeros((10, 2), np.float32))
    with pytest.raises(ValueError):
        delaunay(np.zeros((3, 3), np.float32))
    with pytest.raises(TypeError):
        delaunay(torch.zeros((10, 3), dtype=torch.float16))
    with pytest.raises(RuntimeError):
        delaunay(torch.zeros((10, 3), dtype=torch.float32))  # a CPU tensor: no CPU fallback
    with pytest.raises(ValueError, match="capacity"):
        delaunay(np.zeros((10, 3), np.float32), capacity=2 ** 29 + 1)


def test_abi_symbols_and_kernel_names():
    from superpoint_graph_b200 import _lib
    names = ["spg_dt_workspace", "spg_dt_setup", "spg_dt_init", "spg_dt_cavities", "spg_dt_commit", "spg_dt_grow",
             "spg_dt_output"]
    protos = _lib.protos()
    for n in names:
        assert n in protos
    lib = _lib.lib()
    kernels = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("dt_setup", "dt_init", "dt_nominate", "dt_grow", "dt_check", "dt_commit", "dt_relocate", "dt_output"):
        assert k in kernels


# ------------------------------------------------------------------------------------------------- GPU
def _dev(xyz, **kw):
    from superpoint_graph_b200.spg_delaunay import delaunay
    s = delaunay(torch.from_numpy(np.ascontiguousarray(xyz)).cuda(), **kw)
    assert s.is_cuda and s.dtype == torch.int32
    return s.cpu().numpy().astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["room", "lidar", "offset"])
def test_device_equals_oracle_on_golden_clouds(name):
    clouds, _ = _golden()
    xyz = clouds[name]
    assert np.array_equal(_dev(xyz), R.delaunay(xyz))


@pytest.mark.gpu
@pytest.mark.parametrize("cloud", ["grid", "mixed", "offset_room"])
def test_device_equals_oracle_on_degenerate_clouds(cloud):
    if cloud == "grid":
        xyz = _grid(10)
    elif cloud == "mixed":
        xyz = _mixed(400, 5)
    else:
        xyz = (_room(1200, 6, noise=0.0) + np.float32(1e4)).astype(np.float32)
    want = R.delaunay(xyz)
    got = _dev(xyz)
    assert np.array_equal(got, want)
    assert R.certificate(xyz, got)


@pytest.mark.gpu
@pytest.mark.parametrize("cloud", ["uniform", "room"])
def test_device_equals_scipy_in_general_position(cloud):
    from scipy.spatial import Delaunay
    xyz = _uniform(20000, 7) if cloud == "uniform" else _room(20000, 8)
    got = _dev(xyz)
    assert _sets(got) == _sets(Delaunay(xyz).simplices)


@pytest.mark.gpu
def test_certificate_and_reproducibility_on_a_room_with_exact_planes():
    xyz = _room(200000, 9, exact_planes=True)
    a = _dev(xyz)
    ok, why = R.certificate(xyz, a, return_reason=True)
    assert ok, why
    assert np.array_equal(a, _dev(xyz))


@pytest.mark.gpu
def test_store_grows_on_two_skew_lines():
    from superpoint_graph_b200.spg_delaunay import last_stats
    xyz = _skew_lines(300)
    got = _dev(xyz, capacity=1024)
    st = last_stats()
    assert st["grows"] > 0 and st["capacity"] > 1024
    assert len(got) > 80000
    assert np.array_equal(got, R.delaunay(xyz))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["room", "lidar", "offset"])
def test_sp_graph_on_device_simplices_equals_the_oracle(name):
    """compute_sp_graph given delaunay(xyz) against oracle/sp_graph_ref.py given the same simplices, within
    test_sp_graph.py's bounds."""
    import test_sp_graph as T
    from oracle import sp_graph_ref as sref
    from superpoint_graph_b200.spg_delaunay import delaunay
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, comp, _ = T._cloud(name)
    labels = T._labels(name, "1d")
    d_max = float(T.META["d_max"][name])
    tets = delaunay(torch.from_numpy(xyz).cuda())
    s = tets.cpu().numpy()
    got = T._np(compute_sp_graph(xyz, d_max, comp, T._components(comp), labels, T.N_LABELS, simplices=tets))
    ora = sref.compute_sp_graph(xyz, d_max, comp, labels, T.N_LABELS, s)
    assert got["source"].shape[0] > 0
    T._check_against(got, ora, ora["u"], T._delta_max(xyz, comp, s, d_max, ora), 1e-6, 1e-6)
    T._check_ratios(got)


@pytest.mark.gpu
def test_sp_graph_on_device_simplices_equals_scipy_in_general_position():
    from scipy.spatial import Delaunay

    import test_sp_graph as T
    from superpoint_graph_b200.spg_delaunay import delaunay
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz = _uniform(5000, 13)
    _, comp = np.unique(np.floor(xyz / 2.5).astype(np.int64), axis=0, return_inverse=True)
    comp = comp.reshape(-1)
    x = torch.from_numpy(xyz).cuda()
    tets = delaunay(x)
    sc = Delaunay(xyz).simplices
    assert _sets(tets.cpu().numpy()) == _sets(sc)
    a = T._np(compute_sp_graph(x, 1.0, comp, T._components(comp), [], 0, simplices=tets))
    b = T._np(compute_sp_graph(x, 1.0, comp, T._components(comp), [], 0, simplices=sc))
    for k in a:
        if k != "is_nn":
            assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
def test_workspace_contract():
    from superpoint_graph_b200 import _lib, ops
    xyz = torch.from_numpy(_uniform(500, 10)).cuda()
    n, cap = 500, 4096
    nbytes = torch.zeros(1, dtype=torch.int64)
    _lib.call("spg_dt_workspace", n, cap, nbytes)
    need = int(nbytes[0])
    assert need % 256 == 0
    big = torch.full((need + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
    ws = big[:need]
    out = torch.zeros(8, dtype=torch.int64)
    s = _lib.current_stream()
    _lib.call("spg_dt_setup", xyz, n, cap, ws, need, out, s)
    _lib.call("spg_dt_init", n, cap, ws, need, out, s)
    while True:
        _lib.call("spg_dt_cavities", n, cap, ws, need, -1, out, s)
        if int(out[0]) == 0:
            break
        _lib.call("spg_dt_commit", n, cap, ws, need, out, s)
        assert int(out[0]) == 0
    cnt = torch.zeros(1, dtype=torch.int64)
    _lib.call("spg_dt_output", n, cap, ws, need, cnt, None, s)
    sim = torch.empty((int(cnt[0]), 4), dtype=torch.int32, device="cuda")
    _lib.call("spg_dt_output", n, cap, ws, need, cnt, sim, s)
    torch.cuda.synchronize()
    assert bool((big[need:] == 0xA5).all())
    assert np.array_equal(sim.cpu().numpy().astype(np.int64), _dev(xyz.cpu().numpy()))
    mis = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="misaligned"):
        _lib.call("spg_dt_setup", xyz, n, cap, mis[16:], need, out, s)
    with pytest.raises(RuntimeError, match="bad argument"):
        _lib.call("spg_dt_setup", xyz, n, cap, mis, need - 1, out, s)
    del ops


@pytest.mark.gpu
def test_device_validation():
    from superpoint_graph_b200.spg_delaunay import delaunay
    x = _uniform(100, 11)
    x[5, 1] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        delaunay(torch.from_numpy(x).cuda())
    flat = _uniform(100, 12)
    flat[:, 2] = 1.0
    with pytest.raises(ValueError, match="affinely independent"):
        delaunay(torch.from_numpy(flat).cuda())
    same = np.tile(np.float32([[1, 2, 3]]), (10, 1))
    with pytest.raises(ValueError, match="affinely independent"):
        delaunay(same)


@pytest.mark.gpu
def test_prune_geometry_cut_pursuit_delaunay_sp_graph_on_device():
    """prune -> compute_graph_nn_2 -> compute_geof -> cutpursuit -> delaunay -> compute_sp_graph, device tensors."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    from superpoint_graph_b200 import spg_geometry, spg_prune, spg_sp_graph
    from superpoint_graph_b200.spg_delaunay import delaunay
    rng = np.random.default_rng(7)
    m = 6000
    xyz = np.concatenate([np.c_[rng.uniform(0, 6, m), rng.uniform(0, 5, m), np.zeros(m)],
                          np.c_[np.zeros(m), rng.uniform(0, 5, m), rng.uniform(0, 3, m)],
                          np.c_[rng.uniform(0, 6, m), np.zeros(m), rng.uniform(0, 3, m)]])
    xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)
    rgb = np.repeat(np.array([[200, 30, 30], [30, 200, 30], [30, 30, 200]], np.uint8), m, 0)
    pruned = spg_prune.prune(torch.from_numpy(xyz).cuda(), 0.05, torch.from_numpy(rgb).cuda(), None, None, 0, 0)
    xyz_p, rgb_p = pruned[0], pruned[1]
    graph, target2 = spg_geometry.compute_graph_nn_2(xyz_p, 10, 20)
    geof = spg_geometry.compute_geof(xyz_p, target2, 20)
    geof[:, 3] *= 2
    features = torch.cat([geof, rgb_p.float() / 255], 1).contiguous()
    d = graph["distances"]
    w = (1 / (1 + d / d.mean())).float()
    comps, inc = cp.cutpursuit(features, graph["source"], graph["target"], w, 0.1)
    simplices = delaunay(xyz_p)
    assert simplices.is_cuda
    g = spg_sp_graph.compute_sp_graph(xyz_p, 1.0, inc, comps, [], 0, simplices=simplices)
    assert int(g["sp_point_count"].sum()) == xyz_p.shape[0]
    assert R.certificate(xyz_p.cpu().numpy(), simplices.cpu().numpy())
