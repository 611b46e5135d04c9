"""Voxel pruning (superpoint_graph_b200.spg_prune, csrc/prune.cu).

CPU: the numpy oracle (oracle/prune_ref.py) against the reference's own outputs (prune.npz, from ply_c.cpp's `prune`
compiled by oracle/build_ref.py) bit for bit; the golden's coverage; host validation; the ABI symbols and kernel
names; the recipe's hash check (with a reference checkout).
GPU: every golden case bit for bit; 10^6 points against the oracle and the reference binary (when built); a voxel
of 2^24 + 3 points; a stray point that needs keys wider than 64 bits; one point per voxel; one point; the chunked
form; two runs bit-identical; the error cases; to_numpy's dtypes; prune -> compute_graph_nn_2 -> compute_sp_graph
against the same chain fed the oracle's cloud.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import build_ref, prune_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prune.npz")
_Z = np.load(GOLDEN, allow_pickle=False)
G = {k: _Z[k] for k in _Z.files}
META = json.loads(str(G["meta"]))
CASES = {c["name"]: c for c in META["cases"]}
OUTS = ("out_xyz", "out_rgb", "out_labels", "out_objects")


def _inputs(name):
    c = CASES[name]
    return (G[name + ".xyz"], c["voxel"], G[name + ".rgb"], G[name + ".labels"], G[name + ".objects"],
            c["n_labels"], c["n_objects"])


def _same(got, want):
    """Bitwise equality of the four outputs, shapes included (integer histograms compared by value)."""
    for k, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape, (k, a.shape, b.shape)
        if k == 0:
            assert np.array_equal(a.astype(np.float32).view(np.uint32), b.astype(np.float32).view(np.uint32)), k
        else:
            assert np.array_equal(a.astype(np.int64), b.astype(np.int64)), k


def _oracle(name):
    args = _inputs(name)
    rows = CASES[name]["chunk_rows"]
    return prune_ref.prune_chunked(*args, rows) if rows else prune_ref.prune(*args)


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_golden(name):
    _same(_oracle(name), [G["%s.%s" % (name, k)] for k in OUTS])


def test_golden_records_versions_and_covers_every_case():
    assert META["numpy"] and META["gxx"] and META["extract_sha256"] == build_ref.SHA256
    assert os.path.getsize(GOLDEN) < 1 << 20
    c = CASES
    assert c["room"]["n_labels"] > 0 and c["room"]["n_objects"] > 0
    assert c["labels_only"]["n_labels"] > 0 and c["labels_only"]["n_objects"] == 0
    assert c["neither"]["n_labels"] == 0 and c["neither"]["n_objects"] == 0
    assert c["objects_no_labels"]["n_labels"] == 0 and c["objects_no_labels"]["n_objects"] > 0
    assert G["objects_no_labels.out_objects"].shape[1] == c["objects_no_labels"]["n_objects"] + 1
    assert not G["objects_no_labels.out_objects"].any() and not G["neither.out_labels"].any()
    assert G["room.out_objects"].any() and G["room.out_labels"].any()
    assert np.abs(G["offset.xyz"]).max(1).min() > 9e3
    dup = G["dup_zero.xyz"]
    assert len(np.unique(dup, axis=0)) < len(dup)
    zeros = dup == 0
    assert (zeros & np.signbit(dup)).any() and (zeros & ~np.signbit(dup)).any()
    assert (dup.min(0) == 0).any()  # a zero of either sign is an axis minimum
    edge = G["boundary.xyz"]
    q = (edge - edge.min(0)) / np.float32(c["boundary"]["voxel"])
    assert ((q == np.floor(q)) & (q > 0)).any()
    ch = c["chunked"]
    assert 0 < ch["chunk_rows"] < ch["n"] and ch["n"] % ch["chunk_rows"] != 0


def test_host_validation():
    from superpoint_graph_b200.spg_prune import prune
    xyz, v, rgb, lab, obj, nl, no = _inputs("room")
    with pytest.raises(TypeError, match="float32"):
        prune(xyz.astype(np.float64), v, rgb, lab, obj, nl, no)
    with pytest.raises(TypeError, match="rgb"):
        prune(xyz, v, rgb.astype(np.int32), lab, obj, nl, no)
    with pytest.raises(TypeError, match="labels"):
        prune(xyz, v, rgb, lab.astype(np.float32), obj, nl, no)
    with pytest.raises(TypeError, match="objects"):
        prune(xyz, v, rgb, lab, obj.astype(np.float64), nl, no)
    with pytest.raises(ValueError, match="at least one point"):
        prune(xyz[:0], v, rgb[:0], lab[:0], obj[:0], nl, no)
    with pytest.raises(ValueError, match=r"\[n, 3\]"):
        prune(xyz[:, :2], v, rgb, lab, obj, nl, no)
    for bad in (0.0, -0.1, float("nan"), float("inf"), 1e-50):  # 1e-50 rounds to float32 0
        with pytest.raises(ValueError, match="voxel_size"):
            prune(xyz, bad, rgb, lab, obj, nl, no)
    with pytest.raises(ValueError, match="rgb has shape"):
        prune(xyz, v, rgb[:-1], lab, obj, nl, no)
    with pytest.raises(ValueError, match="labels has shape"):
        prune(xyz, v, rgb, lab[:-1], obj, nl, no)
    with pytest.raises(ValueError, match="objects has shape"):
        prune(xyz, v, rgb, lab, obj[:-1], nl, no)
    with pytest.raises(ValueError, match="n_labels"):
        prune(xyz, v, rgb, lab, obj, -1, no)
    with pytest.raises(ValueError, match="chunk_rows"):
        prune(xyz, v, rgb, lab, obj, nl, no, chunk_rows=-5)
    with pytest.raises(ValueError, match="chunks"):
        prune(np.zeros((70000, 3), np.float32), v, np.zeros((70000, 3), np.uint8), None, None, 0, 0, chunk_rows=1)


def test_abi_symbols_and_kernel_names():
    from superpoint_graph_b200 import _lib
    protos = _lib.protos()
    lib = _lib.lib()
    for n in ("spg_prune_workspace", "spg_prune_bounds", "spg_prune_voxels", "spg_prune_reduce"):
        assert n in protos, n
        assert getattr(lib, n) is not None
    kn = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("prune_bounds", "prune_keys", "prune_rows", "prune_reduce"):
        assert k in kn, k


def test_recipe_checks_the_extract_hash(tmp_path):
    ref = os.environ.get("SPG_REFERENCE")
    if not ref or not os.path.exists(os.path.join(ref, build_ref.SOURCE)):
        pytest.skip("no reference checkout (SPG_REFERENCE)")
    body = build_ref.extract(ref)
    assert body.startswith(build_ref.START) and body.rstrip().endswith("}")
    src = tmp_path / build_ref.SOURCE
    src.parent.mkdir(parents=True)
    src.write_text(open(os.path.join(ref, build_ref.SOURCE)).read().replace("acc_xyz.at(bin).at(0) + x",
                                                                            "acc_xyz.at(bin).at(0) - x", 1))
    with pytest.raises(RuntimeError, match="sha256"):
        build_ref.extract(str(tmp_path))
    src.write_text("int main() {}\n")
    with pytest.raises(RuntimeError, match="markers"):
        build_ref.extract(str(tmp_path))


# ------------------------------------------------------------------------------------------------- GPU
def _run(*args, **kw):
    from superpoint_graph_b200.spg_prune import prune
    out = prune(*args, **kw)
    for t in out:
        assert torch.is_tensor(t) and t.is_cuda
    assert [t.dtype for t in out] == [torch.float32, torch.uint8, torch.int64, torch.int64]
    return [t.cpu().numpy() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_on_device(name):
    got = _run(*_inputs(name), chunk_rows=CASES[name]["chunk_rows"])
    _same(got, [G["%s.%s" % (name, k)] for k in OUTS])


def _room_cloud(n, seed, n_labels=13, n_objects=50):
    rng = np.random.default_rng(seed)
    m = n // 4
    xyz = np.concatenate([np.c_[rng.uniform(0, 20, m), rng.uniform(0, 15, m), np.zeros(m)],
                          np.c_[rng.uniform(0, 20, m), np.zeros(m), rng.uniform(0, 4, m)],
                          np.c_[np.zeros(m), rng.uniform(0, 15, m), rng.uniform(0, 4, m)],
                          rng.uniform([2, 2, 0], [18, 13, 3], (n - 3 * m, 3))])
    xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)
    return (xyz, rng.integers(0, 256, (n, 3)).astype(np.uint8), rng.integers(0, n_labels + 1, n).astype(np.uint8),
            rng.integers(0, n_objects + 1, n).astype(np.uint32))


@pytest.mark.gpu
def test_million_points_against_oracle_and_reference_and_bitwise_reproducible():
    xyz, rgb, lab, obj = _room_cloud(1_000_000, 11)
    args = (xyz, 0.03, rgb, lab, obj, 13, 50)
    runs = [_run(*args) for _ in range(2)]
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    _same(runs[0], prune_ref.prune(*args))
    ref = build_ref.load_prune()
    if ref is not None:
        _same(runs[0], ref(*args))
    # the same cloud as tensors, labels as int64
    t = _run(torch.from_numpy(xyz).cuda(), 0.03, torch.from_numpy(rgb).cuda(),
             torch.from_numpy(lab.astype(np.int64)).cuda(), torch.from_numpy(obj.astype(np.int32)).cuda(), 13, 50)
    _same(t, runs[0])


@pytest.mark.gpu
def test_voxel_of_2_24_plus_3_points():
    n = (1 << 24) + 3
    rng = np.random.default_rng(5)
    xyz = rng.uniform(0.0, 0.5, (n, 3)).astype(np.float32)
    rgb = np.full((n, 3), 255, np.uint8)
    rgb[:, 1] = rng.integers(200, 256, n)
    rgb[:, 2] = 7
    lab = rng.integers(0, 3, n).astype(np.uint8)
    args = (xyz, 1.0, rgb, lab, np.zeros(1, np.uint8), 2, 0)
    got = _run(*args)
    assert got[0].shape == (1, 3)
    assert int(np.float32(n)) != n  # float(count) rounds
    want = prune_ref.prune(*args)
    _same(got, want)
    ref = build_ref.load_prune()
    if ref is not None:
        _same(got, ref(*args))


@pytest.mark.gpu
def test_stray_point_forces_wide_keys():
    xyz, rgb, lab, obj = _room_cloud(200_000, 3, 5, 7)
    xyz[1234] = (1e6, -1e6, 1e6)  # 25 bits per axis at 0.03, plus the room's: more than 64 bits of key
    args = (xyz, 0.03, rgb, lab, obj, 5, 7)
    b = prune_ref.bins(xyz, 0.03).max(0)
    assert sum(int(v).bit_length() for v in b) > 64
    _same(_run(*args), prune_ref.prune(*args))


@pytest.mark.gpu
def test_every_point_its_own_voxel_and_one_point():
    rng = np.random.default_rng(2)
    g = rng.permutation(np.stack(np.meshgrid(np.arange(40), np.arange(30), np.arange(20)), -1).reshape(-1, 3))
    xyz = (g * 0.5 + 0.25).astype(np.float32)
    rgb = rng.integers(0, 256, xyz.shape).astype(np.uint8)
    got = _run(xyz, 0.5, rgb, np.zeros(1, np.uint8), np.zeros(1, np.uint8), 0, 0)
    assert np.array_equal(got[0], xyz) and np.array_equal(got[1], rgb)
    _same(got, prune_ref.prune(xyz, 0.5, rgb, None, None, 0, 0))
    one = _run(xyz[7:8], 0.1, rgb[7:8], np.array([3], np.uint8), np.array([2], np.uint32), 4, 2)
    assert np.array_equal(one[0], xyz[7:8]) and np.array_equal(one[1], rgb[7:8])
    assert one[2].tolist() == [[0, 0, 0, 1, 0]] and one[3].tolist() == [[0, 0, 1]]


@pytest.mark.gpu
def test_chunked_form_is_the_stack_of_the_chunks():
    xyz, rgb, lab, obj = _room_cloud(300_000, 8, 8, 0)
    xyz[150_000:] += np.float32(5.0)  # the later chunks have their own minimum
    for rows in (70_000, 100_000, 300_000, 10 ** 7):
        args = (xyz, 0.05, rgb, lab, obj, 8, 0)
        _same(_run(*args, chunk_rows=rows), prune_ref.prune_chunked(*args, rows))


@pytest.mark.gpu
def test_error_cases():
    from superpoint_graph_b200.spg_prune import prune
    xyz, v, rgb, lab, obj, nl, no = _inputs("room")
    for bad in (np.nan, np.inf, -np.inf):
        x = xyz.copy()
        x[100, 1] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            prune(x, v, rgb, lab, obj, nl, no)
    x = xyz.copy()
    x[5] = (1e30, 0, 0)
    with pytest.raises(ValueError, match="2\\^32"):
        prune(x, v, rgb, lab, obj, nl, no)
    with pytest.raises(IndexError, match="labels"):
        prune(xyz, v, rgb, np.where(np.arange(len(lab)) == 9, nl + 1, lab), obj, nl, no)
    with pytest.raises(IndexError, match="labels"):
        prune(xyz, v, rgb, lab.astype(np.int64) - 1, obj, nl, no)
    with pytest.raises(IndexError, match="objects"):
        prune(xyz, v, rgb, lab, np.where(np.arange(len(obj)) == 3, no + 1, obj), nl, no)
    # objects are read only with labels: out-of-range objects are ignored when n_labels = 0, as in the reference
    got = _run(xyz, v, rgb, lab, obj + 1000, 0, no)
    assert not got[3].any() and got[3].shape[1] == no + 1


@pytest.mark.gpu
def test_to_numpy_has_the_reference_dtypes():
    from superpoint_graph_b200.spg_prune import prune, to_numpy
    out = to_numpy(prune(*_inputs("room")))
    assert [a.dtype for a in out] == [np.float32, np.uint8, np.uint32, np.uint32]
    for a, k in zip(out, OUTS):
        want = G["room." + k]
        assert a.dtype == want.dtype and np.array_equal(a.view(np.uint8), want.view(np.uint8)), k


@pytest.mark.gpu
def test_chain_prune_knn_sp_graph_matches_oracle_fed_chain():
    from scipy.spatial import Delaunay

    from superpoint_graph_b200.spg_geometry import compute_graph_nn_2
    from superpoint_graph_b200.spg_prune import prune
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph
    xyz, rgb, lab, obj = _room_cloud(80_000, 21, 8, 0)
    args = (xyz, 0.05, rgb, lab, obj, 8, 0)
    dev = prune(*args)
    ora = prune_ref.prune(*args)
    results = []
    for p_xyz, p_labels in ((dev[0], dev[2]), (ora[0], ora[2])):
        graph_nn, target_fea = compute_graph_nn_2(p_xyz, 10, 45)
        host = p_xyz.cpu().numpy() if torch.is_tensor(p_xyz) else p_xyz
        _, comp = np.unique(np.floor(host / np.float32(1.0)).astype(np.int64), axis=0, return_inverse=True)
        comp = comp.reshape(-1)  # a stand-in voxel partition for cut pursuit
        comps = np.split(np.argsort(comp, kind="stable"), np.cumsum(np.bincount(comp))[:-1])
        g = compute_sp_graph(p_xyz, 1.5, comp, comps, p_labels, 8, simplices=Delaunay(host).simplices)
        res = {k: v.cpu().numpy() for k, v in graph_nn.items() if torch.is_tensor(v)}
        res["target_fea"] = target_fea.cpu().numpy()
        res.update({k: v.cpu().numpy() for k, v in g.items() if torch.is_tensor(v)})
        results.append(res)
    a, b = results
    assert a.keys() == b.keys() and a["sp_labels"].shape[1] == 9
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
