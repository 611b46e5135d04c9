"""The learned partition's graph structure on the device (superpoint_graph_b200/spg_structure.py, csrc/structure.cu)
against tests/golden/structure.npz (the reference's own graph_processing.py:144-190 on three clouds) and
oracle/structure_ref.py.

The k-NN lists of the reference (sklearn's kd-tree) and of the device agree wherever distances are untied
(test_geometry.py); exact duplicates tie.  So the device is compared with the oracle fed the device's own neighbour
lists and the golden simplices, and the oracle fed the golden's neighbour lists is compared with the golden, on the
CPU: together the device is the reference's formula bit for bit."""
import ctypes
import json
import os
import types

import numpy as np
import pytest

from oracle import structure_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "structure.npz")
G = np.load(GOLDEN)
META = json.loads(str(G["meta"]))
CASES = [c["case"] for c in META["cases"]]
K_ADJ, K_LOCAL = META["k_nn_adj"], META["k_nn_local"]


def _case(case):
    c = next(c for c in META["cases"] if c["case"] == case)
    cloud = c["cloud"]
    return c, {k: G["%s.%s" % (cloud, k)] for k in ("xyz", "rgb", "labels", "objects", "neighbors")}, \
        (G[cloud + ".simplices"] if c["use_voronoi"] > 0 else None)


def _oracle(case, neighbors, simplices=None, plane=None):
    c, d, simp = _case(case)
    labels = None if c["dataset"] == "sema3d" else d["labels"]
    return structure_ref.structure(c["dataset"], d["xyz"], labels, d["objects"], neighbors, K_ADJ, K_LOCAL,
                                   c["use_voronoi"], simp if simplices is None else simplices, True, plane)


# ------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_golden(case):
    c, d, _ = _case(case)
    plane = None
    if c["plane_model"]:
        p = G[case + ".plane"]
        plane = (p[:2], p[2])
    got = _oracle(case, d["neighbors"], plane=plane)
    for k in ("source", "target", "is_transition", "labels", "objects", "xyn"):
        want = G["%s.%s" % (case, k)]
        assert np.array_equal(np.asarray(got[k]).astype(want.dtype), want), (case, k)
        assert np.asarray(got[k]).shape == want.shape, (case, k)
    if c["use_voronoi"] > 0:
        assert got["distances"].dtype == np.float32
        assert np.array_equal(got["distances"], G[case + ".distances"])
    assert np.array_equal(got["target_local_geometry"], d["neighbors"].astype(np.int64))
    want = G[case + ".elevation"]
    if plane is None:
        assert np.array_equal(got["elevation"], want)
    else:  # the reference's float32 predict against fp64 rounded once
        assert np.abs(got["elevation"].astype(np.float64) - want).max() <= 2 * np.spacing(np.abs(want).max())


def test_oracle_threshold_is_float32_and_distances_are_squared():
    xyz = np.array([[0, 0, 0], [0.3, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    simp = np.array([[0, 1, 2, 3]])
    nb = np.array([[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]])
    d2 = np.float32(0.3) * np.float32(0.3)
    s, t, dist = structure_ref.voronoi_graph(xyz, simp, nb, 1, float(d2) + 1e-12)  # float32(v) == d2: not kept
    assert dist.size == 0
    s, t, dist = structure_ref.voronoi_graph(xyz, simp, nb, 1, float(np.nextafter(d2, np.float32(1))))
    assert np.array_equal(dist, [d2]) and dist.dtype == np.float32
    assert np.all(np.diff(t * 4 + s) > 0)


def test_oracle_connected_comp_reads_signed_chars():
    src, tgt = np.array([0, 1, 2, 3]), np.array([1, 2, 3, 4])
    comps, inc = structure_ref.connected_comp(5, src, tgt, np.array([2, 127, 128, 255], np.uint8))
    assert list(inc) == [0, 0, 0, 1, 2] and [list(c) for c in comps] == [[0, 1, 2], [3], [4]]


def test_host_validation():
    from superpoint_graph_b200 import spg_structure as st

    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=10, use_voronoi=0.0, compute_geof=0, plane_model=0)
    xyz = np.zeros((20, 3), np.float32)
    with pytest.raises(ValueError, match="unknown data set"):
        st.compute_structure(args, "custom_dataset", xyz, xyz, None)
    with pytest.raises(NotImplementedError, match="cutpursuit2"):
        st.compute_structure(args, "sema3d", xyz, xyz, np.zeros((20, 9), np.uint32))
    with pytest.raises(ValueError, match="s3dis needs objects"):
        st.compute_structure(args, "s3dis", xyz, xyz, np.zeros((20, 9), np.uint32))
    with pytest.raises(ValueError, match="args has no field"):
        st.compute_structure(types.SimpleNamespace(), "s3dis", xyz, xyz, None)
    e = np.zeros(3, np.int64)
    with pytest.raises(NotImplementedError, match="cutoff > 0"):
        st.connected_comp(4, e, e, np.ones(3, np.uint8), 2)
    with pytest.raises(ValueError, match="cutoff"):
        st.connected_comp(4, e, e, np.ones(3, np.uint8), -1)
    with pytest.raises(ValueError, match="n_ver"):
        st.connected_comp(0, e, e, np.ones(3, np.uint8))
    with pytest.raises(TypeError, match="active_edg"):
        st.connected_comp(4, e, e, np.ones(3, np.int32))
    from superpoint_graph_b200 import spg_geometry

    with pytest.raises(NotImplementedError, match="spg_structure"):
        spg_geometry.compute_graph_nn_2(xyz, 5, 10, voronoi=0.5)


def test_abi_symbols_and_kernel_names():
    from superpoint_graph_b200 import _lib

    names = ("spg_st_vor_blocks", "spg_st_vor_workspace", "spg_st_vor_count", "spg_st_vor_build", "spg_st_cc_workspace",
             "spg_st_cc", "spg_st_argmax", "spg_st_transitions", "spg_st_select_workspace", "spg_st_select",
             "spg_st_gather_rows", "spg_st_points")
    protos = _lib.protos()
    for nm in names:
        assert nm in protos, nm
    lib = _lib.lib()
    kernels = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("st_vor", "st_cc", "st_labels", "st_select", "st_points"):
        assert k in kernels


# ------------------------------------------------------------------------------------------ GPU
def _np(t):
    return t.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("cloud", ["room", "scan", "dup"])
def test_voronoi_graph_from_golden_simplices(cloud):
    from superpoint_graph_b200 import spg_structure as st

    c = next(c for c in META["cases"] if c["cloud"] == cloud and c["use_voronoi"] > 0)
    xyz, simp, case = G[cloud + ".xyz"], G[cloud + ".simplices"], c["case"]
    graph, target2 = st.compute_graph_nn_2(xyz, K_ADJ, K_LOCAL, voronoi=c["use_voronoi"], simplices=simp)
    nb = _np(target2).reshape(len(xyz), K_LOCAL)
    assert graph["source"].dtype == graph["target"].dtype == target2.dtype
    assert str(graph["source"].dtype) == "torch.int64"
    s, t, d = structure_ref.voronoi_graph(xyz, simp, nb, K_ADJ, c["use_voronoi"])
    assert np.array_equal(_np(graph["source"]), s) and np.array_equal(_np(graph["target"]), t)
    assert np.array_equal(_np(graph["distances"]), G[case + ".distances"])
    gold_nb = G[cloud + ".neighbors"].astype(np.int64)
    agree = (nb == gold_nb).all(1)
    if cloud != "dup":  # no exact duplicates: every list untied, the golden's own edges
        assert agree.all()
        assert np.array_equal(_np(graph["source"]), G[case + ".source"].astype(np.int64))
        assert np.array_equal(_np(graph["target"]), G[case + ".target"].astype(np.int64))
    else:
        assert agree.mean() > 0.5


def _vor_properties(xyz, simp, graph, nb, voronoi):
    src, tgt = _np(graph["source"]), _np(graph["target"])
    n = len(xyz)
    key = tgt * n + src
    assert np.all(np.diff(key) > 0)
    have = set(key.tolist())
    knn = set((nb[:, :K_ADJ].reshape(-1) * n + np.repeat(np.arange(n), K_ADJ)).tolist())
    assert knn <= have
    pairs = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
    cs = np.concatenate([simp[:, a] for a, _ in pairs]).astype(np.int64)
    ct = np.concatenate([simp[:, b] for _, b in pairs]).astype(np.int64)
    dd = xyz[cs] - xyz[ct]
    d2 = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
    keep = d2 < np.float32(voronoi)
    assert set((ct[keep] * n + cs[keep]).tolist()) <= have
    extra = have - knn - set((ct[keep] * n + cs[keep]).tolist())
    assert not extra
    assert graph["distances"].shape[0] == int(keep.sum())


@pytest.mark.gpu
def test_voronoi_graph_from_device_simplices_and_threshold():
    import torch

    from superpoint_graph_b200 import spg_delaunay
    from superpoint_graph_b200 import spg_structure as st

    for cloud, vor in (("room", 0.05), ("scan", 1.0), ("dup", 0.05)):
        xyz = G[cloud + ".xyz"]
        graph, target2 = st.compute_graph_nn_2(xyz, K_ADJ, K_LOCAL, voronoi=vor)
        simp = spg_delaunay.to_numpy(spg_delaunay.delaunay(torch.from_numpy(xyz).cuda()))
        nb = _np(target2).reshape(len(xyz), K_LOCAL)
        s, t, d = structure_ref.voronoi_graph(xyz, simp, nb, K_ADJ, vor)
        assert np.array_equal(_np(graph["source"]), s) and np.array_equal(_np(graph["target"]), t), cloud
        assert np.array_equal(_np(graph["distances"]), d), cloud
        _vor_properties(xyz, simp, graph, nb, vor)
    # a threshold between float32(v) and v: a candidate with d2 == float32(v) is dropped, one below kept
    xyz = G["room.xyz"]
    simp = G["room.simplices"].astype(np.int64)
    dd = xyz[simp[:, 0]] - xyz[simp[:, 1]]
    d2 = np.sort((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2])
    v32 = d2[len(d2) // 2]
    v = float(v32) + float(np.spacing(v32)) / 4  # rounds to v32 in float32, above it in float64
    assert np.float32(v) == v32 and v > float(v32)
    graph, target2 = st.compute_graph_nn_2(xyz, K_ADJ, K_LOCAL, voronoi=v, simplices=simp)
    nb = _np(target2).reshape(len(xyz), K_LOCAL)
    s, t, d = structure_ref.voronoi_graph(xyz, simp, nb, K_ADJ, v)
    assert np.array_equal(_np(graph["distances"]), d) and not (d == v32).any()
    assert np.array_equal(_np(graph["source"]), s) and np.array_equal(_np(graph["target"]), t)
    _vor_properties(xyz, simp, graph, nb, v)


def _check_cc(n, src, tgt, active):
    from superpoint_graph_b200 import spg_structure as st

    comps, inc = st.connected_comp(n, src, tgt, active, 0)
    want_c, want_i = structure_ref.connected_comp(n, src, tgt, active)
    assert np.array_equal(_np(inc), want_i.astype(np.int64))
    assert len(comps) == len(want_c)
    off, mem = _np(comps.offsets), _np(comps.members)
    assert np.array_equal(mem, np.concatenate(want_c).astype(np.int64))
    assert np.array_equal(np.diff(off), [len(c) for c in want_c])
    return comps, inc


@pytest.mark.gpu
def test_connected_comp():
    rng = np.random.default_rng(5)
    n = 300
    src = rng.integers(0, n - 20, 400)  # the last 20 vertices are isolated
    tgt = rng.integers(0, n - 20, 400)
    src[:10] = tgt[:10]  # self-loops
    src = np.concatenate([src, src[:30]])  # duplicate edges
    tgt = np.concatenate([tgt, tgt[:30]])
    for active in (rng.integers(0, 2, len(src)).astype(np.uint8), np.ones(len(src), np.uint8),
                   np.zeros(len(src), np.uint8), rng.choice(np.array([0, 2, 127, 128, 255], np.uint8), len(src)),
                   rng.integers(0, 2, len(src)).astype(bool)):
        _check_cc(n, src, tgt, active)
    comps, inc = _check_cc(5, np.array([0, 1, 2, 3]), np.array([1, 2, 3, 4]),
                           np.array([2, 127, 128, 255], np.uint8))
    assert list(_np(inc)) == [0, 0, 0, 1, 2]
    # a 10^6-vertex path, edges listed from the far end: deep union-find chains
    n = 10 ** 6
    s = np.arange(n - 1)[::-1].copy()
    comps, inc = _check_cc(n, s, s + 1, np.ones(n - 1, np.uint8))
    assert len(comps) == 1
    with pytest.raises(IndexError):
        from superpoint_graph_b200 import spg_structure as st
        st.connected_comp(3, np.array([0]), np.array([3]), np.ones(1, np.uint8))


@pytest.mark.gpu
def test_lp_xpart_unchanged_on_the_partition_golden():
    import torch

    from superpoint_graph_b200 import ops

    p = np.load(os.path.join(os.path.dirname(GOLDEN), "partition.npz"))
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    src, tgt = d(p["main.src"]), d(p["main.tgt"])
    is_tr = d(p["main.is_tr"].astype(np.uint8))
    pic = d(p["main.pic"])
    w, inx, size, n_comp = ops.lp_xpart(src, tgt, is_tr, pic, pic.shape[0], 5.0)
    assert np.array_equal(_np(inx).astype(np.int64), p["main.in_comp_x"])
    c = int(n_comp.item()) if torch.is_tensor(n_comp) else int(n_comp)
    assert np.array_equal(_np(size)[:c].astype(np.int64), p["main.comp_x_size"])
    from oracle import partition_ref
    src_np, tgt_np = p["main.src"], p["main.tgt"]
    want = partition_ref.compute_weights_XPART_sorted(p["main.pic"], src_np, tgt_np, p["main.is_tr"], 5.0)
    assert np.array_equal(_np(w), want)


def _args(c, geof=0):
    return types.SimpleNamespace(k_nn_adj=K_ADJ, k_nn_local=K_LOCAL, use_voronoi=c["use_voronoi"], compute_geof=geof,
                                 plane_model=c["plane_model"])


def _run_case(case, **kw):
    from superpoint_graph_b200 import spg_structure as st

    c, d, simp = _case(case)
    labels = None if c["dataset"] == "sema3d" else d["labels"]
    objects = d["objects"] if c["dataset"] == "s3dis" else None
    return st.compute_structure(_args(c, **kw), c["dataset"], d["xyz"], d["rgb"], labels, objects, True,
                                simplices=simp)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_compute_structure(case):
    c, d, _ = _case(case)
    if c["plane_model"]:
        pytest.importorskip("sklearn")
    got = _run_case(case)
    nb = _np(got["target_local_geometry"])
    want = _oracle(case, nb)
    for k in ("source", "target", "is_transition", "objects", "xyn"):
        assert np.array_equal(_np(got[k] if k not in ("source", "target") else got["graph_nn"][k]),
                              np.asarray(want[k]).astype(np.asarray(want[k]).dtype)), (case, k)
    assert np.array_equal(_np(got["labels"]), np.asarray(want["labels"]).astype(np.int64)), case
    assert np.array_equal(nb, want["target_local_geometry"])
    if c["dataset"] != "sema3d":
        assert np.array_equal(_np(got["labels"]), G[case + ".labels"].astype(np.int64))
    if c["cloud"] != "dup":  # untied k-NN: the golden's own arrays
        assert (nb == d["neighbors"]).all()
        for k in ("is_transition", "objects"):
            assert np.array_equal(_np(got[k]).astype(np.int64), G["%s.%s" % (case, k)].astype(np.int64)), (case, k)
    assert np.array_equal(_np(got["xyn"]), G[case + ".xyn"])
    e = _np(got["elevation"])
    if not c["plane_model"]:
        assert np.array_equal(e, G[case + ".elevation"])
    else:
        wantp = G[case + ".elevation"]
        ulp = np.spacing(np.maximum(np.abs(wantp), np.abs(e)).astype(np.float32))
        assert (np.abs(e.astype(np.float64) - wantp) <= np.maximum(ulp, np.spacing(np.float32(
            np.abs(wantp).max())))).all()
        from superpoint_graph_b200 import spg_structure as st
        out = st.to_numpy(got)
        assert out["elevation"].dtype == np.float32 and out["objects"].dtype == np.uint32
    assert got["geof"] is None


@pytest.mark.gpu
def test_geof_column_3_doubled_and_inpainting_problem():
    import torch

    from superpoint_graph_b200 import spg_geometry
    from superpoint_graph_b200 import spg_structure as st

    got = _run_case("scan_vkitti", geof=1)
    xyz = G["scan.xyz"]
    g = spg_geometry.compute_geof(xyz, got["target_local_geometry"], K_LOCAL)
    g[:, 3] = 2.0 * g[:, 3]
    assert torch.equal(got["geof"], g)
    labels = G["scan.labels"].copy()
    labels[::7, 1:] = 0  # vertices without labels
    hard, s, t, ew, nw = st.inpainting_problem(labels, got["graph_nn"])
    want = structure_ref.inpainting_problem(labels, _np(got["graph_nn"]["source"]), _np(got["graph_nn"]["target"]))
    for a, b in zip((hard, s, t, ew, nw), want):
        assert np.array_equal(_np(a), b) and _np(a).dtype == b.dtype


@pytest.mark.gpu
def test_end_to_end_prune_structure_store_batch():
    import torch

    from superpoint_graph_b200 import spg_delaunay, spg_prune
    from superpoint_graph_b200 import spg_structure as st
    from superpoint_graph_b200.spg_partition_loader import PartitionStore, load_batch

    rng = np.random.default_rng(11)
    n = 6000
    xyz = (rng.uniform(0, 4, (n, 3)) * [1, 1, 0.6]).astype(np.float32)
    rgb = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    lab = (np.floor(xyz[:, 0]) * 3 + np.floor(xyz[:, 2] * 2)).astype(np.int64) % 13 + 1
    pxyz, prgb, plab, _ = spg_prune.prune(xyz, 0.1, rgb, lab, np.zeros(1, np.int64), 13, 0)
    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=10, use_voronoi=0.05, compute_geof=0, plane_model=0)
    dev = st.compute_structure(args, "vkitti", pxyz, prgb, plab)
    tri = spg_delaunay.to_numpy(spg_delaunay.delaunay(pxyz))  # the triangulation compute_structure made
    nb = _np(dev["target_local_geometry"])
    ref = structure_ref.structure("vkitti", _np(pxyz), _np(plab), None, nb, 5, 10, 0.05, tri)
    host = (_np(pxyz), _np(prgb).astype(np.float32), ref["source"], ref["target"], ref["is_transition"].astype(np.uint8),
            nb.astype(np.uint32), ref["labels"].astype(np.int32), ref["objects"].astype(np.uint32), ref["elevation"],
            ref["xyn"])
    bargs = types.SimpleNamespace(ver_value="ptn", k_nn_local=10, use_rgb=1, global_feat="eXYrgb", pc_augm_rot=0,
                                  pc_augm_jitter=0, max_ver_train=0, learned_embeddings_geof=0)
    outs = []
    for tup in (st.as_read_structure(dev, False), host):
        store = PartitionStore()
        store.add("A/f.h5", *tup)
        store.finalize(torch.device("cuda"))
        np.random.seed(0)
        outs.append(load_batch(store, ["A/f.h5"], False, bargs))
    a, b = outs
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        xs, ys = (x, y) if isinstance(x, tuple) else ((x,), (y,))
        for u, v in zip(xs, ys):
            if torch.is_tensor(u):
                assert torch.equal(u, v)
            else:
                assert (u is None and v is None) or np.array_equal(np.asarray(u), np.asarray(v))


@pytest.mark.gpu
def test_two_runs_are_bit_identical():
    import torch

    a = _run_case("scan_vkitti_vor")
    b = _run_case("scan_vkitti_vor")
    for k in ("is_transition", "objects", "elevation", "xyn", "target_local_geometry"):
        assert torch.equal(a[k], b[k]), k
    for k in ("source", "target", "distances"):
        assert torch.equal(a["graph_nn"][k], b["graph_nn"][k]), k


# ------------------------------------------------------------------------------------------ workspaces
SPG_E_BADARG, SPG_E_ALIGN = -1, -3
SENTINEL, TAIL = 0xA5, 4096


def _ws_contract(query, sizes, call):
    """call(ws_ptr, ws_bytes) -> rc, outputs.  Exact bytes with a sentinel tail vs a generous workspace."""
    import torch

    from superpoint_graph_b200 import _lib, ops

    lib = _lib.lib()
    nb = ctypes.c_int64(-1)
    assert getattr(lib, query)(*sizes, ctypes.byref(nb)) == 0
    rep = nb.value
    assert rep > 0 and rep % 256 == 0
    exact = torch.full((rep + TAIL,), SENTINEL, dtype=torch.uint8, device="cuda")
    big = torch.full((2 * rep + TAIL,), 0x5A, dtype=torch.uint8, device="cuda")
    before = ops.total_launches()
    assert call(exact.data_ptr() + 16, rep)[0] == SPG_E_ALIGN
    assert call(exact.data_ptr(), rep - 1)[0] == SPG_E_BADARG
    assert ops.total_launches() == before
    rc, got = call(exact.data_ptr(), rep)
    assert rc == 0
    rc, want = call(big.data_ptr(), 2 * rep)
    assert rc == 0
    torch.cuda.synchronize()
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert bool((exact[rep:] == SENTINEL).all())


@pytest.mark.gpu
def test_workspaces_meet_the_contract():
    import torch

    from superpoint_graph_b200 import _lib, ops

    lib = _lib.lib()
    stream = _lib.current_stream()
    xyz = torch.from_numpy(G["room.xyz"]).cuda()
    simp = torch.from_numpy(G["room.simplices"].astype(np.int32)).cuda()
    n, T = xyz.shape[0], simp.shape[0]
    knn = torch.from_numpy(G["room.neighbors"][:, :K_ADJ].astype(np.int64).reshape(-1)).cuda()
    counts, status = ops.st_vor_count(xyz, simp, 0.05)
    kept = int(counts[-1])

    def vor(ptr, nbytes):
        outs = [torch.zeros(kept, dtype=torch.float32, device="cuda")] + [
            torch.zeros(kept + n * K_ADJ, dtype=torch.int64, device="cuda") for _ in range(2)] + [
            torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")]
        rc = lib.spg_st_vor_build(xyz.data_ptr(), n, simp.data_ptr(), 0, T, ctypes.c_float(0.05), counts.data_ptr(),
                                  knn.data_ptr(), K_ADJ, kept, ctypes.c_void_p(ptr), nbytes,
                                  *[o.data_ptr() for o in outs], ctypes.c_void_p(stream))
        return rc, outs

    _ws_contract("spg_st_vor_workspace", (n, T, n * K_ADJ, kept), vor)
    rng = np.random.default_rng(3)
    V, E = 500, 900
    src = torch.from_numpy(rng.integers(0, V, E)).cuda()
    tgt = torch.from_numpy(rng.integers(0, V, E)).cuda()
    act = torch.from_numpy(rng.integers(0, 256, E).astype(np.uint8)).cuda()

    def cc(ptr, nbytes):
        outs = [torch.zeros(V, dtype=torch.int64, device="cuda"), torch.zeros(V + 1, dtype=torch.int64, device="cuda"),
                torch.zeros(V, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"),
                torch.zeros(1, dtype=torch.int32, device="cuda")]
        rc = lib.spg_st_cc(src.data_ptr(), tgt.data_ptr(), act.data_ptr(), V, E, ctypes.c_void_p(ptr), nbytes,
                           *[o.data_ptr() for o in outs], ctypes.c_void_p(stream))
        return rc, outs

    _ws_contract("spg_st_cc_workspace", (V,), cc)

    def sel(ptr, nbytes):
        outs = [torch.zeros(E, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")]
        rc = lib.spg_st_select(act.data_ptr(), E, 1, ctypes.c_void_p(ptr), nbytes, *[o.data_ptr() for o in outs],
                               ctypes.c_void_p(stream))
        return rc, outs

    _ws_contract("spg_st_select_workspace", (E,), sel)
