"""The partition stages' shared input rules (superpoint_graph_b200/_inputs.py).

CPU: the checks refuse the dtypes the stages refuse, treat a numpy array and a CPU tensor alike, and refuse a cloud of
2^31 - 1 points from its shape alone.
GPU: every public entry point of the device stages synchronises with the host as often as recorded, for CUDA-tensor
and numpy inputs: the number of host read-backs and uploads is part of what these entry points promise.
"""
import types
import warnings

import numpy as np
import pytest
import torch

CPU = torch.device("cpu")


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("dtype", ["float16", "float64", "bool", "complex64", "int32"])
def test_check_dtype_refuses_every_other_dtype(dtype):
    from superpoint_graph_b200._inputs import check_dtype
    a = np.zeros((4, 3), dtype)
    for x in (a, torch.from_numpy(a)):
        with pytest.raises(TypeError, match="xyz must be float32 \\(got (torch\\.)?%s\\)" % dtype):
            check_dtype(x, "xyz", "float32")
    with pytest.raises(TypeError, match="rgb must be uint8"):
        check_dtype(a, "rgb", "uint8")


@pytest.mark.parametrize("dtype", ["float16", "float32", "float64", "bool", "complex64"])
def test_check_ints_refuses_non_integers(dtype):
    from superpoint_graph_b200._inputs import check_ints
    a = np.zeros(5, dtype)
    for x in (a, torch.from_numpy(a)):
        with pytest.raises(TypeError, match="ids must hold integers \\(got (torch\\.)?%s\\)" % dtype):
            check_ints(x, "ids")


def test_numpy_and_cpu_tensor_alike():
    from superpoint_graph_b200._inputs import check_dtype, check_ints, on_device, simplices_on
    rng = np.random.default_rng(0)
    xyz = rng.random((7, 3), dtype=np.float32)
    assert check_dtype(xyz, "xyz", "float32") == check_dtype(torch.from_numpy(xyz), "xyz", "float32") == (7, 3)
    for dtype in (np.uint8, np.int8, np.int32, np.uint32, np.int64):
        ids = rng.integers(0, 100, (6, 2)).astype(dtype)
        assert check_ints(ids, "ids") == (6, 2)
        got = on_device(ids.T, CPU, int64=True)
        assert got.dtype == torch.int64 and got.is_contiguous() and np.array_equal(got.numpy(), ids.T)
        if dtype != np.uint32:  # torch has no general uint32 tensor
            t = torch.from_numpy(ids)
            assert check_ints(t, "ids") == (6, 2)
            assert torch.equal(on_device(t.T, CPU, int64=True), got)
    got = on_device(xyz.T, CPU)  # floats are never cast
    assert got.dtype == torch.float32 and got.is_contiguous()
    assert torch.equal(got, on_device(torch.from_numpy(xyz).T, CPU))
    s = rng.integers(0, 7, (5, 4))
    assert simplices_on(s.astype(np.int32), CPU).dtype == torch.int32
    assert simplices_on(torch.from_numpy(s.astype(np.int32)), CPU).dtype == torch.int32
    for x in (s.astype(np.uint16), torch.from_numpy(s.astype(np.int16))):
        out = simplices_on(x, CPU)
        assert out.dtype == torch.int64 and np.array_equal(out.numpy(), s)
    with pytest.raises(ValueError, match="simplices must be \\[T, 4\\]"):
        simplices_on(s[:, :3], CPU)
    with pytest.raises(TypeError, match="simplices must hold integers"):
        simplices_on(s.astype(np.float64), CPU)


def test_point_limit_from_a_broadcast_view():
    from superpoint_graph_b200._inputs import check_dtype, n_points
    huge = np.broadcast_to(np.zeros(3, np.float32), (2 ** 31 - 1, 3))  # about 26 GB if it were ever materialised
    for x in (huge, torch.zeros(3).expand(2 ** 31 - 1, 3)):
        with pytest.raises(ValueError, match="2\\^31 - 1 points or more"):
            n_points(check_dtype(x, "xyz", "float32"))
    assert n_points((2 ** 31 - 2, 3)) == 2 ** 31 - 2
    for shape in ((5,), (5, 2), (5, 3, 1)):
        with pytest.raises(ValueError, match="xyz must be \\[n, 3\\]"):
            n_points(shape)


# ---------------------------------------------------------------------------------------------------- GPU
# Synchronising operations torch reports for one call of each entry point after a warm-up call, with every array
# argument a CUDA tensor ("cuda") or a numpy array ("numpy"): each .item(), .cpu() and upload from pageable host memory
# counts once.  Status words that the library itself copies to host memory (cut pursuit's and the triangulation's) are
# not seen by torch.  Recorded on an H100.
SYNCS = {
    "compute_graph_nn/cuda":              2, "compute_graph_nn/numpy":              3,
    "compute_graph_nn_2/cuda":            2, "compute_graph_nn_2/numpy":            3,
    "compute_geof/cuda":                  1, "compute_geof/numpy":                  3,
    "prune/cuda":                         2, "prune/numpy":                         6,
    "compute_sp_graph/cuda":              5, "compute_sp_graph/numpy":              9,
    "cutpursuit/cuda":                    0, "cutpursuit/numpy":                    4,
    "delaunay/cuda":                      0, "delaunay/numpy":                      1,
    "structure.compute_graph_nn_2/cuda":  5, "structure.compute_graph_nn_2/numpy":  8,
    "connected_comp/cuda":                2, "connected_comp/numpy":                5,
    "compute_structure.s3dis/cuda":       4, "compute_structure.s3dis/numpy":       8,
    "compute_structure.vkitti/cuda":      7, "compute_structure.vkitti/numpy":      10,
}


def _syncs(fn):
    fn()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchronizing" in str(w.message) for w in caught)


def _cloud(n=2000, seed=0):
    rng = np.random.default_rng(seed)
    xyz = rng.random((n, 3), dtype=np.float32)
    _, comp = np.unique(np.floor(xyz * 3).astype(np.int64), axis=0, return_inverse=True)
    hist = np.zeros((n, 5), np.int64)
    hist[np.arange(n), rng.integers(0, 5, n)] = 1
    obj = np.zeros((n, 4), np.int64)
    obj[np.arange(n), rng.integers(1, 4, n)] = 1
    return dict(xyz=xyz, rgb=rng.integers(0, 256, (n, 3)).astype(np.uint8), comp=comp.reshape(-1),
                labels=rng.integers(0, 5, n), hist=hist, obj=obj, obs=rng.random((n, 3), dtype=np.float32))


def sync_counts():
    """{"<entry point>/<cuda|numpy>": synchronising operations}; the same body measures any revision."""
    from scipy.spatial import Delaunay

    from superpoint_graph_b200 import spg_structure
    from superpoint_graph_b200.spg_cut_pursuit import cutpursuit
    from superpoint_graph_b200.spg_delaunay import delaunay
    from superpoint_graph_b200.spg_geometry import compute_geof, compute_graph_nn, compute_graph_nn_2
    from superpoint_graph_b200.spg_prune import prune
    from superpoint_graph_b200.spg_sp_graph import compute_sp_graph

    c = _cloud()
    n = c["xyz"].shape[0]
    graph, target2 = compute_graph_nn_2(c["xyz"], 10, 20)
    c["target2"] = target2.cpu().numpy()
    c["source"], c["target"] = graph["source"].cpu().numpy(), graph["target"].cpu().numpy()
    c["weight"] = np.ones(c["source"].shape[0], np.float32)
    c["active"] = (np.random.default_rng(1).random(c["source"].shape[0]) < 0.7).astype(np.uint8)
    c["simplices"] = Delaunay(c["xyz"]).simplices.astype(np.int32)
    n_com = int(c["comp"].max()) + 1
    _syncs(lambda: torch.ones(1, device="cuda").item())  # torch reports one more in the first block measured
    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=10, use_voronoi=0.0, compute_geof=1, plane_model=0)
    out = {}
    for kind in ("cuda", "numpy"):
        a = {k: torch.from_numpy(v).cuda() for k, v in c.items()} if kind == "cuda" else c
        calls = {
            "compute_graph_nn": lambda: compute_graph_nn(a["xyz"], 10),
            "compute_graph_nn_2": lambda: compute_graph_nn_2(a["xyz"], 10, 20),
            "compute_geof": lambda: compute_geof(a["xyz"], a["target2"], 20),
            "prune": lambda: prune(a["xyz"], 0.05, a["rgb"], a["labels"], a["comp"], 4, n_com),
            "compute_sp_graph": lambda: compute_sp_graph(a["xyz"], 0.5, a["comp"], range(n_com), a["labels"], 4,
                                                         simplices=a["simplices"]),
            "cutpursuit": lambda: cutpursuit(a["obs"], a["source"], a["target"], a["weight"], 0.05),
            "delaunay": lambda: delaunay(a["xyz"]),
            "structure.compute_graph_nn_2": lambda: spg_structure.compute_graph_nn_2(
                a["xyz"], 5, 20, voronoi=0.01, simplices=a["simplices"]),
            "connected_comp": lambda: spg_structure.connected_comp(n, a["source"], a["target"], a["active"], 0),
            "compute_structure.s3dis": lambda: spg_structure.compute_structure(
                args, "s3dis", a["xyz"], a["rgb"], a["hist"], a["obj"]),
            "compute_structure.vkitti": lambda: spg_structure.compute_structure(
                args, "vkitti", a["xyz"], a["rgb"], a["hist"]),
        }
        for name, fn in calls.items():
            out["%s/%s" % (name, kind)] = _syncs(fn)
    return out


@pytest.mark.gpu
def test_entry_points_synchronise_as_often_as_recorded():
    assert sync_counts() == SYNCS
