"""The learned partition's batch builder (superpoint_graph_b200.spg_partition_loader, csrc/partition_loader.cu).

CPU: the oracle (oracle/partition_loader_ref.py) against the reference's own outputs (partition_loader.npz, from the
unmodified source text of graph_loader / graph_collate / augment_cloud_whole) bit for bit; the product's host draws
against the reference's augmentation draw for draw; host validation; compute_partition's host copies for libcp.
GPU: every golden case without rotation bit for bit; the rotation within 1 ulp and the clouds built from it bit for
bit; device_rng; the resident store left unchanged; tails and an empty selection; a learned-partition step on the
device batch and on the golden batch; compute_partition on the device batch's CUDA edges.
"""
import json
import math
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import partition_loader_ref as lref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "partition_loader.npz")
KEYS = ("xyz", "rgb", "src", "tgt", "is_tr", "lg", "labels", "objects", "elevation", "xyn")
OUTS = ("edg_source", "edg_target", "is_transition", "labels", "objects", "clouds", "clouds_global", "xyz")


def _golden():
    z = np.load(GOLDEN, allow_pickle=False)
    return {k: z[k] for k in z.files}


G = _golden()
META = json.loads(str(G["meta"]))
NAMES = [f["name"] for f in META["files"]]
FILES = {nm: tuple(G["file%d.%s" % (i, k)] for k in KEYS) for i, nm in enumerate(NAMES)}


def _case(tag):
    return next(c for c in META["cases"] if c["tag"] == tag)


def _args(case):
    return SimpleNamespace(**case["args"])


def _names(case):
    return [NAMES[i] for i in case["files"]]


def _masks(case):
    if not case["subsampled"]:
        return None
    return [G["%s.mask.%d" % (case["tag"], b)] for b in range(len(case["files"]))]


def _draws(case, device_rng=False):
    from superpoint_graph_b200.spg_partition_loader import host_draws
    np.random.seed(case["seed"])
    args = _args(case)
    return [host_draws(FILES[nm][0].shape[0], args, bool(args.use_rgb), device_rng) for nm in _names(case)]


def _flat(batch):
    fname, src, tgt, tr, labels, objects, (clouds, cglob, nei), xyz = batch
    out = dict(edg_source=src, edg_target=tgt, is_transition=tr, labels=labels, objects=objects, clouds=clouds,
               clouds_global=cglob, xyz=xyz)
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()}, fname, nei


def _oracle(case, draws=None):
    return lref.load_batch(FILES, _names(case), case["train"], _args(case), draws if case["train"] else None,
                           _masks(case))


# ---------------------------------------------------------------------------------------------------- CPU
def test_golden_records_numpy_version_and_seeds():
    assert META["numpy"] and all("seed" in c for c in META["cases"])
    tags = {c["tag"] for c in META["cases"]}
    assert {"eval_b1", "eval_b3", "train_sub", "train_jitter", "train_rot_b1", "train_rot_nojitter_b1"} <= tags


def test_golden_has_diameter_zero_neighbourhoods():
    """The coincident blob's neighbourhoods: diameter exactly 0, their clouds divided by 1e-10 alone."""
    for tag in ("eval_b1", "eval_b3", "train_sub"):
        d = G[tag + ".clouds_global"][:, 0]
        assert (d == 0).any(), tag
        assert not G[tag + ".clouds"][d == 0, :3].any(), tag


@pytest.mark.parametrize("tag", [c["tag"] for c in META["cases"]])
def test_oracle_reproduces_golden(tag):
    case = _case(tag)
    got, fname, nei = _flat(_oracle(case, _draws(case)))
    for k in OUTS:
        want = G["%s.%s" % (tag, k)]
        assert got[k].shape == want.shape and np.array_equal(got[k].view(np.uint8), want.view(np.uint8)), k
    assert list(fname) == case["fname"]
    assert np.array_equal(nei, G[tag + ".nei"])


@pytest.mark.parametrize("tag", [c["tag"] for c in META["cases"] if c["train"]])
def test_host_draws_match_the_references_augmentation(tag):
    case = _case(tag)
    draws = _draws(case)
    for b, nm in enumerate(_names(case)):
        xyz, rgb = lref.augment(FILES[nm][0], FILES[nm][1] / 255, draws[b])
        assert np.array_equal(xyz, G["%s.aug_xyz.%d" % (tag, b)]), (b, "xyz")
        assert np.array_equal(rgb, G["%s.aug_rgb.%d" % (tag, b)]), (b, "rgb")


def test_rotation_matrix_is_transforms3d():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compat"))
    try:
        import transforms3d
    finally:
        sys.path.pop(0)
    from superpoint_graph_b200.spg_partition_loader import rotation_matrix
    for a in np.random.default_rng(0).uniform(0, 2 * math.pi, 50):
        want = transforms3d.axangles.axangle2mat([0, 0, 1], a).astype("f4")
        assert np.array_equal(rotation_matrix(a).view(np.uint32), want.view(np.uint32))


def test_global_columns_follow_the_substring_tests():
    from superpoint_graph_b200.spg_partition_loader import global_columns
    assert global_columns("eXYrgb")[1] == 7
    assert global_columns("e")[1] == 2
    assert global_columns("")[1] == 1
    assert global_columns("exy")[1] == 4


def _store(device="cpu", names=None):
    from superpoint_graph_b200.spg_partition_loader import PartitionStore
    st = PartitionStore()
    for nm in names or NAMES:
        st.add(nm, *FILES[nm])
    return st.finalize(device)


def test_store_validation():
    from superpoint_graph_b200.spg_partition_loader import PartitionStore
    f = list(FILES[NAMES[2]])
    n = f[0].shape[0]
    bad_edge = list(f)
    bad_edge[3] = f[3].copy()
    bad_edge[3][5] = n
    with pytest.raises(IndexError):
        PartitionStore().add("a/b", *bad_edge)
    bad_lg = list(f)
    bad_lg[5] = f[5].copy()
    bad_lg[5][2, 7] = n + 3
    with pytest.raises(IndexError):
        PartitionStore().add("a/b", *bad_lg)
    short = list(f)
    short[1] = f[1][:-1]
    with pytest.raises(ValueError):
        PartitionStore().add("a/b", *short)
    tr = list(f)
    tr[4] = f[4][:-2]
    with pytest.raises(ValueError):
        PartitionStore().add("a/b", *tr)
    st = _store()
    assert st.file(NAMES[0])["xyz"].shape == (400, 3)
    assert st.resident_bytes() == sum((36 + 4 * (30 + 14 + 1)) * v["n_ver"] + 9 * 5 * 2 * v["n_ver"]
                                      for v in META["files"])


def test_subsampling_without_mask_or_libply_c_raises(monkeypatch):
    from superpoint_graph_b200.spg_partition_loader import load_batch
    monkeypatch.setitem(sys.modules, "libply_c", None)
    monkeypatch.setitem(sys.modules, "partition.ply_c", None)
    case = _case("train_sub")
    with pytest.raises(RuntimeError, match="selected="):
        load_batch(_store(), _names(case), True, _args(case))


def test_geof_branches_point_to_the_reference():
    from superpoint_graph_b200.spg_partition_loader import load_batch
    for vv in ("geof", "geofrgb"):
        with pytest.raises(ValueError, match="graph_loader"):
            load_batch(_store(), NAMES[:1], False, SimpleNamespace(ver_value=vv))


def _libcp(seen):
    def cutpursuit(ver_value, s, t, w, *a, **k):
        seen.append((ver_value, s, t))
        return [np.arange(3, dtype=np.uint32)], np.zeros(3, np.uint32)
    return types.SimpleNamespace(cutpursuit=cutpursuit)


def test_compute_partition_hands_uint32_host_arrays_to_libcp(monkeypatch):
    from superpoint_graph_b200 import spg_partition as sp
    seen = []
    monkeypatch.setitem(sys.modules, "libcp", _libcp(seen))
    monkeypatch.setattr(sp, "partition_edge_weight", lambda args, diff: np.ones(4, np.float32))
    args = SimpleNamespace(spatial_emb=0.5, reg_strength=1.0, k_nn_adj=5, CP_cutoff=10, edge_weight_threshold=-0.5)
    emb = torch.randn(3, 4)
    src, tgt = np.array([0, 1, 2, 0]), np.array([1, 2, 0, 2])
    xyz = np.random.default_rng(1).normal(size=(3, 3)).astype(np.float32)
    sp.compute_partition(args, emb, src, tgt, None, xyz)
    sp.compute_partition(args, emb, torch.from_numpy(src), torch.from_numpy(tgt), None, torch.from_numpy(xyz))
    (v0, s0, t0), (v1, s1, t1) = seen
    assert s0.dtype == np.uint32 and t0.dtype == np.uint32 and np.array_equal(s0, s1) and np.array_equal(t0, t1)
    assert s1.dtype == np.uint32 and np.array_equal(v0, v1) and v0.shape == (3, 7)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def store(dev):
    return _store(dev)


def _device_batch(store, case, **kw):
    from superpoint_graph_b200.spg_partition_loader import load_batch
    np.random.seed(case["seed"])
    return load_batch(store, _names(case), case["train"], _args(case), selected=_masks(case), **kw)


def _ulps(a, b):
    """Distance in units in the last place between float32 arrays."""
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


@pytest.mark.gpu
@pytest.mark.parametrize("tag", [c["tag"] for c in META["cases"] if not c["args"]["pc_augm_rot"]])
def test_device_matches_golden_bit_for_bit(dev, store, tag):
    case = _case(tag)
    batch = _device_batch(store, case)
    got, fname, nei = _flat(batch)
    assert batch[1].dtype == torch.int64 and batch[3].dtype == torch.uint8 and batch[5].dtype == torch.int64
    assert batch[6][0].is_contiguous() and batch[1].is_cuda
    for k in OUTS:
        want = G["%s.%s" % (tag, k)]
        g = got[k]
        assert g.shape == want.shape, (k, g.shape, want.shape)
        if want.dtype.kind == "f":
            assert np.array_equal(g.view(np.uint32), want.view(np.uint32)), k
        else:
            assert np.array_equal(g.astype(np.int64), want.astype(np.int64)), k
    assert list(fname) == case["fname"] and np.array_equal(nei, G[tag + ".nei"])


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["train_rot_b1", "train_rot_nojitter_b1"])
def test_rotation_within_one_ulp_and_clouds_from_its_xyz(dev, store, tag):
    case = _case(tag)  # one file, nothing sub-sampled: the output xyz is the whole augmented file
    got, _, _ = _flat(_device_batch(store, case))
    assert _ulps(got["xyz"], G[tag + ".xyz"]).max() <= 1
    for k in ("edg_source", "edg_target", "is_transition", "labels", "objects"):
        assert np.array_equal(got[k].astype(np.int64), G[tag + "." + k].astype(np.int64)), k
    # the oracle's clouds built from the device's own augmented xyz and the (rotation-free) augmented rgb
    nm = _names(case)[0]
    ref, _, _ = _flat(lref.graph_collate([lref.graph_loader(
        nm, FILES[nm], True, _args(case), augmented=(got["xyz"], G[tag + ".aug_rgb.0"]))]))
    for k in ("clouds", "clouds_global"):
        assert np.array_equal(got[k].view(np.uint32), ref[k].view(np.uint32)), k
    if not case["args"]["pc_augm_jitter"]:
        # nothing is drawn on the device without jitter: device_rng gives the same batch
        again, _, _ = _flat(_device_batch(store, case, device_rng=True, seed=9))
        for k in OUTS:
            assert np.array_equal(again[k], got[k]), k


@pytest.mark.gpu
def test_rotation_with_subsampling_batch_of_three(dev, store):
    got3, _, _ = _flat(_device_batch(store, _case("train_rot_b3")))
    assert _ulps(got3["xyz"], G["train_rot_b3.xyz"]).max() <= 1
    for k in ("edg_source", "edg_target", "is_transition", "labels", "objects"):
        assert np.array_equal(got3[k].astype(np.int64), G["train_rot_b3." + k].astype(np.int64)), k


def _big_store(dev, n=40000, seed=3):
    from superpoint_graph_b200.spg_partition_loader import PartitionStore
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, 20, (n, 3)).astype(np.float32)
    lg = np.concatenate([np.arange(n)[:, None], rng.integers(0, n, (n, 24))], 1).astype(np.uint32)
    src = rng.integers(0, n, 5 * n)
    tgt = rng.integers(0, n, 5 * n)
    obj = rng.integers(0, 50, n)
    st = PartitionStore().add("big/f.h5", xyz, rng.integers(0, 256, (n, 3)).astype(np.float32), src, tgt,
                              (obj[src] != obj[tgt]).astype(np.uint8), lg,
                              rng.integers(0, 5, (n, 14)).astype(np.uint32), obj,
                              rng.normal(size=n).astype(np.float32), rng.normal(size=(n, 2)).astype(np.float32))
    return st.finalize(dev), xyz


def _jitter_args(**kw):
    a = dict(ver_value="ptn", k_nn_local=20, use_rgb=1, global_feat="eXYrgb", pc_augm_rot=0, pc_augm_jitter=1,
             max_ver_train=0)
    a.update(kw)
    return SimpleNamespace(**a)


@pytest.mark.gpu
def test_device_rng_jitter(dev):
    from superpoint_graph_b200.spg_partition_loader import load_batch
    st, xyz0 = _big_store(dev)
    args = _jitter_args()
    a = _flat(load_batch(st, ["big/f.h5"], True, args, device_rng=True, seed=5))[0]
    b = _flat(load_batch(st, ["big/f.h5"], True, args, device_rng=True, seed=5))[0]
    c = _flat(load_batch(st, ["big/f.h5"], True, args, device_rng=True, seed=6))[0]
    for k in OUTS:
        assert np.array_equal(a[k], b[k]), k
    assert not np.array_equal(a["xyz"], c["xyz"]) and not np.array_equal(a["clouds"], c["clouds"])
    jit = (a["xyz"].astype(np.float64) - xyz0.astype(np.float64)).reshape(-1)
    assert np.abs(jit).max() <= 0.005 + 1e-6
    # clip(N(0, 0.002^2), +-0.005): standard deviation by quadrature
    x = np.linspace(-0.005, 0.005, 200001)
    pdf = np.exp(-0.5 * (x / 0.002) ** 2) / (0.002 * math.sqrt(2 * math.pi))
    tail = 0.5 * math.erfc(2.5 / math.sqrt(2))
    std = math.sqrt(np.trapezoid(x * x * pdf, x) + 2 * tail * 0.005 ** 2)
    assert abs(jit.mean()) < 4 * std / math.sqrt(jit.size)  # four standard errors
    assert abs(jit.std() / std - 1) < 0.02, (jit.std(), std)
    rgb = a["clouds_global"][:, 2:5]
    assert rgb.min() >= -1 and rgb.max() <= 1
    assert a["clouds"][:, 3:].min() >= -1 and a["clouds"][:, 3:].max() <= 1


@pytest.mark.gpu
def test_store_unchanged_by_training_batches(dev, store):
    before = [t.clone() for t in (store.floats, store.ints, store.bytes)]
    _device_batch(store, _case("train_rot_b3"))
    _device_batch(store, _case("train_rot_b3"), device_rng=True, seed=3)
    for a, b in zip(before, (store.floats, store.ints, store.bytes)):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_tails_and_an_empty_selection(dev, store):
    from superpoint_graph_b200.spg_partition_loader import load_batch
    case = _case("train_sub")
    masks = _masks(case)
    args = _args(case)
    # 120 + 0 + 119 kept vertices: a row count that is not a multiple of the 8 warps per CTA
    m2 = masks[2].copy()
    m2[np.nonzero(m2)[0][0]] = False
    empty = np.zeros_like(masks[1])
    got, _, _ = _flat(load_batch(store, _names(case), True, args, selected=[masks[0], empty, m2]))
    names = [_names(case)[0], _names(case)[2]]
    want, _, _ = _flat(lref.load_batch(FILES, names, True, args, [(None,) * 4] * 2, [masks[0], m2]))
    assert got["xyz"].shape[0] == 239
    for k in OUTS:
        assert np.array_equal(got[k], want[k].astype(got[k].dtype)), k


def _lp_model(dev, n_global):
    from superpoint_graph_b200.spg_pointnet import PointNet, STNkD
    torch.manual_seed(4)
    model = torch.nn.Module()
    model.stn = STNkD(2, [16, 64], [32, 16], norm="layer", n_group=1)
    model.ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=0, nfeat_global=n_global + 4,
                         norm="layer", n_group=1)
    return model.to(dev).train()


def _step(model, batch, dev):
    from superpoint_graph_b200 import spg_partition as sp
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder
    _, src, tgt, is_tr, _, objects, (clouds, cglob, _), xyz = batch
    model.zero_grad()
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1)).run_batch(model, clouds, cglob)
    emb.retain_grad()
    args = SimpleNamespace(loss_weight="crosspartition", loss="TVH_zhang", dist_type="euclidian",
                           transition_factor=5.0, k_nn_adj=5, edge_weight_threshold=-0.5, spatial_emb=0)
    vox = np.floor(xyz.cpu().numpy() / 1.5).astype(np.int64)
    _, pic = np.unique(vox[:, 0] * 10000 + vox[:, 1] * 100 + vox[:, 2], return_inverse=True)
    comps = [np.nonzero(pic == c)[0].astype(np.uint32) for c in range(int(pic.max()) + 1)]
    diff = sp.compute_dist(emb, src, tgt, args.dist_type)
    w = sp.compute_weight_loss(args, emb, objects, src, tgt, is_tr, diff, False, partition=(comps, pic))
    l1, l2 = sp.compute_loss(args, diff, is_tr, w)
    loss = (l1 + l2) / w.shape[0] * 1000
    loss.backward()
    return loss.detach().cpu(), emb.grad.detach().cpu()


@pytest.mark.gpu
def test_learned_partition_step_on_the_device_batch(dev, store):
    case = _case("train_jitter")
    batch = _device_batch(store, case)
    t = lambda k, dt=None: torch.from_numpy(np.ascontiguousarray(G["train_jitter." + k])).to(dev)
    gold = (None, t("edg_source"), t("edg_target"), t("is_transition"), t("labels").long(), t("objects"),
            (t("clouds"), t("clouds_global"), None), t("xyz"))
    model = _lp_model(dev, 7)
    l_dev, g_dev = _step(model, batch, dev)
    l_gold, g_gold = _step(model, gold, dev)
    assert torch.isfinite(l_dev) and np.array_equal(l_dev.numpy().view(np.uint32), l_gold.numpy().view(np.uint32))
    assert torch.equal(g_dev, g_gold)


@pytest.mark.gpu
def test_compute_partition_on_cuda_edges(dev, store, monkeypatch):
    from superpoint_graph_b200 import spg_partition as sp
    seen = []
    monkeypatch.setitem(sys.modules, "libcp", _libcp(seen))
    case = _case("train_sub")
    _, src, tgt, _, _, _, _, xyz = _device_batch(store, case)
    args = SimpleNamespace(spatial_emb=0.2, reg_strength=1.0, k_nn_adj=5, CP_cutoff=10, edge_weight_threshold=-0.5)
    emb = torch.nn.functional.normalize(torch.randn(xyz.shape[0], 4, device=dev))
    diff = sp.compute_dist(emb, src, tgt, "euclidian")
    sp.compute_partition(args, emb, src, tgt, diff, xyz)
    sp.compute_partition(args, emb, G["train_sub.edg_source"], G["train_sub.edg_target"], diff, G["train_sub.xyz"])
    (v0, s0, t0), (v1, s1, t1) = seen
    assert s0.dtype == np.uint32 and np.array_equal(s0, s1) and np.array_equal(t0, t1)
    assert np.array_equal(v0, v1)
