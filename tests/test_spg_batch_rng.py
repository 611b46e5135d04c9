"""The superpoint graph's batch with its draws on the device (spg_loader.load_batch(device_rng=True),
csrc/batch_rng.cu).

CPU: the oracle's restated draws (oracle/spg_batch_rng_ref.py) have the reference's distributions: uniform
permutations, uniform centre subsets independent of the permutation, uniform resample indices with the original points
first, scales in [1/a, a], uniform angles, mirror frequencies p/2 and clipped N(0, 0.01) jitter; the edge cases draw
nothing.  GPU: the device draws against the oracle's (integers and mirror choices bit for bit, matrices within 4
float64 ulp, jitter within 1 float32 ulp); whole batches against the oracle's batch on the golden graphs and on a
10^5-vertex / 10^6-edge graph; seeds, positions and evaluation keys; untouched host generators; one synchronisation
for 1 and for 4 graphs; the collate's exceptions and KeyError; main.py's training-step body.
"""
import json
import os
import random
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import cut_pursuit_ref
from oracle import spg_batch_rng_ref as rref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spg_batch.npz")
ARGS = dict(spg_augm_nneigh=8, spg_augm_order=1, spg_augm_hardcutoff=20, ptn_minpts=40, ptn_npts=16,
            pc_attribs="xyzrgbe", pc_xyznormalize=1, pc_augm_scale=1.3, pc_augm_rot=1, pc_augm_mirror_prob=0.5,
            pc_augm_jitter=1)


def test_vector_philox_matches_scalar_restatement():
    c = np.array([0, 1, 7, 0xFFFFFFFF, 123456789], dtype=np.uint64)
    w = rref.philox(c, c + np.uint64(3), 5, 0x103, 0x89ABCDEF, 0x01234567)
    for i, ci in enumerate(c.tolist()):
        ref = cut_pursuit_ref.philox4x32_10(ci, (ci + 3) & 0xFFFFFFFF, 5, 0x103, 0x89ABCDEF, 0x01234567)
        assert tuple(int(x[i]) for x in w) == ref


def test_permutation_positions_are_uniform():
    n, seeds = 6, 3000
    counts = np.zeros((n, n), np.int64)
    for s in range(seeds):
        perm, _, cut = rref.graph_draws(n, s, 0, True, 3, 0)
        assert sorted(perm.tolist()) == list(range(n)) and cut == 3
        counts[np.arange(n), perm] += 1
    assert stats.chisquare(counts.ravel()).pvalue > 1e-3


def test_centres_are_uniform_and_independent_of_the_permutation():
    n, k, seeds = 12, 4, 4000
    freq = np.zeros(n, np.int64)
    table = np.zeros((n, 2), np.int64)  # new id of vertex 0  x  is that new id a centre
    for s in range(seeds):
        perm, centres, _ = rref.graph_draws(n, s, 1, True, 5, k)
        assert len(set(centres.tolist())) == k
        freq[centres] += 1
        table[perm[0], int(perm[0] in set(centres.tolist()))] += 1
    assert stats.chisquare(freq).pvalue > 1e-3
    assert abs(freq.sum() / (n * seeds) - k / n) < 1e-12
    assert stats.chi2_contingency(table).pvalue > 1e-3
    assert abs(table[:, 1].sum() / seeds - k / n) < 0.03


def test_resample_indices_are_uniform_with_the_original_points_first():
    L = 128
    many = np.concatenate([rref.sample_indices(3, sp, 0, 7, L, True) for sp in range(200)])
    assert many.min() >= 0 and many.max() < 7 and stats.chisquare(np.bincount(many, minlength=7)).pvalue > 1e-3
    few = rref.sample_indices(3, 5, 1, 50, L, True)
    assert np.array_equal(few[:50], np.arange(50)) and few[50:].max() < 50
    assert np.array_equal(rref.sample_indices(3, 5, 1, L, L, True), np.arange(L))
    ev = rref.sample_indices(3, 5, 1, 500, L, False, 2)
    assert np.array_equal(ev, rref.sample_indices(3, 4, 9, 500, L, False, 3))  # id + offset, not the position
    assert not np.array_equal(ev, rref.sample_indices(3, 5, 1, 500, L, False, 0))


def test_augmentation_distributions():
    a, p, N = 1.3, 0.5, 4000
    u = np.stack([rref.augment_uniforms(11, sp, sp % 3) for sp in range(N)])
    M = [rref.augment_matrix(11, sp, sp % 3, a, 1, p) for sp in range(N)]
    s = np.array([abs(np.linalg.det(m)) ** (1 / 3) for m in M])
    assert s.min() >= 1 / a - 1e-12 and s.max() <= a + 1e-12
    assert stats.kstest(2 * np.pi * u[:, 1], stats.uniform(0, 2 * np.pi).cdf).pvalue > 1e-3
    for col in (2, 3):
        f = float((u[:, col] < p / 2).mean())
        assert abs(f - p / 2) < 4 * np.sqrt(p / 2 * (1 - p / 2) / N)
    mirrored = np.array([np.linalg.det(m) < 0 for m in M])
    assert np.array_equal(mirrored, (u[:, 2] < p / 2) ^ (u[:, 3] < p / 2))


def test_jitter_is_clipped_normal():
    j = np.concatenate([rref.jitter(5, sp, 0, 128, 7).ravel() for sp in range(40)])
    assert j.dtype == np.float32 and np.abs(j).max() <= np.float32(0.05)
    assert abs(float(j.mean())) < 2e-4 and abs(float(j.std()) - 0.01) < 2e-4


def test_edge_cases_draw_nothing():
    assert rref.graph_draws(20, 1, 0, True, 20, 3)[0] is None  # hardcutoff >= n
    assert rref.graph_draws(20, 1, 0, True, 5, 20)[1] is None  # nneigh >= n
    assert rref.graph_draws(20, 1, 0, False, 5, 3) == (None, None, 0)
    g, meta = _golden()
    args = SimpleNamespace(**dict(ARGS, pc_augm_jitter=1))
    out = rref.build_batch(_oracle_graphs(g, meta, [0]), _parsed_all(g, meta), False, args, 4)
    assert all(M is None and noise is None for _, M, noise in out[-1])


# ------------------------------------------------------------------------------------------------------ helpers

def _golden():
    z = np.load(GOLDEN, allow_pickle=False)
    g = {k: z[k] for k in z.files}
    return g, json.loads(str(g["meta"]))


def _room(g, i):
    return tuple(g["room%d.%s" % (i, k)] for k in ("node_gt", "node_gt_size", "edges", "edge_feats"))


def _parsed_all(g, meta):
    return {r["name"]: {sp: g["room%d.sp%d" % (i, sp)] for sp in range(r["n_sp"])} for i, r in enumerate(meta["rooms"])}


def _oracle_graphs(g, meta, rooms):
    out = []
    for i in rooms:
        node_gt, node_gt_size, edges, feats = _room(g, i)
        out.append((meta["rooms"][i]["name"], node_gt.shape[0], edges, node_gt_size.sum(1),
                    np.concatenate([node_gt, node_gt_size], 1).astype(np.int64), feats))
    return out


def _stores(g, meta, skip=None):
    from superpoint_graph_b200 import spg_loader

    gs, cs = spg_loader.GraphStore(), spg_loader.SuperpointStore()
    for i, r in enumerate(meta["rooms"]):
        gs.add(*_room(g, i), r["name"])
        cs.add(r["name"], {sp: P for sp, P in _parsed_all(g, meta)[r["name"]].items() if (r["name"], sp) != skip})
    return gs.finalize("cuda"), cs.finalize("cuda")


def _compare(dev_out, ref, tag):
    targets, GIs, (cmeta, cflag, clouds, cglob) = dev_out
    t, idxn, degs, feats, ei, meta, flags, rclouds, rdiam, _ = ref
    gi = GIs[0]
    assert np.array_equal(targets.cpu().numpy(), t), tag
    assert np.array_equal(gi._idxn.cpu().numpy(), idxn) and np.array_equal(gi._degrees_gpu.cpu().numpy(), degs), tag
    assert np.array_equal(gi._edgefeats.cpu().numpy(), feats) and np.array_equal(gi._edge_indexes.cpu().numpy(), ei)
    assert cmeta == meta and cflag.dtype == torch.int64 and not cflag.is_cuda and np.array_equal(cflag.numpy(), flags)
    assert clouds.is_cuda and cglob.is_cuda and clouds.shape == rclouds.shape, tag
    np.testing.assert_allclose(clouds.cpu().numpy(), rclouds, rtol=1e-6, atol=1e-6, err_msg=tag)
    np.testing.assert_array_equal(cglob.cpu().numpy(), rdiam, err_msg=tag)


# ------------------------------------------------------------------------------------------------------ GPU

@pytest.mark.gpu
def test_device_draws_match_oracle():
    from superpoint_graph_b200 import ops

    for n, seed, pos, hc, nn in ((1, 0, 0, 0, 0), (37, 5, 0, 10, 4), (1000, 2 ** 63 + 7, 3, 512, 100),
                                 (100_000, 9, 1, 512, 100)):
        perm, centres = ops.batch_draw(n, seed, pos, 0 < hc < n, nn if 0 < nn < n else 0, "cuda")
        rp, rc, _ = rref.graph_draws(n, seed, pos, True, hc, nn)
        assert (perm is None) == (rp is None) and (centres is None) == (rc is None)
        if rp is not None:
            assert np.array_equal(perm.cpu().numpy(), rp)
        if rc is not None:
            assert np.array_equal(centres.cpu().numpy(), rc)
    rng = np.random.default_rng(1)
    nv, L, F = 300, 64, 7
    counts = rng.integers(1, 200, size=nv).astype(np.int32)
    counts[:3] = (L, L - 1, L + 1)
    ids, pos = rng.integers(0, 10 ** 6, size=nv), rng.integers(0, 4, size=nv)
    keys = (pos.astype(np.int64) << 32) | ids
    dk, dc = torch.from_numpy(keys).cuda(), torch.from_numpy(counts).cuda()
    for train, seed, off in ((True, 17, 0), (False, 17, 0), (False, 17, 2 ** 32 + 3)):
        idx, M, noise = ops.batch_cloud_draw(dk, dc, nv, L, F, seed, train, off, 1.3, 1, 0.5, jitter=True)
        idx = idx.cpu().numpy()
        assert (M is not None and noise is not None) == train
        for c in range(nv):
            assert np.array_equal(idx[c], rref.sample_indices(seed, ids[c], pos[c], counts[c], L, train, off))
        if not train:
            continue
        M, noise = M.cpu().numpy().reshape(nv, 3, 3), noise.cpu().numpy()
        for c in range(nv):
            rm = rref.augment_matrix(seed, ids[c], pos[c], 1.3, 1, 0.5)
            assert M[c, 2, 2] == rm[2, 2]  # the scale, bit for bit
            assert np.array_equal(np.sign(np.linalg.det(M[c])), np.sign(np.linalg.det(rm)))  # mirrors
            assert np.abs(M[c] - rm).max() <= 4 * np.spacing(1.0)
            rj = rref.jitter(seed, ids[c], pos[c], L, F)
            assert np.abs(noise[c] - rj).max() <= np.spacing(np.float32(0.05))


@pytest.mark.gpu
def test_golden_graphs_match_oracle_batch():
    from superpoint_graph_b200 import spg_loader

    g, meta = _golden()
    gs, cs = _stores(g, meta)
    parsed = _parsed_all(g, meta)
    for case in meta["cases"]:
        for seed in (0, 12345):
            args = SimpleNamespace(**dict(case["args"], pc_augm_scale=1.3, pc_augm_mirror_prob=0.5)) \
                if case["train"] else SimpleNamespace(**case["args"])
            names = [meta["rooms"][i]["name"] for i in case["rooms"]]
            tag = "%s/%d" % (case["tag"], seed)
            try:
                ref = rref.build_batch(_oracle_graphs(g, meta, case["rooms"]), parsed, case["train"], args, seed,
                                       case["test_seed_offset"])
            except (RuntimeError, TypeError) as e:
                with pytest.raises(type(e)):
                    spg_loader.load_batch(gs, cs, names, case["train"], args, case["test_seed_offset"],
                                          device_rng=True, seed=seed)
                continue
            _compare(spg_loader.load_batch(gs, cs, names, case["train"], args, case["test_seed_offset"],
                                           device_rng=True, seed=seed), ref, tag)


@pytest.mark.gpu
def test_large_graph_matches_oracle_batch():
    from superpoint_graph_b200 import spg_loader

    rng = np.random.default_rng(5)
    n, E = 100_000, 1_000_000
    edges = rng.integers(0, n, size=(E, 2))
    node_gt = rng.integers(0, 13, size=(n, 1))
    node_gt_size = rng.integers(0, 40, size=(n, 3))
    feats = rng.standard_normal((E, 4)).astype(np.float32)
    pts = rng.integers(1, 60, size=n)
    parsed = {"big": {i: rng.standard_normal((int(pts[i]), 7)).astype(np.float32) for i in range(n)}}
    gs = spg_loader.GraphStore().add(node_gt, node_gt_size, edges, feats, "big").finalize("cuda")
    cs = spg_loader.SuperpointStore()
    cs.add("big", parsed["big"])
    cs.finalize("cuda")
    graphs = [("big", n, edges, node_gt_size.sum(1), np.concatenate([node_gt, node_gt_size], 1), feats)]
    args = SimpleNamespace(**dict(ARGS, spg_augm_hardcutoff=5000, spg_augm_nneigh=50, spg_augm_order=3,
                                  ptn_minpts=20, ptn_npts=32))
    _compare(spg_loader.load_batch(gs, cs, ["big"], True, args, device_rng=True, seed=3),
             rref.build_batch(graphs, parsed, True, args, 3), "big")


def _batch(gs, cs, names, train, args, **kw):
    from superpoint_graph_b200 import spg_loader

    t, GIs, (m, fl, c, cg) = spg_loader.load_batch(gs, cs, names, train, args, device_rng=True, **kw)
    return [t, GIs[0]._idxn, GIs[0]._degrees_gpu, GIs[0]._edgefeats, c, cg], [x for x, f in zip(m, fl) if f == 0]


@pytest.mark.gpu
def test_seed_and_position_key_the_draws():
    g, meta = _golden()
    gs, cs = _stores(g, meta)
    args = SimpleNamespace(**ARGS)
    a, b = meta["rooms"][0]["name"], meta["rooms"][1]["name"]
    x, mx = _batch(gs, cs, [a, b], True, args, seed=7)
    y, _ = _batch(gs, cs, [a, b], True, args, seed=7)
    assert all(torch.equal(p, q) for p, q in zip(x, y))
    z, _ = _batch(gs, cs, [a, b], True, args, seed=8)
    assert not torch.equal(x[0], z[0]) or not torch.equal(x[4], z[4])
    # a graph listed twice gets different draws at each position
    from superpoint_graph_b200 import ops

    n = gs.file(a)["n"]
    p0, c0 = ops.batch_draw(n, 7, 0, True, 8, "cuda")
    p1, c1 = ops.batch_draw(n, 7, 1, True, 8, "cuda")
    assert not torch.equal(p0, p1) and not torch.equal(c0, c1)
    w, mw = _batch(gs, cs, [a, a], True, args, seed=7)
    first, second = {}, {}  # ids are unique within a graph, so an id seen again is from position 1
    for i, k in enumerate(mw):
        (second if k in first else first)[k] = w[4][i]
    assert second and all(not torch.equal(first[k], second[k]) for k in second)


@pytest.mark.gpu
def test_evaluation_clouds_depend_on_id_and_offset_only():
    g, meta = _golden()
    gs, cs = _stores(g, meta)
    args = SimpleNamespace(**ARGS)
    a, b = meta["rooms"][0]["name"], meta["rooms"][1]["name"]
    x, mx = _batch(gs, cs, [a, b], False, args, seed=1, test_seed_offset=0)
    y, my = _batch(gs, cs, [b, a], False, args, seed=1, test_seed_offset=0)
    cx, cy = dict(zip(mx, x[4])), dict(zip(my, y[4]))
    assert set(cx) == set(cy) and all(torch.equal(cx[k], cy[k]) for k in cx)
    z, mz = _batch(gs, cs, [a, b], False, args, seed=1, test_seed_offset=2)
    assert mz == mx and not torch.equal(z[4], x[4])
    assert torch.equal(x[0], z[0])  # no graph draws in evaluation


@pytest.mark.gpu
def test_host_generators_untouched():
    g, meta = _golden()
    gs, cs = _stores(g, meta)
    random.seed(3)
    np.random.seed(3)
    py, npst = random.getstate(), np.random.get_state()
    _batch(gs, cs, [r["name"] for r in meta["rooms"][:2]], True, SimpleNamespace(**ARGS), seed=2)
    _batch(gs, cs, [r["name"] for r in meta["rooms"][:2]], False, SimpleNamespace(**ARGS), seed=2)
    st = np.random.get_state()
    assert random.getstate() == py and all(np.array_equal(p, q) for p, q in zip(st[1:], npst[1:]))


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


@pytest.mark.gpu
def test_one_synchronisation_per_batch():
    g, meta = _golden()
    gs, cs = _stores(g, meta)
    args = SimpleNamespace(**ARGS)
    rooms = [r["name"] for r in meta["rooms"]]
    _syncs(lambda: _batch(gs, cs, rooms[:1], True, args, seed=0))  # torch reports one extra in its first block
    one = _syncs(lambda: _batch(gs, cs, rooms[:1], True, args, seed=0))
    four = _syncs(lambda: _batch(gs, cs, [rooms[0], rooms[1], rooms[0], rooms[1]], True, args, seed=0))
    evl = _syncs(lambda: _batch(gs, cs, rooms[:2], False, args, seed=0))
    assert (one, four, evl) == (1, 1, 1)


@pytest.mark.gpu
def test_collate_exceptions():
    g, meta = _golden()
    args = SimpleNamespace(**ARGS)
    a, b = meta["rooms"][0]["name"], meta["rooms"][1]["name"]
    from superpoint_graph_b200 import spg_loader

    gs, cs = _stores(g, meta)
    # a graph without edges: first, and alone
    node_gt, node_gt_size, _, feats = _room(g, 0)
    gs2 = spg_loader.GraphStore()
    gs2.add(node_gt, node_gt_size, np.zeros((0, 2), np.int64), feats[:0], "bare")
    gs2.add(*_room(g, 0), a)
    gs2.finalize("cuda")
    cs2 = spg_loader.SuperpointStore()
    cs2.add("bare", _parsed_all(g, meta)[a])
    cs2.add(a, _parsed_all(g, meta)[a])
    cs2.finalize("cuda")
    with pytest.raises(RuntimeError):
        spg_loader.load_batch(gs2, cs2, ["bare"], True, args, device_rng=True)
    with pytest.raises(TypeError):
        spg_loader.load_batch(gs2, cs2, ["bare", a], True, args, device_rng=True)
    # every cloud below ptn_minpts
    with pytest.raises(TypeError):
        spg_loader.load_batch(gs, cs, [a], True, SimpleNamespace(**dict(ARGS, ptn_minpts=10 ** 6)), device_rng=True)
    # a superpoint the store lacks, in a batch that keeps every vertex
    gs3, cs3 = _stores(g, meta, skip=(b, 3))
    with pytest.raises(KeyError):
        spg_loader.load_batch(gs3, cs3, [a, b], False, args, device_rng=True)
    spg_loader.load_batch(gs3, cs3, [a], False, args, device_rng=True)


@pytest.mark.gpu
def test_training_step_on_device_rng_batch_matches_oracle_batch():
    """main.py:199-213 with the drop-in modules on the device_rng batch and on the oracle's batch of the same
    draws, collated on the host: set_info(GIs, cuda), CloudEmbedder.run, cross-entropy, backward."""
    from superpoint_graph_b200 import spg_loader
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_pointnet import CloudEmbedder
    from superpoint_graph_b200.trainer import create_model, make_args

    g, meta = _golden()
    gs, cs = _stores(g, meta)
    args = SimpleNamespace(**ARGS)
    rooms = [0, 1]
    names = [meta["rooms"][i]["name"] for i in rooms]
    ref = rref.build_batch(_oracle_graphs(g, meta, rooms), _parsed_all(g, meta), True, args, 21)
    margs = make_args(model_config="gru_10_1_1_1_0,f_13", node_feats=7, ptn_nfeat_stn=7, edge_feats=13)
    torch.manual_seed(4)
    model = create_model(margs).cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    targets, GIs, clouds_data = spg_loader.load_batch(gs, cs, names, True, args, device_rng=True, seed=21)
    ref_gi = GraphConvInfo.from_arrays(ref[1], ref[2], ref[3])
    ref_clouds = (ref[5], torch.from_numpy(ref[6]), torch.from_numpy(ref[7]), torch.from_numpy(ref[8]))
    runs = []
    for tg, gis, cd in ((targets, GIs, clouds_data), (torch.from_numpy(ref[0]), [ref_gi], ref_clouds)):
        model.load_state_dict(state)
        model.train()
        model.zero_grad()
        embedder = CloudEmbedder(margs)
        model.ecc.set_info(gis, True)
        label_mode = tg[:, 0].cuda()
        outputs = model.ecc(embedder.run(model, *cd))
        loss = torch.nn.functional.cross_entropy(outputs, label_mode)
        loss.backward()
        embedder.bw_hook()
        runs.append((outputs.detach(), loss.detach()))
    (o_dev, l_dev), (o_ref, l_ref) = runs
    assert torch.isfinite(l_dev) and o_dev.shape == o_ref.shape
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
    assert rel(o_dev, o_ref) < 1e-4 and rel(l_dev, l_ref) < 1e-4
