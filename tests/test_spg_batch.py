"""The superpoint graph's batch builder (superpoint_graph_b200.spg_loader.GraphStore / load_batch, csrc/spg_batch.cu).

CPU: the oracle (oracle/spg_batch_ref.py) against the reference's own outputs (spg_batch.npz, from the unmodified
source text of loader / eccpc_collate / GraphConvInfo.set_batch on the compat igraph) bit for bit; the product's host
draws against the reference's draw for draw, with both generators' states after every case; host validation.
GPU: every golden case (vertices, targets and clouds bit for bit, edges equal to the stable-order collate and, per
target, to the reference's collate as multisets, generator states, the collate's exceptions, and in the cases where
the collate raises, the device's selection against the reference's kept vertices); a 10^5-vertex / 10^6-edge graph
against the oracle; repeatability and an unchanged store; main.py's training-step body on the device batch and on
the reference's collated batch.
"""
import json
import os
import random
from collections import Counter
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import spg_batch_ref as sref
from superpoint_graph_b200 import spg_loader

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spg_batch.npz")


def _golden():
    z = np.load(GOLDEN, allow_pickle=False)
    g = {k: z[k] for k in z.files}
    return g, json.loads(str(g["meta"]))


def _room(g, i):
    return tuple(g["room%d.%s" % (i, k)] for k in ("node_gt", "node_gt_size", "edges", "edge_feats"))


def _room_name(meta, i):
    return meta["rooms"][i]["name"]


def _parsed(g, i):
    n = g["room%d.node_gt" % i].shape[0]
    return {sp: g["room%d.sp%d" % (i, sp)] for sp in range(n)}


def _seed(case):
    random.seed(case["seed"])
    np.random.seed(case["seed"])


def _states():
    py, st = random.getstate(), np.random.get_state()
    return np.array(py[1], dtype=np.int64), np.concatenate([st[1].astype(np.int64), [st[2], st[3]]])


def _cloud_draws(parsed, ids, args, train, offset):
    """The host draws of load_superpoints (spg_loader.py), made without a device."""
    ncols = len(spg_loader.attrib_columns(args.pc_attribs, 7))
    for s in ids:
        n = parsed[s].shape[0]
        if n < args.ptn_minpts:
            continue
        rs = np.random.random.__self__ if train else np.random.RandomState(seed=int(s) + offset)
        spg_loader.sample_indices(n, args.ptn_npts, rs)
        if train:
            spg_loader.augment_matrix(args)
            if args.pc_augm_jitter:
                np.random.randn(args.ptn_npts, ncols)


def _replay(g, meta, case):
    """The product's host draws and the oracle's selection for one case: [(ids, sub-graph edges) or None]."""
    args = SimpleNamespace(**case["args"])
    _seed(case)
    out = []
    for i in case["rooms"]:
        node_gt, node_gt_size, edges, _ = _room(g, i)
        n = node_gt.shape[0]
        perm, centres, cut = spg_loader.graph_draws(n, case["train"], args)
        ids, sub, _ = sref.sample_graph(n, edges, node_gt_size.sum(1), perm, centres, args.spg_augm_order,
                                        args.ptn_minpts, cut)
        if sub.shape[0]:
            _cloud_draws(_parsed(g, i), ids.tolist(), args, case["train"], case["test_seed_offset"])
            out.append((ids, sub))
        else:
            out.append(None)
    return out


def _per_target(idxn, edge_index, feats):
    c = Counter()
    for s, t, f in zip(idxn.tolist(), edge_index[1].tolist(), feats):
        c[(t, s, f.tobytes())] += 1
    return c


@pytest.fixture(scope="module")
def golden():
    return _golden()


def test_oracle_and_host_draws_match_golden(golden):
    g, meta = golden
    for case in meta["cases"]:
        p = case["tag"] + "."
        picks = _replay(g, meta, case)
        py, npst = _states()
        assert np.array_equal(py, g[p + "py_state"]), case["tag"]
        assert np.array_equal(npst, g[p + "np_state"]), case["tag"]
        assert [x is not None for x in picks] == case["kept"], case["tag"]
        graphs = []
        for b, (x, i) in enumerate(zip(picks, case["rooms"])):
            if x is None:
                continue
            ids, sub = x
            assert np.array_equal(ids, g[p + "ids.%d" % b]), case["tag"]
            assert np.array_equal(sub, g[p + "sub_edges.%d" % b]), case["tag"]
            node_gt, node_gt_size, edges, feats = _room(g, i)
            remap = -np.ones(node_gt.shape[0], dtype=np.int64)
            remap[ids] = np.arange(ids.size)
            keep = (remap[edges[:, 0]] >= 0) & (remap[edges[:, 1]] >= 0)
            graphs.append((np.concatenate([node_gt, node_gt_size], 1)[ids], sub, feats[keep]))
        if case["error"] is not None:
            continue
        targets, idxn, degs, feats, edge_index = sref.collate(graphs, kind="quicksort")
        assert np.array_equal(targets, g[p + "targets"])
        assert np.array_equal(idxn, g[p + "idxn"]) and np.array_equal(degs, g[p + "degs"])
        assert np.array_equal(feats, g[p + "edgefeats"]) and np.array_equal(edge_index, g[p + "edge_index"])
        # the stable order is the same multiset per target
        _, idxn_s, degs_s, feats_s, ei_s = sref.collate(graphs, kind="stable")
        assert np.array_equal(degs_s, degs)
        assert _per_target(idxn_s, ei_s, feats_s) == _per_target(idxn, edge_index, feats)


def test_graph_draws_follow_the_reference_conditions():
    a = SimpleNamespace(spg_augm_hardcutoff=10, spg_augm_nneigh=4)
    random.seed(3)
    perm, centres, cut = spg_loader.graph_draws(20, True, a)
    random.seed(3)
    p2 = list(range(20))
    random.shuffle(p2)
    assert perm == p2 and centres == random.sample(range(20), k=4) and cut == 10
    perm, centres, _ = spg_loader.graph_draws(8, True, a)  # 10 >= 8 and 4 < 8: centres only
    assert perm is None and len(centres) == 4
    random.seed(3)
    state = random.getstate()
    assert spg_loader.graph_draws(20, False, a) == (None, None, 0) and random.getstate() == state


def test_add_validation():
    st = spg_loader.GraphStore()
    gt, gs = np.zeros((4, 1), np.int64), np.ones((4, 3), np.int64)
    e = np.array([[0, 1], [2, 3]])
    f = np.zeros((2, 5), np.float32)
    st.add(gt, gs, e, f, "ok")
    with pytest.raises(IndexError):
        st.add(gt, gs, np.array([[0, 4]]), f[:1], "x")
    with pytest.raises(IndexError):
        st.add(gt, gs, np.array([[-1, 0]]), f[:1], "x")
    with pytest.raises(ValueError):
        st.add(gt, gs, e, f[:1], "x")
    with pytest.raises(ValueError):
        st.add(gt, gs[:3], e, f, "x")
    with pytest.raises(ValueError):
        st.add(gt, gs, np.array([0, 1]), f, "x")
    with pytest.raises(TypeError):
        st.add(gt, gs, e, f.astype(np.float64), "x")
    with pytest.raises(TypeError):
        st.add(gt, gs, e.astype(np.float32), f, "x")
    with pytest.raises(ValueError, match="added already"):
        st.add(gt, gs, e, f, "ok")
    with pytest.raises(ValueError, match="2\\^31"):
        st.add(np.broadcast_to(gt[:1], (2 ** 31, 1)), gs, e, f, "x")


# ------------------------------------------------------------------------------------------------------ GPU

def _stores(g, meta, args):
    gs, cs = spg_loader.GraphStore(), spg_loader.SuperpointStore()
    for i in range(len(meta["rooms"])):
        gs.add(*_room(g, i), _room_name(meta, i))
        cs.add(_room_name(meta, i), _parsed(g, i))
    return gs.finalize("cuda"), cs.finalize("cuda")


@pytest.mark.gpu
def test_golden_cases_on_device(golden):
    g, meta = golden
    gs, cs = _stores(g, meta, None)
    for case in meta["cases"]:
        p = case["tag"] + "."
        args = SimpleNamespace(**case["args"])
        names = [_room_name(meta, i) for i in case["rooms"]]
        _seed(case)
        if case["error"] is not None:
            with pytest.raises(TypeError):
                spg_loader.load_batch(gs, cs, names, case["train"], args, case["test_seed_offset"])
            _check_selection(g, meta, case, gs)
        else:
            targets, GIs, (cmeta, cflag, clouds, cglob) = spg_loader.load_batch(gs, cs, names, case["train"], args,
                                                                                case["test_seed_offset"])
            gi = GIs[0]
            assert targets.is_cuda and gi._idxn.is_cuda and gi._degrees_gpu.is_cuda and gi._edgefeats.is_cuda
            assert np.array_equal(targets.cpu().numpy(), g[p + "targets"]), case["tag"]
            assert cmeta == case["clouds_meta"] and np.array_equal(cflag.numpy(), g[p + "clouds_flag"])
            assert np.array_equal(clouds.cpu().numpy(), g[p + "clouds"]), case["tag"]
            assert np.array_equal(cglob.cpu().numpy(), g[p + "clouds_global"]), case["tag"]
            # edges: equal to the stable-order collate, and per target to the reference's as multisets
            graphs = []
            for b, i in enumerate(case["rooms"]):
                if not case["kept"][b]:
                    continue
                node_gt, node_gt_size, edges, feats = _room(g, i)
                ids = g[p + "ids.%d" % b]
                remap = -np.ones(node_gt.shape[0], dtype=np.int64)
                remap[ids] = np.arange(ids.size)
                keep = (remap[edges[:, 0]] >= 0) & (remap[edges[:, 1]] >= 0)
                graphs.append((np.concatenate([node_gt, node_gt_size], 1)[ids], g[p + "sub_edges.%d" % b],
                               feats[keep]))
            _, idxn, degs, feats, ei = sref.collate(graphs, kind="stable")
            assert np.array_equal(gi._idxn.cpu().numpy(), idxn), case["tag"]
            assert np.array_equal(gi._degrees_gpu.cpu().numpy(), degs), case["tag"]
            assert np.array_equal(gi._edgefeats.cpu().numpy(), feats), case["tag"]
            assert np.array_equal(gi._edge_indexes.cpu().numpy(), ei), case["tag"]
            assert _per_target(gi._idxn.cpu().numpy(), gi._edge_indexes.cpu().numpy(), gi._edgefeats.cpu().numpy()) \
                == _per_target(g[p + "idxn"], g[p + "edge_index"], g[p + "edgefeats"])
            csr = gi.graph().to(gi._idxn.device)
            assert int(csr["tgt_rowptr"][-1]) == ei.shape[1]
        py, npst = _states()
        assert np.array_equal(py, g[p + "py_state"]) and np.array_equal(npst, g[p + "np_state"]), case["tag"]


def _check_selection(g, meta, case, gs):
    """ops.batch_select with the case's replayed draws against the reference's kept vertices and sub-graph edge
    count, graph by graph (the cloud draws in between are replayed on the host)."""
    from superpoint_graph_b200 import ops

    args = SimpleNamespace(**case["args"])
    dev = lambda a: None if a is None else torch.tensor(a, dtype=torch.int32).cuda()
    _seed(case)
    for b, i in enumerate(case["rooms"]):
        f = gs.file(_room_name(meta, i))
        perm, centres, cut = spg_loader.graph_draws(f["n"], case["train"], args)
        _, _, out = ops.batch_select(f["src"], f["tgt"], f["adjacency"], f["s"], dev(perm), dev(centres),
                                     args.spg_augm_order, args.ptn_minpts, cut)
        out = out.cpu().numpy()
        n_kept, n_edges = int(out[0]), int(out[1])
        assert (n_edges > 0) == case["kept"][b], case["tag"]
        if n_edges:
            assert np.array_equal(out[2:2 + n_kept], g[case["tag"] + ".ids.%d" % b]), case["tag"]
            assert n_edges == g[case["tag"] + ".sub_edges.%d" % b].shape[0], case["tag"]
            _cloud_draws(_parsed(g, i), out[2:2 + n_kept].tolist(), args, case["train"], case["test_seed_offset"])


@pytest.mark.gpu
def test_training_step_on_device_batch_matches_reference_batch(golden):
    """main.py:199-213 with the drop-in modules, once on load_batch's batch and once on the reference's collated
    batch of the same case: set_info(GIs, cuda), CloudEmbedder.run, cross-entropy, backward."""
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_pointnet import CloudEmbedder
    from superpoint_graph_b200.trainer import create_model, make_args

    g, meta = golden
    gs, cs = _stores(g, meta, None)
    case = [c for c in meta["cases"] if c["tag"] == "train_both"][0]
    p = case["tag"] + "."
    margs = make_args(model_config="gru_10_1_1_1_0,f_13", node_feats=7, ptn_nfeat_stn=7, edge_feats=13)
    torch.manual_seed(4)
    model = create_model(margs).cuda()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    _seed(case)
    targets, GIs, clouds_data = spg_loader.load_batch(gs, cs, [_room_name(meta, i) for i in case["rooms"]], True,
                                                      SimpleNamespace(**case["args"]))
    ref_gi = GraphConvInfo.from_arrays(g[p + "idxn"], g[p + "degs"], g[p + "edgefeats"])
    ref_clouds = (case["clouds_meta"], torch.from_numpy(g[p + "clouds_flag"]), torch.from_numpy(g[p + "clouds"]),
                  torch.from_numpy(g[p + "clouds_global"]))
    runs = []
    for tg, gis, cd in ((targets, GIs, clouds_data), (torch.from_numpy(g[p + "targets"]), [ref_gi], ref_clouds)):
        model.load_state_dict(state)
        model.train()
        model.zero_grad()
        embedder = CloudEmbedder(margs)
        model.ecc.set_info(gis, True)
        label_mode = tg[:, 0].cuda()
        embeddings = embedder.run(model, *cd)
        outputs = model.ecc(embeddings)
        loss = torch.nn.functional.cross_entropy(outputs, label_mode)
        loss.backward()
        embedder.bw_hook()
        runs.append((outputs.detach(), loss.detach(), {k: q.grad.clone() for k, q in model.named_parameters()}))
    (o_dev, l_dev, g_dev), (o_ref, l_ref, g_ref) = runs
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
    assert o_dev.shape == o_ref.shape and rel(o_dev, o_ref) < 1e-4
    assert rel(l_dev, l_ref) < 1e-4
    assert max(rel(g_dev[k], g_ref[k]) for k in g_ref if g_ref[k].abs().max() > 0) < 1e-3


@pytest.mark.gpu
def test_large_graph_matches_oracle():
    from superpoint_graph_b200 import ops

    rng = np.random.default_rng(5)
    n, E = 100_000, 1_000_000
    edges = rng.integers(0, n, size=(E, 2))
    node_gt = rng.integers(0, 13, size=(n, 1))
    node_gt_size = rng.integers(0, 40, size=(n, 3))
    feats = rng.standard_normal((E, 4)).astype(np.float32)
    gs = spg_loader.GraphStore().add(node_gt, node_gt_size, edges, feats, "big").finalize("cuda")
    f = gs.file("big")
    args = SimpleNamespace(spg_augm_hardcutoff=5000, spg_augm_nneigh=50, spg_augm_order=3, ptn_minpts=40)
    random.seed(9)
    perm, centres, cut = spg_loader.graph_draws(n, True, args)
    s = node_gt_size.sum(1)
    ids, sub, sel = sref.sample_graph(n, edges, s, perm, centres, 3, 40, cut)
    dev = lambda a: torch.tensor(a, dtype=torch.int32).cuda()
    new_index, edge_pos, out = ops.batch_select(f["src"], f["tgt"], f["adjacency"], f["s"], dev(perm), dev(centres),
                                                3, 40, cut)
    out = out.cpu().numpy()
    assert int(out[0]) == ids.size and int(out[1]) == sub.shape[0]
    assert np.array_equal(out[2:2 + ids.size], ids)
    nk, ne = ids.size, sub.shape[0]
    i64 = dict(dtype=torch.int64, device="cuda")
    ei, degs = torch.empty((2, ne), **i64), torch.empty(nk, **i64)
    fo, to = torch.empty((ne, 4), dtype=torch.float32, device="cuda"), torch.empty((nk, 4), **i64)
    ops.batch_edges(f["src"], f["tgt"], new_index, edge_pos, dev(ids), nk, ne, 7, f["feats"], f["targets"], ei[0],
                    ei[1], degs, fo, to)
    targets, idxn, degs_r, feats_r, ei_r = sref.collate([(np.concatenate([node_gt, node_gt_size], 1)[ids], sub,
                                                          feats[sel])], kind="stable")
    assert np.array_equal(ei.cpu().numpy(), ei_r + 7) and np.array_equal(degs.cpu().numpy(), degs_r)
    assert np.array_equal(fo.cpu().numpy(), feats_r) and np.array_equal(to.cpu().numpy(), targets)


@pytest.mark.gpu
def test_repeatable_and_store_unchanged(golden):
    g, meta = golden
    gs, cs = _stores(g, meta, None)
    case = [c for c in meta["cases"] if c["tag"] == "train_both"][0]
    args = SimpleNamespace(**case["args"])
    names = [_room_name(meta, i) for i in case["rooms"]]
    snap = {k: {f: v.clone() for f, v in gs.file(k).items() if torch.is_tensor(v)} for k in names}
    adj = {k: {f: v.clone() for f, v in gs.file(k)["adjacency"].items() if torch.is_tensor(v)} for k in names}
    runs = []
    for _ in range(2):
        _seed(case)
        t, GIs, (m, fl, c, cg) = spg_loader.load_batch(gs, cs, names, True, args)
        runs.append([t, GIs[0]._idxn, GIs[0]._degrees_gpu, GIs[0]._edgefeats, c, cg])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    for k in names:
        for f, v in snap[k].items():
            assert torch.equal(gs.file(k)[f], v)
        for f, v in adj[k].items():
            assert torch.equal(gs.file(k)["adjacency"][f], v)
