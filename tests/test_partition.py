"""The learned partition's objective and evaluation (superpoint_graph_b200.spg_partition, csrc/partition.cu).

CPU: the oracle (oracle/partition_ref.py) against the reference's own outputs (partition.npz, from the unmodified
source text of losses.py / provider.py / metrics.py): integers and masks exactly, weights exactly, distances,
losses and gradients at 1e-6 relative; the C-ABI symbols and kernel names.
GPU: every public function against the golden and against the float64 oracle (integers, masks, components and
weights bit-exact; losses 1e-6 relative; embedding gradients <= 1e-5 of the tensor maximum), bit-identical
repeats at the benchmark size, and a full learned-partition step from LocalCloudEmbedder to the gradients.
"""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import partition_ref as pref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "partition.npz")


def _golden():
    z = np.load(GOLDEN, allow_pickle=False)
    return {k: z[k] for k in z.files}


def _meta(g):
    return json.loads(str(g["meta"]))


def _components(pic):
    return [np.nonzero(pic == c)[0].astype(np.uint32) for c in range(int(pic.max()) + 1)]


def _args(**kw):
    a = dict(loss_weight="crosspartition", loss="TVH_zhang", dist_type="euclidian", transition_factor=5.0,
             k_nn_adj=5, edge_weight_threshold=-0.5, spatial_emb=0, reg_strength=1.0, CP_cutoff=10, cuda=1)
    a.update(kw)
    return SimpleNamespace(**a)


def _close(a, b, rtol, what=""):
    """max |a - b| <= rtol * max |b|, NaNs at the same places."""
    a = torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a), dtype=torch.float64)
    b = torch.as_tensor(np.asarray(b.detach().cpu() if torch.is_tensor(b) else b), dtype=torch.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN pattern differs" % what
    a, b = a[~na], b[~nb]
    if b.numel() == 0:
        return
    err = float((a - b).abs().max())
    scale = float(b.abs().max())
    assert err <= rtol * max(scale, 1e-30), "%s: max err %g vs scale %g" % (what, err, scale)


def _cases(g):
    return _meta(g)["cases"]


# ------------------------------------------------------------------------------------------------- CPU
def test_golden_records_numpy_version():
    m = _meta(_golden())
    assert m["numpy"].split(".")[0] == np.__version__.split(".")[0], "float32/float64 promotion is numpy-2's"


def test_oracle_reproduces_golden():
    g = _golden()
    m = _meta(g)
    for c in _cases(g):
        p = c + "."
        src, tgt, is_tr, pic = g[p + "src"], g[p + "tgt"], g[p + "is_tr"], g[p + "pic"].astype(np.uint32)
        V = g[p + "emb"].shape[0]
        emb0 = torch.from_numpy(g[p + "emb"])
        comps = _components(pic)
        for dt in m["dist_types"]:
            _close(pref.compute_dist(emb0, src, tgt, dt), g[p + "diff." + dt], 1e-6, p + dt)
            for loss in m["losses"]:
                key = "%s.%s" % (dt, loss)
                emb = emb0.clone().requires_grad_(True)
                l1, l2 = pref.compute_loss(_args(loss=loss, dist_type=dt), pref.compute_dist(emb, src, tgt, dt),
                                           torch.from_numpy(is_tr), torch.from_numpy(g[p + "w.crosspartition"]))
                (l1 + l2).backward()
                _close(l1, g[p + "loss1." + key], 1e-6, p + key)
                _close(l2, g[p + "loss2." + key], 1e-6, p + key)
                _close(emb.grad, g[p + "grad." + key], 1e-6, p + key)
        for scheme in m["schemes"]:
            want = g[p + "w." + scheme]
            args = _args(loss_weight=scheme)
            if want.dtype.kind == "U":
                with pytest.raises(ZeroDivisionError):
                    pref.compute_weight_loss(args, g[p + "obj"], src, tgt, is_tr, (comps, pic))
                continue
            got = pref.compute_weight_loss(args, g[p + "obj"], src, tgt, is_tr, (comps, pic))
            assert got.dtype == want.dtype and np.array_equal(got, want), p + scheme
        diff = torch.from_numpy(g[p + "diff.euclidian"])
        for thr in (-0.5, 2.0):
            want = g[p + "edge_weight.%g" % thr]
            got = pref.partition_edge_weight(_args(edge_weight_threshold=thr), diff)
            assert got.dtype == want.dtype and np.array_equal(got, want), thr
        pred_tr = g[p + "pred_tr"]
        for tol in (1, 2):
            rp = pref.relax_edge_binary(pred_tr, src, tgt, V, tol)
            rt = pref.relax_edge_binary(torch.from_numpy(is_tr), src, tgt, V, tol)
            assert np.array_equal(rp, g[p + "relax_pred.%d" % tol]) and np.array_equal(rt, g[p + "relax_tr.%d" % tol])
            n, d = pref.boundary_counts(is_tr, rp)
            with np.errstate(invalid="ignore", divide="ignore"):
                np.testing.assert_equal(100 * np.int64(n) / np.int64(d), g[p + "BR.%d" % tol])
                n, d = pref.boundary_counts(pred_tr, rt)
                np.testing.assert_equal(100 * np.int64(n) / np.int64(d), g[p + "BP.%d" % tol])
        assert np.array_equal(pref.perfect_prediction(comps, g[p + "labels"]), g[p + "perfect"])
        inx, sizes = pref.xpart_components(pic, src, tgt, is_tr)
        assert np.array_equal(inx, g[p + "in_comp_x"]) and np.array_equal(sizes, g[p + "comp_x_size"])


def test_relax_indexing_is_the_references():
    """losses.py:184 indexes with the uint8 vertex marks: it sets edges 0 and 1, not the edges at marked sources."""
    src, tgt = np.array([0, 1, 2, 3, 4]), np.array([1, 2, 3, 4, 0])
    r = pref.relax_edge_binary(np.array([0, 0, 0, 1, 0], dtype=np.uint8), src, tgt, 5, 1)
    # marks 3 and 4; edge 3 (3->4) and 2 (2->3) by target; edges 0 and 1 by the uint8 index
    assert r.tolist() == [1, 1, 1, 1, 0]


def test_loss_kinds_follow_the_reference_order():
    from superpoint_graph_b200.spg_partition import loss_kinds
    assert loss_kinds("TVH_zhang") == ("TVH", "zhang")
    assert loss_kinds("tv_TVminus") == ("tv", "TVminus")
    assert loss_kinds("laplacian_zhang") == ("laplacian", "zhang")
    assert loss_kinds("TVH_TVminus") == ("TVH", "TVminus")
    with pytest.raises(ValueError, match="unknown argument of parameter --loss"):
        loss_kinds("huber_zhang")
    for name in ("TVH_zhang", "tv_zhang", "laplacian_TVminus", "TVH"):
        assert pref.loss_kinds(name) == loss_kinds(name), name


def test_abi_symbols_and_kernel_names_with_one_lp_workspace_query():
    from superpoint_graph_b200 import _lib
    names = ["spg_lp_workspace", "spg_lp_incidence", "spg_lp_dist_fwd", "spg_lp_dist_bwd",
             "spg_lp_loss_partials", "spg_lp_loss_fwd", "spg_lp_loss_bwd", "spg_lp_xpart", "spg_lp_seal",
             "spg_lp_fill_weights", "spg_lp_count", "spg_lp_edge_weight", "spg_lp_relax",
             "spg_lp_perfect_prediction"]
    protos = _lib.protos()
    lib = _lib.lib()
    for n in names:
        assert n in protos, n
        assert getattr(lib, n) is not None
    kn = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("lp_incidence", "lp_dist_fwd", "lp_dist_bwd", "lp_loss_fwd", "lp_loss_bwd", "lp_cc", "lp_xpart",
              "lp_seal", "lp_weights", "lp_relax", "lp_metrics"):
        assert k in kn, k


def test_unknown_dist_type_raises_the_references_error():
    from superpoint_graph_b200.spg_partition import compute_dist
    with pytest.raises(ValueError, match=" cosine is an unknown argument of parameter --dist_type"):
        compute_dist(torch.zeros(2, 4), np.zeros(1, np.int64), np.zeros(1, np.int64), "cosine")


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _grad_close(got, want, what):
    """<= 1e-5 of the tensor maximum, NaNs at the same places."""
    _close(got, want, 1e-5, what)


@pytest.mark.gpu
def test_device_against_golden_and_float64_oracle(dev):
    from superpoint_graph_b200 import spg_partition as sp
    g = _golden()
    m = _meta(g)
    for c in _cases(g):
        p = c + "."
        src, tgt, is_tr, pic = g[p + "src"], g[p + "tgt"], g[p + "is_tr"], g[p + "pic"]
        V = g[p + "emb"].shape[0]
        is_tr_t = torch.from_numpy(is_tr)  # graph_collate gives a CPU tensor; supervized_partition moves it
        comps = _components(pic)
        emb64 = torch.from_numpy(g[p + "emb"]).double()
        for dt in m["dist_types"]:
            diff = sp.compute_dist(torch.from_numpy(g[p + "emb"]).to(dev), src, tgt, dt)
            _close(diff, g[p + "diff." + dt], 1e-6, p + dt)
            _close(diff, pref.compute_dist(emb64, src, tgt, dt), 1e-6, p + dt + " f64")
            w = torch.from_numpy(g[p + "w.crosspartition"])
            for loss in m["losses"]:
                key = p + "%s.%s" % (dt, loss)
                args = _args(loss=loss, dist_type=dt)
                emb = torch.from_numpy(g[p + "emb"]).to(dev).requires_grad_(True)
                l1, l2 = sp.compute_loss(args, sp.compute_dist(emb, src, tgt, dt), is_tr_t.to(dev), w.to(dev))
                assert l1.dim() == 0 and l1.is_cuda and l1.dtype == torch.float32
                (l1 + l2).backward()
                e64 = emb64.clone().requires_grad_(True)
                o1, o2 = pref.compute_loss(args, pref.compute_dist(e64, src, tgt, dt), is_tr_t, w.double())
                (o1 + o2).backward()
                for got, gold, ora, name in ((l1, "loss1.", o1, "loss1"), (l2, "loss2.", o2, "loss2")):
                    _close(got, g[p + gold + "%s.%s" % (dt, loss)], 1e-6, key + name)
                    _close(got, ora, 1e-6, key + name + " f64")
                _grad_close(emb.grad, g[p + "grad.%s.%s" % (dt, loss)], key + " grad")
                _grad_close(emb.grad, e64.grad, key + " grad f64")
        diff = torch.from_numpy(g[p + "diff.euclidian"]).to(dev)
        emb = torch.from_numpy(g[p + "emb"]).to(dev)
        for scheme in m["schemes"]:
            want = g[p + "w." + scheme]
            args = _args(loss_weight=scheme)
            objects = torch.from_numpy(g[p + "obj"]).to(dev)
            if want.dtype.kind == "U":
                with pytest.raises(ZeroDivisionError):
                    sp.compute_weight_loss(args, emb, objects, src, tgt, is_tr_t, diff, False, partition=(comps, pic))
                continue
            got, pc, pi = sp.compute_weight_loss(args, emb, objects, src, tgt, is_tr_t.to(dev), diff, True,
                                                 partition=(comps, pic))
            assert got.is_cuda and got.dtype == torch.float32 and pi is pic
            assert np.array_equal(got.cpu().numpy(), want), p + scheme
        # crosspartition components, sizes and count
        from superpoint_graph_b200 import ops
        e_s, e_t = torch.from_numpy(src).to(dev), torch.from_numpy(tgt).to(dev)
        _, inx, size, ncomp = ops.lp_xpart(e_s, e_t, is_tr_t.to(dev), torch.from_numpy(pic).to(dev), V, 50.0)
        n = int(ncomp[0])
        assert n == len(g[p + "comp_x_size"])
        assert np.array_equal(inx.cpu().numpy(), g[p + "in_comp_x"])
        assert np.array_equal(size[:n].cpu().numpy(), g[p + "comp_x_size"])
        _, wc = ops.lp_seal(e_s, e_t, is_tr_t.to(dev), torch.from_numpy(pic).to(dev),
                            torch.from_numpy(g[p + "obj"]).to(dev), len(comps), 5.0)
        want_wc = [len(cc) - pref.mode_frequency(g[p + "obj"][cc]) for cc in comps]
        assert wc.cpu().tolist() == want_wc
        for thr in (-0.5, 2.0):
            want = g[p + "edge_weight.%g" % thr]
            got = sp.partition_edge_weight(_args(edge_weight_threshold=thr), diff)
            assert got.dtype == want.dtype
            if thr > 0:
                assert np.array_equal(got, want)
            else:  # expf on the device against torch's CPU exp: a float32 ulp
                _close(got, want, 2e-7, "edge weight")
        pred_tr = g[p + "pred_tr"]
        for tol in (1, 2):
            rp = sp.relax_edge_binary(torch.from_numpy(pred_tr).to(dev), src, tgt, V, tol)
            rt = sp.relax_edge_binary(is_tr_t, src, tgt, V, tol)
            assert rp.dtype == torch.bool and rt.dtype == torch.uint8
            assert np.array_equal(rp.cpu().numpy(), g[p + "relax_pred.%d" % tol])
            assert np.array_equal(rt.cpu().numpy(), g[p + "relax_tr.%d" % tol])
            np.testing.assert_equal(sp.compute_boundary_recall(is_tr_t.to(dev), rp), g[p + "BR.%d" % tol])
            np.testing.assert_equal(sp.compute_boundary_precision(rt, torch.from_numpy(pred_tr).to(dev)),
                                    g[p + "BP.%d" % tol])
        per = sp.perfect_prediction(comps, g[p + "labels"])
        assert np.array_equal(per.cpu().numpy(), g[p + "perfect"].astype(np.int64))
        from superpoint_graph_b200.spg_metrics import ConfusionMatrix
        cm_dev, cm_ref = ConfusionMatrix(13), ConfusionMatrix(13)
        cm_dev.count_predicted_batch(g[p + "labels"][:, 1:], per.cpu().numpy())
        cm_ref.count_predicted_batch(g[p + "labels"][:, 1:], g[p + "perfect"])
        assert np.array_equal(cm_dev.confusion_matrix, cm_ref.confusion_matrix)


@pytest.mark.gpu
def test_edge_cases(dev):
    from superpoint_graph_b200 import spg_partition as sp
    args = _args()
    emb = torch.nn.functional.normalize(torch.randn(5, 4)).to(dev).requires_grad_(True)
    # zero edges: empty sums are 0, the gradient is 0
    e0 = np.zeros(0, np.int64)
    d = sp.compute_dist(emb, e0, e0, "euclidian")
    w = sp.compute_weight_loss(_args(loss_weight="crosspartition"), emb, torch.zeros(5, dtype=torch.int64), e0, e0,
                               torch.zeros(0, dtype=torch.uint8), d, False,
                               partition=(_components(np.arange(5)), np.arange(5)))
    l1, l2 = sp.compute_loss(args, d, torch.zeros(0, dtype=torch.uint8), w)
    assert float(l1.detach()) == 0.0 and float(l2.detach()) == 0.0
    (l1 + l2).backward()
    assert torch.equal(emb.grad, torch.zeros_like(emb))
    # one edge: losses.py:184 needs edge 1 when a source is marked -> numpy's IndexError
    with pytest.raises(IndexError):
        sp.relax_edge_binary(np.array([1], np.uint8), np.array([0]), np.array([1]), 5, 1)
    # the reference's --loss without an inter term leaves loss2 unbound
    with pytest.raises(UnboundLocalError):
        sp.compute_loss(_args(loss="TVH"), d, torch.zeros(0, dtype=torch.uint8), w)
    with pytest.raises(RuntimeError, match="libcp"):
        sp.compute_weight_loss(args, emb, torch.zeros(5, dtype=torch.int64), e0, e0, torch.zeros(0), d, True)


def _bench_graph(V, k, n_obj, seed, dev):
    """Random learned-partition batch on the device: k neighbours per vertex in a window of the vertex order,
    objects and predicted components as runs of vertices."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    src = torch.arange(V).repeat_interleave(k)
    tgt = (src + torch.randint(1, 40, (V * k,), generator=gen)) % V
    obj = torch.div(torch.arange(V) * n_obj, V, rounding_mode="floor")
    obj = obj ^ (torch.rand(V, generator=gen) < 0.02).long()
    pic = torch.div(torch.arange(V) + torch.randint(0, 3, (V,), generator=gen), 37, rounding_mode="floor")
    is_tr = (obj[src] != obj[tgt]).to(torch.uint8)
    emb = torch.nn.functional.normalize(torch.randn(V, 4, generator=gen))
    return dict(src=src.to(dev), tgt=tgt.to(dev), obj=obj.to(dev), pic=pic, is_tr=is_tr.to(dev), emb=emb.to(dev))


def _objective(b, args):
    from superpoint_graph_b200 import spg_partition as sp
    emb = b["emb"].clone().requires_grad_(True)
    diff = sp.compute_dist(emb, b["src"], b["tgt"], args.dist_type)
    comps = None
    w = sp.compute_weight_loss(args, emb, b["obj"], b["src"], b["tgt"], b["is_tr"], diff, False,
                               partition=(comps, b["pic"]))
    l1, l2 = sp.compute_loss(args, diff, b["is_tr"], w)
    loss = (l1 + l2) / w.shape[0] * 1000
    loss.backward()
    return diff.detach(), w, l1.detach(), l2.detach(), emb.grad


@pytest.mark.gpu
@pytest.mark.parametrize("dist_type", ["euclidian", "intrinsic"])
def test_bit_identical_at_benchmark_size(dev, dist_type):
    """5 x 10^4 vertices, 2.5 x 10^5 edges: two calls give the same bits; the weights equal the oracle's."""
    b = _bench_graph(50000, 5, 60, 1, dev)
    args = _args(dist_type=dist_type)
    r1 = _objective(b, args)
    r2 = _objective(b, args)
    for x, y in zip(r1, r2):
        assert torch.equal(x, y)
    pic = b["pic"].numpy()
    want = pref.compute_weights_XPART(None, pic, None, b["src"].cpu().numpy(), b["tgt"].cpu().numpy(),
                                      b["is_tr"].cpu().numpy(), 50.0)
    assert np.array_equal(r1[1].cpu().numpy(), want)
    # against float64
    e64 = b["emb"].double().cpu().requires_grad_(True)
    d64 = pref.compute_dist(e64, b["src"].cpu(), b["tgt"].cpu(), dist_type)
    o1, o2 = pref.compute_loss(args, d64, b["is_tr"].cpu(), torch.from_numpy(want).double())
    ((o1 + o2) / len(want) * 1000).backward()
    _close(r1[2], o1, 1e-6, "loss1")
    _close(r1[3], o2, 1e-6, "loss2")
    _grad_close(r1[4], e64.grad, "grad")


@pytest.mark.gpu
def test_seal_and_proportional_at_benchmark_size(dev):
    b = _bench_graph(50000, 5, 60, 2, dev)
    pic = b["pic"].numpy()
    comps = _components(pic)
    from superpoint_graph_b200 import spg_partition as sp
    s, t, tr, obj = (b[k].cpu().numpy() for k in ("src", "tgt", "is_tr", "obj"))
    for scheme in ("seal", "proportional"):
        args = _args(loss_weight=scheme)
        got = sp.compute_weight_loss(args, b["emb"], b["obj"], b["src"], b["tgt"], b["is_tr"],
                                     torch.zeros(len(s), device=dev), False, partition=(comps, pic))
        want = pref.compute_weight_loss(args, obj, s, t, tr, (comps, pic))
        assert np.array_equal(got.cpu().numpy(), want), scheme


def _lp_models(dev):
    from superpoint_graph_b200.spg_pointnet import PointNet, STNkD
    torch.manual_seed(4)
    model = torch.nn.Module()
    model.stn = STNkD(2, [16, 64], [32, 16], norm="layer", n_group=1)
    model.ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=0, nfeat_global=11 + 4,
                         norm="layer", n_group=1)
    torch.manual_seed(5)
    with torch.no_grad():
        model.stn.proj.weight.normal_(0, 0.1)
    sd_s = {k: v.clone().double() for k, v in model.stn.state_dict().items()}
    sd_p = {k: v.clone().double() for k, v in model.ptn.state_dict().items()}
    model.to(dev).train()
    return model, sd_s, sd_p


@pytest.mark.gpu
def test_learned_partition_step_vs_oracle(dev):
    """LocalCloudEmbedder -> compute_dist -> compute_weight_loss(partition=...) -> compute_loss -> backward
    (supervized_partition.py:218-230), against the float64 oracle composition (norm='layer', whose oracle is
    oracle/pointnet_gn_ref.py).  Loss 1e-5; parameter gradients within the bounds of test_group_norm.py."""
    import torch.nn.functional as F
    from oracle import pointnet_gn_ref as gref
    from superpoint_graph_b200 import spg_partition as sp
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder
    model, sd_s, sd_p = _lp_models(dev)
    V = 3000
    b = _bench_graph(V, 5, 20, 3, dev)
    torch.manual_seed(6)
    clouds, glob = torch.randn(V, 6, 20) * 0.5, torch.randn(V, 11)
    args = _args()
    pic = b["pic"].numpy()
    part = (_components(pic), pic)
    emb_mod = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    embeddings = emb_mod.run_batch(model, clouds.to(dev), glob.to(dev))
    diff = sp.compute_dist(embeddings, b["src"], b["tgt"], args.dist_type)
    w, _, _ = sp.compute_weight_loss(args, embeddings, b["obj"], b["src"], b["tgt"], b["is_tr"], diff, True,
                                     partition=part)
    l1, l2 = sp.compute_loss(args, diff, b["is_tr"], w)
    loss = (l1 + l2) / w.shape[0] * 1000
    loss.backward()
    # float64 oracle
    sd_s64 = {k: v.clone().requires_grad_(True) for k, v in sd_s.items()}
    sd_p64 = {k: v.clone().requires_grad_(True) for k, v in sd_p.items()}
    x = clouds.double()
    T = gref.stn_forward(x[:, :2], sd_s64, "", 2, 2, 1)
    xy = torch.bmm(x[:, :2].transpose(1, 2), T).transpose(1, 2)
    pcfg = dict(n_conv=2, n_fc=4, n_conv_stn=0, n_fc_stn=0, nfeat_stn=0, prelast_do=0)
    e64 = F.normalize(gref.pointnet_forward(torch.cat([xy, x[:, 2:]], 1), torch.cat([glob.double(), T.view(-1, 4)], 1),
                                            sd_p64, pcfg, 1))
    s, t = b["src"].cpu(), b["tgt"].cpu()
    w_ref = pref.compute_weight_loss(args, b["obj"].cpu().numpy(), s.numpy(), t.numpy(), b["is_tr"].cpu().numpy(),
                                     part)
    assert np.array_equal(w.cpu().numpy(), w_ref)
    o1, o2 = pref.compute_loss(args, pref.compute_dist(e64, s, t, args.dist_type), b["is_tr"].cpu(),
                               torch.from_numpy(w_ref).double())
    ref_loss = (o1 + o2) / len(w_ref) * 1000
    ref_loss.backward()
    _close(loss, ref_loss, 1e-5, "loss")
    got = {"stn." + k: p.grad for k, p in model.stn.named_parameters()}
    got.update({"ptn." + k: p.grad for k, p in model.ptn.named_parameters()})
    want = {"stn." + k: v.grad for k, v in sd_s64.items() if v.grad is not None}
    want.update({"ptn." + k: v.grad for k, v in sd_p64.items() if v.grad is not None})
    for k, wv in want.items():
        gk = got[k].detach().double().cpu()
        scale = max(float(wv.abs().max()), 1e-12)
        tol = 5e-2 if (k.startswith("ptn.convs.") or k.startswith("stn.convs.")) else 3e-3
        assert float((gk - wv).abs().max()) <= tol * scale + 1e-7, k
