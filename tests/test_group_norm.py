"""norm='layer' | 'group' PointNets (nn.GroupNorm, learning/pointnet.py:24-47,75-118) on the device.

CPU: the oracle (oracle/pointnet_gn_ref.py) against the reference's own outputs (pointnet_gn.npz), the
parsing of GroupNorm chains and the state-dict keys of our modules.
GPU, kernel level: ops.group_norm_fwd / group_norm_bwd against float64 F.group_norm and its autograd, 1e-5
relative to the largest value.  The ReLU mask of the float64 backward is the device's (out > 0): an element
whose pre-activation is within float32 rounding of 0 may sit on either side.
GPU, module level: PointNet / LocalCloudEmbedder against the float64 oracle; outputs 1e-4, gradients with the
bounds of test_gpu_shapes.py (point-wise layers sit under a max-pool whose float32 arg-max may pick the other
of two near-tied points).  With GroupNorm no gradient is analytically zero, so none is skipped.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pointnet_gn_ref as gref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pointnet_gn.npz")


def _golden():
    z = np.load(GOLDEN, allow_pickle=False)
    return {k: z[k] for k in z.files}


def _sub(g, prefix, dtype=torch.float64):
    return {k[len(prefix):]: torch.from_numpy(v).to(dtype).clone() for k, v in g.items() if k.startswith(prefix)}


def _close(a, b, rtol, atol=0.0):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all(), "non-finite values"
    err = (a - b).abs().max().item()
    scale = b.abs().max().item()
    assert err <= atol + rtol * scale, "max err %g vs scale %g (rel %g)" % (err, scale, err / max(scale, 1e-30))


def _lp_cases(g):
    return json.loads(str(g["cases"]))["lp"]


def _spg_cases(g):
    return json.loads(str(g["cases"]))["spg"]


def _groups(norm, n_group):
    return 1 if norm == "layer" else n_group


def _spg_pcfg(c, prelast_do=0):
    return dict(n_conv=len(c["nf_conv"]), n_fc=len(c["nf_fc"]), n_conv_stn=len(c["nf_conv_stn"]),
                n_fc_stn=len(c["nf_fc_stn"]), nfeat_stn=c["nfeat_stn"], prelast_do=prelast_do)


LP_PCFG = dict(n_conv=2, n_fc=4, n_conv_stn=0, n_fc_stn=0, nfeat_stn=0, prelast_do=0)


def _lp_embed(clouds, glob, sd_s, sd_p, groups, pcfg=LP_PCFG, drop_mask=None):
    """LocalCloudEmbedder.run_batch (learning/pointnet.py:195-207) on the oracle."""
    T = gref.stn_forward(clouds[:, :2], sd_s, "", 2, 2, groups)
    xy = torch.bmm(clouds[:, :2].transpose(1, 2), T).transpose(1, 2)
    c2 = torch.cat([xy, clouds[:, 2:]], 1)
    g2 = torch.cat([glob, T.view(-1, 4)], 1)
    return F.normalize(gref.pointnet_forward(c2, g2, sd_p, pcfg, groups, drop_mask=drop_mask))


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_reproduces_golden():
    g = _golden()
    for norm, ng in _lp_cases(g):
        tag = "lp_%s%d." % (norm, ng)
        groups = _groups(norm, ng)
        sd_s = {k: v.requires_grad_(True) for k, v in _sub(g, tag + "sd0.stn.").items()}
        sd_p = {k: v.requires_grad_(True) for k, v in _sub(g, tag + "sd0.ptn.").items()}
        x = torch.from_numpy(g[tag + "x"]).double().requires_grad_(True)
        xg = torch.from_numpy(g[tag + "xg"]).double()
        out = _lp_embed(x, xg, sd_s, sd_p, groups)
        _close(out, g[tag + "out_train"], 1e-5)
        _close(out, g[tag + "out_eval"], 1e-5)  # GroupNorm: eval computes what training computes
        out.backward(torch.from_numpy(g[tag + "g"]).double())
        _close(x.grad, g[tag + "grad_x"], 1e-4)
        for pre, sd in (("stn.", sd_s), ("ptn.", sd_p)):
            for k, v in sd.items():
                _close(v.grad, g[tag + "grad." + pre + k], 1e-4, 1e-7)
    c = json.loads(str(g["spg_cfg"]))
    for norm, ng in _spg_cases(g):
        tag = "spg_%s%d." % (norm, ng)
        sd = {k: v.requires_grad_(True) for k, v in _sub(g, tag + "sd0.").items()}
        x, xg = torch.from_numpy(g[tag + "x"]).double(), torch.from_numpy(g[tag + "xg"]).double()
        out = gref.pointnet_forward(x, xg, sd, _spg_pcfg(c), _groups(norm, ng))
        _close(out, g[tag + "out_train"], 1e-5)
        _close(out, g[tag + "out_eval"], 1e-5)
        out.backward(torch.from_numpy(g[tag + "g"]).double())
        for k, v in sd.items():
            _close(v.grad, g[tag + "grad." + k], 1e-4, 1e-7)


def test_oracle_ragged_equal_lengths_is_fixed():
    g = _golden()
    c = json.loads(str(g["spg_cfg"]))
    tag = "spg_group2."
    sd = _sub(g, tag + "sd0.")
    x, xg = torch.from_numpy(g[tag + "x"]).double(), torch.from_numpy(g[tag + "xg"]).double()
    B, Fe, L = x.shape
    pts = x.permute(0, 2, 1).reshape(B * L, Fe)
    offsets = torch.arange(B + 1, dtype=torch.int64) * L
    _close(gref.pointnet_forward_ragged(pts, offsets, xg, sd, _spg_pcfg(c), 2),
           gref.pointnet_forward(x, xg, sd, _spg_pcfg(c), 2), 1e-12)


def test_parse_sequential_groupnorm():
    from superpoint_graph_b200.dense import parse_sequential
    seq = torch.nn.Sequential(torch.nn.Linear(5, 34), torch.nn.GroupNorm(2, 34), torch.nn.ReLU(True),
                              torch.nn.Dropout(0.5), torch.nn.Linear(34, 4))
    specs, params = parse_sequential(seq, True)
    assert len(specs) == 2 and len(params) == 6
    sp = specs[0]
    assert sp.gn is seq[1] and sp.bn is None and sp.relu and sp.drop == 0.5
    assert params[sp.gamma] is seq[1].weight and params[sp.beta] is seq[1].bias
    assert specs[1].gn is None and not specs[1].relu
    specs, _ = parse_sequential(seq, False)
    assert specs[0].drop == 0.0
    with pytest.raises(NotImplementedError):
        parse_sequential(torch.nn.Sequential(torch.nn.Linear(5, 8), torch.nn.GroupNorm(2, 8, affine=False)), True)


def test_state_dict_keys_match_reference():
    from superpoint_graph_b200.spg_pointnet import PointNet, STNkD
    g = _golden()
    c = json.loads(str(g["spg_cfg"]))
    for norm, ng in _spg_cases(g):
        ptn = PointNet(c["nf_conv"], c["nf_fc"], c["nf_conv_stn"], c["nf_fc_stn"], c["nfeat"], c["nfeat_stn"],
                       prelast_do=0, norm=norm, n_group=ng)
        want = {k: v.shape for k, v in _sub(g, "spg_%s%d.sd0." % (norm, ng)).items()}
        assert {k: v.shape for k, v in ptn.state_dict().items()} == want
    for norm, ng in _lp_cases(g):
        tag = "lp_%s%d.sd0." % (norm, ng)
        stn = STNkD(2, [16, 64], [32, 16], norm=norm, n_group=ng)
        ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=0, nfeat_global=15, norm=norm, n_group=ng)
        assert {k: v.shape for k, v in stn.state_dict().items()} == \
            {k: v.shape for k, v in _sub(g, tag + "stn.").items()}
        assert {k: v.shape for k, v in ptn.state_dict().items()} == \
            {k: v.shape for k, v in _sub(g, tag + "ptn.").items()}


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _segments(lens, dev):
    """seg tuple of ragged segments of the given lengths."""
    lens_t = torch.tensor(lens, dtype=torch.int64)
    offsets = torch.zeros(len(lens) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lens_t, 0)
    row_seg = torch.repeat_interleave(torch.arange(len(lens), dtype=torch.int32), lens_t)
    return (len(lens), 0, offsets.to(dev), row_seg.to(dev)), offsets


def _gn_ref(y, bounds, C, G, gamma, beta):
    """float64 F.group_norm of every segment [o0, o1) of the rows y [M, C]."""
    out = torch.empty_like(y)
    for o0, o1 in bounds:
        if o1 > o0:
            out[o0:o1] = F.group_norm(y[o0:o1].t().unsqueeze(0), G, gamma, beta, 1e-5)[0].t()
    return out


def _run_case(dev, lens, C, G, relu, shift=0.0, drop=None, seed=0, fixed=None):
    """Forward and backward of the kernels against float64.  lens: ragged segment lengths, or fixed = (B, L)."""
    from superpoint_graph_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    if fixed is not None:
        B, L = fixed
        seg = (B, L, None, None)
        bounds = [(b * L, (b + 1) * L) for b in range(B)]
        M = B * L
    else:
        seg, offsets = _segments(lens, dev)
        bounds = [(int(offsets[b]), int(offsets[b + 1])) for b in range(len(lens))]
        M = int(offsets[-1])
    y = torch.randn(M, C, generator=gen) + shift
    gamma = torch.rand(C, generator=gen) + 0.5
    beta = torch.randn(C, generator=gen) * 0.3
    gy = torch.randn(M, C, generator=gen)
    d = [t.to(dev) for t in (y, gamma, beta, gy)]
    out, mean, rstd = ops.group_norm_fwd(d[0], C, seg, C, G, d[1], d[2], 1e-5, relu, drop=drop)
    dY, dg, db = ops.group_norm_bwd(d[3], C, d[0], C, mean, rstd, d[1], d[2], seg, C, G, relu, drop=drop)
    y64, g64, b64 = (t.double().requires_grad_(True) for t in (y, gamma, beta))
    a = _gn_ref(y64, bounds, C, G, g64, b64)
    out_c = out.cpu().double()
    want = a.detach()
    if relu:
        want = want.clamp_min(0)
    geff = gy.double()
    if drop is not None:
        keep = ops.dropout_mask(drop[1], drop[0], M, C).cpu().bool()
        want = want * keep / (1 - drop[0])
        geff = geff * keep / (1 - drop[0])
    _close(out_c, want, 1e-5)
    if relu:
        geff = geff * (out_c > 0)
    (a * geff).sum().backward()
    _close(dY, y64.grad, 1e-5)
    _close(dg, g64.grad, 1e-5)
    _close(db, b64.grad, 1e-5)
    return out, mean, rstd, dY, dg, db


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 20, 128])
@pytest.mark.parametrize("C,G", [(34, 2), (128, 2), (64, 1), (128, 8)])
@pytest.mark.parametrize("relu", [True, False])
def test_kernels_fixed_length(dev, L, C, G, relu):
    _run_case(dev, None, C, G, relu, fixed=(97, L), seed=L * 1000 + C + G)


@pytest.mark.gpu
@pytest.mark.parametrize("C,G", [(34, 2), (128, 2), (32, 1)])
def test_kernels_ragged(dev, C, G):
    lens = [0, 1, 5, 20, 0, 128, 3, 10003, 7, 0, 64, 2]
    _run_case(dev, lens, C, G, True, seed=C + G)


@pytest.mark.gpu
@pytest.mark.parametrize("C,G", [(128, 2), (34, 1)])
def test_kernels_large_mean(dev, C, G):
    """mean 1e3, std 1: the variance must not come from E[y^2] - E[y]^2."""
    _run_case(dev, None, C, G, True, shift=1e3, fixed=(61, 20), seed=7)
    _run_case(dev, [20, 0, 300, 1], C, G, False, shift=1e3, seed=8)


@pytest.mark.gpu
def test_kernels_bit_reproducible(dev):
    for lens, C, G in (([20] * 3000, 128, 2), ([0, 1, 5000, 30, 17], 34, 2)):
        a = _run_case(dev, lens, C, G, True, seed=3)
        b = _run_case(dev, lens, C, G, True, seed=3)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("C,G,fixed", [(128, 2, (300, 20)), (34, 2, (513, 1)), (32, 1, (1000, 1))])
def test_kernels_dropout(dev, C, G, fixed):
    """drop(relu(gn(y))) with the Philox mask of the slot at index m*C + c (ops.dropout_mask), and the same mask
    in the backward."""
    slot = torch.tensor([0x5EED5EED, 11], dtype=torch.int64, device=dev)
    out = _run_case(dev, None, C, G, True, drop=(0.5, slot), fixed=fixed, seed=C)[0]
    from superpoint_graph_b200 import ops
    keep = ops.dropout_mask(slot, 0.5, fixed[0] * fixed[1], C).bool()
    assert not out[~keep].any()
    assert 0.4 < float(keep.float().mean()) < 0.6


def _lp_models(norm, ng, dev, prelast_do=0):
    from superpoint_graph_b200.spg_pointnet import PointNet, STNkD
    torch.manual_seed(4)
    model = torch.nn.Module()
    model.stn = STNkD(2, [16, 64], [32, 16], norm=norm, n_group=ng)
    model.ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=prelast_do, nfeat_global=11 + 4,
                         norm=norm, n_group=ng)
    torch.manual_seed(5)
    with torch.no_grad():
        model.stn.proj.weight.normal_(0, 0.1)
        for m in model.modules():
            if isinstance(m, torch.nn.GroupNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    sd_s = {k: v.clone().double() for k, v in model.stn.state_dict().items()}
    sd_p = {k: v.clone().double() for k, v in model.ptn.state_dict().items()}
    model.to(dev).train()
    return model, sd_s, sd_p


def _check_grads(got, want, pointwise):
    """got/want {name: grad}; `pointwise(name)`: a layer under the max-pool (bounds of test_gpu_shapes.py)."""
    for k, w in want.items():
        assert got[k] is not None, k
        gk = got[k].detach().double().cpu()
        scale = max(float(w.abs().max()), 1e-12)
        err = float((gk - w).abs().max())
        tol = 5e-2 if pointwise(k) else 3e-3
        assert err <= tol * scale + 1e-7, "%s: grad err %g vs scale %g (rel %g)" % (k, err, scale, err / scale)
        if pointwise(k) and float(w.norm()) > 0:
            assert float((gk - w).norm() / w.norm()) <= 2e-2, k


@pytest.mark.gpu
@pytest.mark.parametrize("norm,ng", [("layer", 1), ("group", 2)])
@pytest.mark.parametrize("B", [700, 50000])
def test_local_cloud_embedder(dev, norm, ng, B):
    """Learned-partition embedder (supervized_partition.py defaults) with a GroupNorm STN and PointNet: training
    forward, backward to every parameter (the STN's through the xy transform and the global features) and to
    the non-transformed features of the input, and eval."""
    from types import SimpleNamespace
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder
    model, sd_s, sd_p = _lp_models(norm, ng, dev)
    torch.manual_seed(B)
    clouds, glob = torch.randn(B, 6, 20) * 0.5, torch.randn(B, 11)
    gy = torch.randn(B, 4)
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    xd = clouds.to(dev).requires_grad_(True)
    out = emb.run_batch(model, xd, glob.to(dev))
    out.backward(gy.to(dev))
    # float64 oracle, chunked over the clouds (every cloud is independent under GroupNorm)
    sd_s64 = {k: v.clone().requires_grad_(True) for k, v in sd_s.items()}
    sd_p64 = {k: v.clone().requires_grad_(True) for k, v in sd_p.items()}
    outs, gx = [], []
    for i in range(0, B, 10000):
        x = clouds[i:i + 10000].double().requires_grad_(True)
        o = _lp_embed(x, glob[i:i + 10000].double(), sd_s64, sd_p64, _groups(norm, ng))
        o.backward(gy[i:i + 10000].double())
        outs.append(o.detach())
        gx.append(x.grad[:, 2:])
    _close(out, torch.cat(outs), 1e-4)
    # the STN takes no input gradient (its input is data): features 2.. reach the input through the PointNet only,
    # under its max-pool (point-wise bounds)
    got = {"input": xd.grad[:, 2:]}
    _check_grads(got, {"input": torch.cat(gx)}, lambda k: True)
    got = {"stn." + k: p.grad for k, p in model.stn.named_parameters()}
    got.update({"ptn." + k: p.grad for k, p in model.ptn.named_parameters()})
    want = {"stn." + k: v.grad for k, v in sd_s64.items()}
    want.update({"ptn." + k: v.grad for k, v in sd_p64.items()})
    _check_grads(got, want, lambda k: k.startswith("ptn.convs.") or k.startswith("stn.convs."))
    model.eval()
    with torch.no_grad():
        out_e = emb.run_batch(model, clouds.to(dev), glob.to(dev))
    _close(out_e, torch.cat(outs), 1e-4)


def _spg_model(g, norm, ng, dev, prelast_do=0):
    from superpoint_graph_b200.spg_pointnet import PointNet
    c = json.loads(str(g["spg_cfg"]))
    ptn = PointNet(c["nf_conv"], c["nf_fc"], c["nf_conv_stn"], c["nf_fc_stn"], c["nfeat"], c["nfeat_stn"],
                   prelast_do=prelast_do, norm=norm, n_group=ng)
    sd = _sub(g, "spg_%s%d.sd0." % (norm, ng), torch.float32)
    ptn.load_state_dict(sd)
    return ptn.to(dev), {k: v.double() for k, v in sd.items()}, c


def _spg_pointwise(k):
    return k.startswith("convs.") or k.startswith("stn.")


@pytest.mark.gpu
@pytest.mark.parametrize("norm,ng", [("layer", 1), ("group", 2), ("group", 4)])
def test_pointnet_train_eval_vs_oracle(dev, norm, ng):
    g = _golden()
    ptn, sd, c = _spg_model(g, norm, ng, dev)
    tag = "spg_%s%d." % (norm, ng)
    x, xg, gy = (torch.from_numpy(g[tag + k]) for k in ("x", "xg", "g"))
    sd64 = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = gref.pointnet_forward(x.double(), xg.double(), sd64, _spg_pcfg(c), _groups(norm, ng))
    ref.backward(gy.double())
    ptn.train()
    out = ptn(x.to(dev), xg.to(dev))
    _close(out, ref, 1e-4)
    _close(out, g[tag + "out_train"], 1e-4)
    out.backward(gy.to(dev))
    _check_grads({k: p.grad for k, p in ptn.named_parameters()}, {k: v.grad for k, v in sd64.items()},
                 _spg_pointwise)
    ptn.eval()
    with torch.no_grad():
        _close(ptn(x.to(dev), xg.to(dev)), ref, 1e-4)


@pytest.mark.gpu
def test_pointnet_eval_chunked(dev, monkeypatch):
    """An eval batch above _EVAL_CHUNK runs in slices; GroupNorm has no batch statistics, so it equals the
    unchunked oracle."""
    from superpoint_graph_b200 import spg_pointnet
    g = _golden()
    ptn, sd, c = _spg_model(g, "group", 2, dev)
    torch.manual_seed(2)
    x, xg = torch.randn(23, 14, 128) * 0.5, torch.rand(23) * 3
    monkeypatch.setattr(spg_pointnet, "_EVAL_CHUNK", 5)
    ptn.eval()
    with torch.no_grad():
        out = ptn(x.to(dev), xg.to(dev))
    _close(out, gref.pointnet_forward(x.double(), xg.double(), sd, _spg_pcfg(c), 2), 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("norm,ng", [("layer", 1), ("group", 4)])
def test_pointnet_ragged(dev, norm, ng):
    """forward_ragged: equal lengths give forward's result and gradients; unequal lengths (an empty superpoint
    included) match the oracle, training forward and backward."""
    g = _golden()
    ptn, sd, c = _spg_model(g, norm, ng, dev)
    groups = _groups(norm, ng)
    tag = "spg_%s%d." % (norm, ng)
    x, xg, gy = (torch.from_numpy(g[tag + k]) for k in ("x", "xg", "g"))
    B, Fe, L = x.shape
    ptn.train()
    out = ptn(x.to(dev), xg.to(dev))
    out.backward(gy.to(dev))
    g_fixed = {k: p.grad.clone() for k, p in ptn.named_parameters()}
    ptn.zero_grad()
    pts = x.permute(0, 2, 1).reshape(B * L, Fe).contiguous()
    offsets = torch.arange(B + 1, dtype=torch.int64) * L
    out_r = ptn.forward_ragged(pts.to(dev), offsets.to(dev), xg.to(dev))
    _close(out_r, out, 1e-6)
    out_r.backward(gy.to(dev))
    for k, p in ptn.named_parameters():
        _close(p.grad, g_fixed[k], 1e-5, 1e-9)
    # unequal lengths
    lens = [40, 0, 128, 7, 300, 1, 64]
    torch.manual_seed(3)
    pts = torch.randn(sum(lens), Fe) * 0.5
    offsets = torch.zeros(len(lens) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(lens), 0)
    xg, gy = torch.rand(len(lens)) * 3, torch.randn(len(lens), c["nf_fc"][-1])
    sd64 = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = gref.pointnet_forward_ragged(pts.double(), offsets, xg.double(), sd64, _spg_pcfg(c), groups)
    ref.backward(gy.double())
    ptn.zero_grad()
    out_r = ptn.forward_ragged(pts.to(dev), offsets.to(dev), xg.to(dev))
    _close(out_r, ref, 1e-4)
    out_r.backward(gy.to(dev))
    _check_grads({k: p.grad for k, p in ptn.named_parameters()}, {k: v.grad for k, v in sd64.items()},
                 _spg_pointwise)


@pytest.mark.gpu
@pytest.mark.parametrize("norm,ng", [("layer", 1), ("group", 2)])
def test_prelast_dropout(dev, norm, ng):
    """prelast_do = 0.5 after a GroupNorm FC layer: the oracle applies the device's mask (ops.dropout_mask of the
    first slot after dropout_manual_seed) and matches output and gradients."""
    from types import SimpleNamespace
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder
    model, sd_s, sd_p = _lp_models(norm, ng, dev, prelast_do=0.5)
    B = 900
    torch.manual_seed(8)
    clouds, glob, gy = torch.randn(B, 6, 20) * 0.5, torch.randn(B, 11), torch.randn(B, 4)
    seed = 4321
    ops.dropout_manual_seed(seed, dev)
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    out = emb.run_batch(model, clouds.to(dev), glob.to(dev))
    out.backward(gy.to(dev))
    mask = ops.dropout_mask(torch.tensor([seed, 0], dtype=torch.int64, device=dev), 0.5, B, 32).cpu()
    sd_s64 = {k: v.clone().requires_grad_(True) for k, v in sd_s.items()}
    sd_p64 = {k: v.clone().requires_grad_(True) for k, v in sd_p.items()}
    ref = _lp_embed(clouds.double(), glob.double(), sd_s64, sd_p64, _groups(norm, ng),
                    dict(LP_PCFG, prelast_do=0.5), drop_mask=mask)
    ref.backward(gy.double())
    _close(out, ref, 1e-4)
    got = {"stn." + k: p.grad for k, p in model.stn.named_parameters()}
    got.update({"ptn." + k: p.grad for k, p in model.ptn.named_parameters()})
    want = {"stn." + k: v.grad for k, v in sd_s64.items()}
    want.update({"ptn." + k: v.grad for k, v in sd_p64.items()})
    _check_grads(got, want, lambda k: k.startswith("ptn.convs.") or k.startswith("stn.convs."))


# Per-kernel launches of two training steps (forward + backward) of a batch-norm PointNet with SPG widths, 512
# clouds of 128 points and prelast_do 0.5, as they were before GroupNorm layers were served.
BN_STEP_LAUNCHES = {"act_bwd_apply": 6, "act_bwd_reduce": 2, "act_bwd_reduce_final": 2, "affine_act": 2, "cloud_rows": 4, "colstats_final": 2, "colsum_final": 4, "colsum_partial": 4, "dropout_bwd_apply": 2, "dropout_bwd_reduce": 2, "dropout_bwd_reduce_final": 2, "dropout_fwd": 2, "dropout_rng_next": 2, "gemm_f32": 22, "gemm_splitk_reduce": 30, "segmax_bwd": 12, "segmax_fwd": 4, "stn_apply_bwd": 2, "tc_dw_3xtf32": 16, "tc_gemm_3xtf32": 44, "tc_merge": 38, "tc_pack_weights": 44}


@pytest.mark.gpu
def test_batch_norm_pointnet_launches_unchanged(dev):
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_pointnet import PointNet
    ptn = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 11, prelast_do=0.5).to(dev)
    ptn.train()
    torch.manual_seed(0)
    x, xg = torch.randn(512, 14, 128, device=dev), torch.rand(512, device=dev)
    out = ptn(x, xg)
    out.backward(torch.randn_like(out))
    torch.cuda.synchronize()
    ops.prof_reset()
    for _ in range(2):
        out = ptn(x, xg)
        out.backward(torch.randn_like(out))
    torch.cuda.synchronize()
    assert {k: v[0] for k, v in ops.prof_collect().items()} == BN_STEP_LAUNCHES
