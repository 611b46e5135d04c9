"""Training-mode dropout (`--ptn_prelast_do`, `d_<p>` model-config tokens) on the device.

The mask is Philox4x32-10 on the logical element index (include/spg_b200.h, spg_dropout_*); `philox4x32_10`
and `dropout_mask_np` below restate it in numpy, pinned on the Random123 known-answer vectors.  The GPU tests
rebuild the masks the device used from its (seed, counter) and hand them to the float64 oracle."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import nets_ref

U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 arrays (or ints) of 32-bit words, key: 2 words -> uint32 [4, n]."""
    c = [np.atleast_1d(np.asarray(x, dtype=np.uint64)) for x in ctr]
    n = max(x.size for x in c)
    c0, c1, c2, c3 = [np.broadcast_to(x, (n,)).copy() for x in c]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & U32
            k1 = (k1 + np.uint64(0xBB67AE85)) & U32
        p0, p1 = m0 * c0, m1 * c2  # 32 x 32 -> 64 bits, exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & U32
    return np.stack([c0, c1, c2, c3]).astype(np.uint32)


def threshold(p):
    p = float(np.float32(p))
    return 0 if p <= 0 else min(int(p * 2.0 ** 32), 0xFFFFFFFF)


def dropout_mask_np(seed, ctr, M, C, p):
    """bool [M, C]: element i = m*C + c is kept iff word i&3 of Philox(counter (i>>2, i>>34, ctr), key seed)
    is >= floor(p * 2^32); p >= 1 keeps nothing."""
    seed, ctr = int(seed) & (2 ** 64 - 1), int(ctr) & (2 ** 64 - 1)
    n = M * C
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    w = philox4x32_10((q & U32, q >> np.uint64(32), ctr & 0xFFFFFFFF, ctr >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    w = w.T.reshape(-1)[:n]  # element 4q + j <- word j of group q
    keep = w >= np.uint32(threshold(p)) if np.float32(p) < 1 else np.zeros(n, dtype=bool)
    return keep.reshape(M, C)


# The reference's dropout placements in float64, built on oracle/nets_ref's pinned building blocks.  The masks
# are explicit: the restatement draws no random numbers, the caller passes the ones the device used.
def ref_dropout(x, mask, p):
    """nn.Dropout(p) in training mode with keep mask `mask` (1 = kept); p >= 1 gives zeros."""
    if p >= 1:
        return torch.zeros_like(x)
    return x * (torch.as_tensor(mask).to(x.dtype) * (1.0 / (1.0 - p)))


def ref_fc_stack(x, sd, prefix, n_layers, training, last_ac=True, masks=None):
    """nets_ref.fc_stack with nn.Dropout(p) after the activation of layer i for every i in masks = {i: (mask,
    p)} (learning/pointnet.py:109-110); every later module index shifts by one, as in the nn.Sequential."""
    shift = 0
    for i in range(n_layers):
        k = 3 * i + shift
        x = F.linear(x, sd['%s%d.weight' % (prefix, k)], sd['%s%d.bias' % (prefix, k)])
        if i < n_layers - 1 or last_ac:
            x = F.relu(nets_ref._bn(x, sd, '%s%d' % (prefix, k + 1), training))
        if masks is not None and i in masks:
            x = ref_dropout(x, *masks[i])
            shift += 1
    return x


def ref_pointnet(x, x_global, sd, cfg, training, masks=None):
    """nets_ref.pointnet_forward (learning/pointnet.py:120-133) with the FC stack of ref_fc_stack."""
    if cfg['nfeat_stn'] > 0:
        T = nets_ref.stn_forward(x[:, :cfg['nfeat_stn'], :], sd, 'stn.', cfg['n_conv_stn'], cfg['n_fc_stn'], training)
        xy = torch.bmm(x[:, :2, :].transpose(1, 2), T).transpose(1, 2)
        x = torch.cat([xy, x[:, 2:, :]], 1)
    x = nets_ref.conv_stack(x, sd, 'convs.', cfg['n_conv'], training)
    x = F.max_pool1d(x, x.size(2)).squeeze(2)
    if x_global is not None:
        x = torch.cat([x, x_global.view(x.shape[0], -1)], 1)
    return ref_fc_stack(x, sd, 'fcs.', cfg['n_fc'], training, last_ac=False, masks=masks)


def ref_pointnet_ragged(points, offsets, x_global, sd, cfg, training, masks=None):
    """nets_ref.pointnet_forward_ragged (CSR segments) with the FC stack of ref_fc_stack."""
    B = len(offsets) - 1
    x = points.t().unsqueeze(0)

    def segmax(y):
        return torch.stack([y[0, :, int(offsets[b]):int(offsets[b + 1])].max(1)[0] for b in range(B)])

    if cfg['nfeat_stn'] > 0:
        h = nets_ref.conv_stack(x[:, :cfg['nfeat_stn'], :], sd, 'stn.convs.', cfg['n_conv_stn'], training)
        h = nets_ref.fc_stack(segmax(h), sd, 'stn.fcs.', cfg['n_fc_stn'], training, last_ac=True)
        T = F.linear(h, sd['stn.proj.weight'], sd['stn.proj.bias']).view(-1, 2, 2)
        T = T + torch.eye(2, dtype=T.dtype).unsqueeze(0)
        seg = torch.repeat_interleave(torch.arange(B), torch.as_tensor(offsets[1:]) - torch.as_tensor(offsets[:-1]))
        xy = torch.bmm(points[:, None, :2], T[seg]).squeeze(1)
        x = torch.cat([xy, points[:, 2:]], 1).t().unsqueeze(0)
    h = segmax(nets_ref.conv_stack(x, sd, 'convs.', cfg['n_conv'], training))
    if x_global is not None:
        h = torch.cat([h, x_global.view(B, -1)], 1)
    return ref_fc_stack(h, sd, 'fcs.', cfg['n_fc'], training, last_ac=False, masks=masks)


def ref_dense(x, sd, tokens, training, first=0, masks=None):
    """A run of GraphNetwork's f_<n> / b[_0] / r / d_<p> tokens (learning/graphnet.py:50-63); token j is module
    `first + j`; masks = {module index: keep mask} for the d_ tokens with p > 0 in training mode."""
    for j, token in enumerate(tokens):
        tok, name = token.strip().split('_'), '%d' % (first + j)
        if tok[0] == 'f':
            x = F.linear(x, sd[name + '.weight'], sd[name + '.bias'])
        elif tok[0] == 'b':
            x = F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'], sd.get(name + '.weight'),
                             sd.get(name + '.bias'), training, 0.1, 1e-5)
        elif tok[0] == 'r':
            x = F.relu(x)
        elif tok[0] == 'd' and training and float(tok[1]) > 0:
            x = ref_dropout(x, masks[first + j], float(tok[1]))
    return x


# ------------------------------------------------------------------------------------------- host
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in philox4x32_10(ctr, key)[:, 0]) == want


def test_mask_restatement_keep_rate():
    for p in (0.1, 0.5, 0.9):
        keep = dropout_mask_np(0x0123456789ABCDEF, 5, 1000, 13, p)
        n = keep.size
        assert abs(int(keep.sum()) - n * (1 - p)) <= 5 * np.sqrt(n * p * (1 - p))
    assert not dropout_mask_np(1, 0, 10, 7, 1.0).any()
    assert dropout_mask_np(1, 0, 10, 7, 0.0).all()
    assert not np.array_equal(dropout_mask_np(1, 0, 64, 64, 0.5), dropout_mask_np(1, 1, 64, 64, 0.5))


def _spec_fields(specs):
    """Everything of the specs but the BatchNorm module (its identity differs between two models)."""
    return [(s.w, s.b, s.gamma, s.beta, s.bn is not None, s.relu, s.cin, s.cout, s.drop) for s in specs]


def _graphnet(config):
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    return GraphNetwork(config, 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0, cuda=True)


def test_parse_places_dropout_on_the_right_spec():
    from superpoint_graph_b200.dense import parse_sequential
    from superpoint_graph_b200.spg_pointnet import PointNet
    net = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=0.5)
    specs, params = parse_sequential(net.fcs, True)
    assert [s.drop for s in specs] == [0.0, 0.5, 0.0]
    assert [s.cout for s in specs] == [256, 64, 32] and specs[1].relu and specs[1].bn is net.fcs[4]
    assert params[specs[2].w] is net.fcs[7].weight
    # eval mode: identity, the specs of a PointNet without the module
    plain = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=0)
    ev, _ = parse_sequential(net.fcs, False)
    ev0, _ = parse_sequential(plain.fcs, False)
    assert _spec_fields(ev) == _spec_fields(ev0) and [s.drop for s in ev] == [0.0] * 3
    # model config f_64,b,r,d_0.5,f_13
    g = _graphnet("gru_3_1_1_1_0,f_64,b,r,d_0.5,f_13")
    run = [g._modules[str(k)] for k in range(1, 6)]
    specs, params = parse_sequential(run, True)
    assert [(s.cin, s.cout, s.bn is not None, s.relu, s.drop) for s in specs] == \
        [(32, 64, True, True, 0.5), (64, 13, False, False, 0.0)]
    assert [s.drop for s in parse_sequential(run, False)[0]] == [0.0, 0.0]


@pytest.mark.parametrize("config", ["f_64,b,r,d_0,f_13", "f_64,b,r,d_0.5,f_13"])
def test_p0_and_eval_give_todays_specs(config):
    from superpoint_graph_b200.dense import parse_sequential
    run0 = list(_graphnet("f_64,b,r,f_13")._modules.values())
    run = list(_graphnet(config)._modules.values())
    modes = (True, False) if config.endswith("d_0,f_13") else (False,)  # p = 0: training mode too
    for training in modes:
        assert _spec_fields(parse_sequential(run, training)[0]) == _spec_fields(parse_sequential(run0, training)[0])


@pytest.mark.parametrize("mods", [
    lambda: [nn.Dropout(0.5), nn.Linear(4, 4)],
    lambda: [nn.Linear(4, 4), nn.Dropout(0.5), nn.BatchNorm1d(4)],
    lambda: [nn.Linear(4, 4), nn.BatchNorm1d(4), nn.Dropout(0.5), nn.ReLU()],
    lambda: [nn.Linear(4, 4), nn.ReLU(), nn.Dropout(0.5), nn.Dropout(0.3)],
])
def test_unsupported_dropout_orders_raise(mods):
    from superpoint_graph_b200.dense import parse_sequential
    with pytest.raises(NotImplementedError):
        parse_sequential(mods(), True)


def test_unsupported_order_message_names_the_supported_order():
    from superpoint_graph_b200.dense import parse_sequential
    with pytest.raises(NotImplementedError, match=r"Linear\|Conv1d, \[BatchNorm1d\], \[ReLU\], Dropout"):
        parse_sequential([nn.Dropout(0.5), nn.Linear(4, 4)], True)


def test_state_dict_keys_unchanged():
    from superpoint_graph_b200.spg_pointnet import PointNet
    net = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=0.5)
    fcs = [k for k in net.state_dict() if k.startswith("fcs.")]
    assert fcs == ["fcs.0.weight", "fcs.0.bias", "fcs.1.weight", "fcs.1.bias", "fcs.1.running_mean",
                   "fcs.1.running_var", "fcs.1.num_batches_tracked", "fcs.3.weight", "fcs.3.bias", "fcs.4.weight",
                   "fcs.4.bias", "fcs.4.running_mean", "fcs.4.running_var", "fcs.4.num_batches_tracked",
                   "fcs.7.weight", "fcs.7.bias"]
    g = _graphnet("gru_3_1_1_1_0,f_64,b,r,d_0.5,f_13")
    assert [k for k in g.state_dict() if not k.startswith("0.")] == [
        "1.weight", "1.bias", "2.weight", "2.bias", "2.running_mean", "2.running_var", "2.num_batches_tracked",
        "5.weight", "5.bias"]


def test_restatement_with_masks_matches_torch_modules():
    torch.manual_seed(0)
    seq = nn.Sequential(nn.Linear(5, 6), nn.BatchNorm1d(6), nn.ReLU(), nn.Linear(6, 4), nn.BatchNorm1d(4), nn.ReLU(),
                        nn.Dropout(0.25), nn.Linear(4, 3)).double()
    sd = {k: v.clone() for k, v in seq.state_dict().items()}
    x = torch.randn(9, 5, dtype=torch.float64)
    mask = torch.rand(9, 4) > 0.25
    h = seq[:6](x)
    want = seq[7](h * mask / 0.75)
    got = ref_fc_stack(x, sd, "", 3, True, last_ac=False, masks={1: (mask, 0.25)})
    assert torch.allclose(got, want)
    g = _graphnet("f_6,b,r,d_0.25,f_3").double()
    sd = {k: v.clone() for k, v in g.state_dict().items()}
    x = torch.randn(9, 32, dtype=torch.float64)
    mask = torch.rand(9, 6) > 0.25
    want = g._modules["4"](g._modules["2"](g._modules["1"](g._modules["0"](x))) * mask / 0.75)
    got = ref_dense(x, sd, ["f_6", "b", "r", "d_0.25", "f_3"], True, masks={3: mask})
    assert torch.allclose(got, want)


def test_restatement_without_masks_is_the_pinned_oracle():
    """With no masks the restatements above are nets_ref's pointnet_forward(_ragged) / graphnet head."""
    from superpoint_graph_b200.spg_pointnet import PointNet
    net = PointNet([16, 32], [32, 16, 8], [8, 16], [16, 8], 6, 6, prelast_do=0)
    torch.manual_seed(3)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.1)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in net.state_dict().items()}
    cfg = dict(n_conv=2, n_fc=3, n_conv_stn=2, n_fc_stn=2, nfeat_stn=6)
    x, xg = torch.randn(5, 6, 20, dtype=torch.float64), torch.rand(5, dtype=torch.float64)
    assert torch.equal(ref_pointnet(x, xg, dict(sd), cfg, True), nets_ref.pointnet_forward(x, xg, dict(sd), cfg, True))
    offsets = np.array([0, 3, 10, 11, 30, 32])
    pts = torch.randn(32, 6, dtype=torch.float64)
    assert torch.equal(ref_pointnet_ragged(pts, offsets, xg, dict(sd), cfg, True),
                       nets_ref.pointnet_forward_ragged(pts, offsets, xg, dict(sd), cfg, True))
    g = _graphnet("f_13").double()
    x = torch.randn(7, 32, dtype=torch.float64)
    assert torch.equal(ref_dense(x, g.state_dict(), ["f_13"], True), F.linear(x, g._modules["0"].weight, g._modules["0"].bias))


# -------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _close(a, b, rtol, atol=0.0):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all(), "non-finite values"
    err, scale = (a - b).abs().max().item(), b.abs().max().item()
    assert err <= atol + rtol * scale, "max err %g vs scale %g (rel %g)" % (err, scale, err / max(scale, 1e-30))


def _rng(dev):
    from superpoint_graph_b200 import ops
    seed, ctr = (int(v) for v in ops.dropout_rng_state(dev).cpu())
    return seed, ctr


def _mask(seed, ctr, M, C, p):
    return torch.from_numpy(dropout_mask_np(seed, ctr, M, C, p))


@pytest.mark.gpu
@pytest.mark.parametrize("M,C", [(1000, 13), (1000, 64), (7, 3), (333, 352)])
@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_device_mask_matches_numpy(dev, M, C, p):
    from superpoint_graph_b200 import ops
    seed, ctr = -0x0123456789ABCDEF, 2 ** 33 + 5
    slot = torch.tensor([seed, ctr], dtype=torch.int64, device=dev)
    want = dropout_mask_np(seed, ctr, M, C, p)
    got = ops.dropout_mask(slot, p, M, C).cpu().numpy().astype(bool)
    assert np.array_equal(got, want)
    n = M * C
    assert abs(int(got.sum()) - n * (1 - p)) <= 5 * np.sqrt(n * p * (1 - p)) + 1
    # the fused forward applies the same mask whatever the leading dimension: BN-apply, ReLU, mask, 1/(1-p)
    ld = C + 4
    y = torch.randn(M, ld, device=dev)
    sc, sh = torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev) * 0.3
    out = ops.dropout_fwd(y, ld, M, C, sc, sh, True, p, slot)
    a = torch.relu(y[:, :C].double() * sc.double() + sh.double()).cpu()
    _close(out, a * torch.from_numpy(want) / (1 - np.float32(p)), 1e-6)


@pytest.mark.gpu
def test_rng_slots_take_consecutive_counters(dev):
    from superpoint_graph_b200 import ops
    ops.dropout_manual_seed(2 ** 64 - 3, dev)
    s0, s1 = ops.dropout_slot(dev), ops.dropout_slot(dev)
    assert s0.tolist() == [-3, 0] and s1.tolist() == [-3, 1]
    assert _rng(dev) == (-3, 2)


def _s3dis_pointnet(dev, p):
    from superpoint_graph_b200.spg_pointnet import PointNet
    net = PointNet([64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64], 14, 14, prelast_do=p)
    torch.manual_seed(8)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
        net.stn.proj.bias.normal_(0, 0.05)
    sd = {k: v.clone().double().requires_grad_(nets_ref.is_param(k)) if v.is_floating_point() else v.clone()
          for k, v in net.state_dict().items()}
    return net.to(dev).train(), sd


PCFG = dict(n_conv=5, n_fc=3, n_conv_stn=3, n_fc_stn=2, nfeat_stn=14)


def _check_pointnet_grads(net, sd, skip=()):
    """Against float64 (DESIGN §6): 1e-3 of the tensor maximum above the max-pool; below it (point-wise
    layers, STN) 5e-2 of the maximum and 2e-2 Frobenius (arg-max ties move single rows).  Pre-BatchNorm
    biases (analytically zero gradients) are skipped."""
    from test_gpu_shapes import pre_bn_bias_keys
    skip = set(skip) | pre_bn_bias_keys(net)
    n = 0
    for k, prm in net.named_parameters():
        if k in skip:
            continue
        want, got = sd[k].grad, prm.grad.cpu().double()
        scale = max(float(want.abs().max()), 1e-12)
        pointwise = k.startswith("convs.") or k.startswith("stn.")
        err = float((got - want).abs().max())
        assert err <= (5e-2 if pointwise else 1e-3) * scale + 1e-7, "%s: rel err %g" % (k, err / scale)
        if pointwise and float(want.norm()) > 0:
            assert float((got - want).norm() / want.norm()) <= 2e-2, k
        n += 1
    assert n > 20


def _check_running_stats(net, sd):
    for k, v in net.state_dict().items():
        if k.endswith("running_mean") or k.endswith("running_var"):
            _close(v, sd[k], 1e-5, 1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["clouds", "ragged"])
def test_pointnet_prelast_dropout_vs_oracle(dev, layout):
    """S3DIS widths, prelast_do=0.5, training forward + backward against the float64 oracle fed with the masks
    rebuilt from the device's (seed, counter): outputs, parameter gradients, BatchNorm running statistics."""
    net, sd = _s3dis_pointnet(dev, 0.5)
    rng = np.random.default_rng(3)
    if layout == "clouds":
        B = 48
        x, xg = torch.randn(B, 14, 128) * 0.4, torch.rand(B) * 3
    else:
        lens = rng.integers(1, 301, size=97)
        offsets = np.concatenate([[0], np.cumsum(lens)])
        B = 97
        pts, xg = torch.randn(int(offsets[-1]), 14) * 0.4, torch.rand(B) * 3
    gout = torch.randn(B, 32)
    seed, ctr = _rng(dev)
    if layout == "clouds":
        out = net(x.to(dev), xg.to(dev))
    else:
        out = net.forward_ragged(pts.to(dev), torch.from_numpy(offsets).to(dev), xg.to(dev))
    assert _rng(dev) == (seed, ctr + 1)  # one dropout site, one counter
    masks = {1: (_mask(seed, ctr, B, 64, 0.5), 0.5)}
    if layout == "clouds":
        ref = ref_pointnet(x.double(), xg.double(), sd, PCFG, True, masks=masks)
    else:
        ref = ref_pointnet_ragged(pts.double(), offsets, xg.double(), sd, PCFG, True, masks=masks)
    _close(out, ref, 1e-4)
    ref.backward(gout.double())
    out.backward(gout.to(dev))
    _check_pointnet_grads(net, sd)
    _check_running_stats(net, sd)


@pytest.mark.gpu
def test_same_seed_is_bit_identical_and_steps_draw_new_masks(dev):
    from superpoint_graph_b200 import ops
    net, _ = _s3dis_pointnet(dev, 0.5)
    torch.manual_seed(4)
    x, xg = (torch.randn(64, 14, 128) * 0.4).to(dev), (torch.rand(64) * 3).to(dev)
    outs, grads = [], []
    for reseed in (True, True, False):
        if reseed:
            ops.dropout_manual_seed(1234, dev)
        net.zero_grad()
        out = net(x, xg)
        out.backward(torch.ones_like(out))
        outs.append(out.detach().clone())
        grads.append([p.grad.clone() for p in net.parameters()])
    assert torch.equal(outs[0], outs[1])
    assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
    assert not torch.equal(outs[1], outs[2])  # third forward: next counter, new mask
    assert _rng(dev) == (1234, 2)


def _dropout_args(**kw):
    from superpoint_graph_b200.trainer import make_args
    d = dict(model_config="gru_3_1_1_1_0,f_64,b,r,d_0.5,f_13", ptn_prelast_do=0.5)
    d.update(kw)
    return make_args(**d)


HEAD = ["f_64", "b", "r", "d_0.5", "f_13"]


@pytest.mark.gpu
def test_trainer_step_with_dropout_vs_oracle(dev):
    """Trainer.train_step on gru_3_1_1_1_0,f_64,b,r,d_0.5,f_13 with ptn_prelast_do=0.5: loss, logits and
    every gradient against the float64 oracle step with the device's masks."""
    from superpoint_graph_b200 import ops, workloads
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    from test_gpu_shapes import _check_grads, _f64, pre_bn_bias_keys
    args = _dropout_args()
    torch.manual_seed(1)
    model = create_model(args)
    sd_ecc = _f64({k: v.clone() for k, v in model.ecc.state_dict().items()})
    sd_ptn = _f64({k: v.clone() for k, v in model.ptn.state_dict().items()})
    # pre-BatchNorm biases (analytically zero gradients); ecc.1 is the f_64 token in front of the b token
    skip = pre_bn_bias_keys(model.ecc, "ecc.") | pre_bn_bias_keys(model.ptn, "ptn.") | {"ecc.1.bias"}
    model.to(dev)
    pcfg, mcfg = workloads.oracle_cfg(args)
    for sd in (sd_ecc, sd_ptn):
        for k, v in sd.items():
            v.requires_grad_(nets_ref.is_param(k))
    tr = Trainer(model, args)
    batch = workloads.batch(workloads.get("s3dis_train"), 1)  # the batch of test_bench_config_train_step_vs_oracle
    db = HostBatch(batch).to_device(dev)
    ops.dropout_manual_seed(77, dev)
    loss, logits = tr.train_step(db)
    assert _rng(dev) == (77, 2)  # PointNet site (counter 0), then the head's d_ token (counter 1)
    nv = int(db.clouds.shape[0])  # PointNet rows = the valid clouds
    masks = dict(ptn={1: (_mask(77, 0, nv, 64, 0.5), 0.5)}, ecc={4: _mask(77, 1, db.n_nodes, 64, 0.5)})
    # the oracle step (learning/main.py:202-205): CloudEmbedder.run, model.ecc, cross entropy, backward
    b = _f64(batch)
    rows = ref_pointnet(b["clouds"], b["clouds_global"], sd_ptn, pcfg, True, masks=masks["ptn"])
    idx_valid = torch.nonzero(b["clouds_flag"].eq(0)).reshape(-1)
    emb = rows.new_zeros((b["clouds_flag"].numel(), rows.shape[1])).index_copy(0, idx_valid, rows)
    x = nets_ref.rnn_ecc_forward(emb, b["edgefeats"], b["idxn"], b["degs"], sd_ecc, "0.", mcfg, True)
    ref_logits = ref_dense(x, sd_ecc, HEAD, True, first=1, masks=masks["ecc"])
    ref_loss_t = F.cross_entropy(ref_logits, b["labels"])
    ref_loss_t.backward()
    ref_loss = float(ref_loss_t.detach())
    ref_grads = {pre + k: v.grad for pre, sd in (("ecc.", sd_ecc), ("ptn.", sd_ptn)) for k, v in sd.items()
                 if nets_ref.is_param(k)}
    _close(logits, ref_logits, 1e-4)
    assert abs(float(loss[0]) - ref_loss) <= 1e-4 * abs(ref_loss)
    _check_grads(model, ref_grads, skip)


@pytest.mark.gpu
def test_capture_replay_with_dropout_matches_eager(dev):
    """As test_cuda_graph_replay_matches_eager, with dropout at two sites: three replays == three eager steps
    from the same dropout_manual_seed, and every replay draws new masks (the counter lives on the device)."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    args = _dropout_args()
    batch = make_batch(n_nodes=200, seed=11)
    results = []
    for mode in ("eager", "graph"):
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        ops.dropout_manual_seed(99, dev)
        losses, ctrs = [], []
        if mode == "eager":
            for _ in range(3):
                loss, logits = tr.train_step(db)
                losses.append(float(loss[0]))
                ctrs.append(_rng(dev)[1])
        else:
            key = tr.capture(db, warmup=1)
            assert _rng(dev) == (99, 0)  # capture() leaves the generator where it found it
            for _ in range(3):
                loss, logits = tr.replay(key)
                losses.append(float(loss[0]))
                ctrs.append(_rng(dev)[1])
        torch.cuda.synchronize()
        assert ctrs == [2, 4, 6]
        results.append((losses, tr.flat.clone(), logits.clone()))
    (l_e, p_e, o_e), (l_g, p_g, o_g) = results
    assert int(torch.isfinite(p_g).all())
    _close(torch.tensor(l_g), torch.tensor(l_e), 1e-5)
    _close(o_g, o_e, 1e-4)
    _close(p_g, p_e, 1e-4, 2.1e-2 * 4)
    # the replays used counters 0..5: their masks differ from each other
    nv = int(db.clouds.shape[0])
    ms = [dropout_mask_np(99, c, nv, 64, 0.5) for c in (0, 2, 4)]
    assert not np.array_equal(ms[0], ms[1]) and not np.array_equal(ms[1], ms[2])


@pytest.mark.gpu
def test_mem_monger_reuses_the_forward_masks(dev):
    """ptn_mem_monger=1 recomputes the PointNet forward in bw_hook with the forward's masks: the gradients
    equal those of ptn_mem_monger=0 at the same seed (the head's d_ token draws in between)."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    batch = make_batch(n_nodes=150, seed=21)
    grads, ctrs = [], []
    for monger in (0, 1):
        args = _dropout_args(model_config="gru_2_1_1_1_0,f_64,b,r,d_0.5,f_13", ptn_mem_monger=monger)
        torch.manual_seed(9)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        ops.dropout_manual_seed(3, dev)
        model.train()
        model.ecc.gconvs[0].set_info(db.gi)
        emb = tr.embedder.run(model, None, batch["clouds_flag"], batch["clouds"], batch["clouds_global"])
        out = model.ecc(emb)
        torch.nn.functional.cross_entropy(out, db.labels).backward()
        tr.embedder.bw_hook()
        grads.append({k: p.grad.clone() for k, p in model.named_parameters()})
        ctrs.append(_rng(dev))
    assert ctrs == [(3, 2), (3, 2)]
    for k, g in grads[0].items():
        _close(grads[1][k], g, 1e-5, 1e-5 * max(float(v.abs().max()) for v in grads[0].values()))


@pytest.mark.gpu
def test_p1_drops_everything_without_nan(dev):
    from superpoint_graph_b200.dense import run_sequential
    net, _ = _s3dis_pointnet(dev, 1.0)
    x, xg = (torch.randn(40, 14, 128) * 0.4).to(dev), (torch.rand(40) * 3).to(dev)
    out = net(x, xg)
    last = net.fcs[7]
    assert torch.equal(out, last.bias.detach().expand_as(out))  # zeros behind the dropout: bias only
    out.backward(torch.randn_like(out))
    for k, prm in net.named_parameters():
        assert torch.isfinite(prm.grad).all(), k
        if k != "fcs.7.bias":
            assert float(prm.grad.abs().max()) == 0.0, k
    # a chain whose last module is the dropout (ChainFunction output), input gradient zero
    seq = nn.Sequential(nn.Linear(32, 64), nn.BatchNorm1d(64), nn.ReLU(), nn.Dropout(1.0)).to(dev).train()
    xin = torch.randn(700, 32, device=dev, requires_grad=True)
    y = run_sequential(seq, xin, True)
    assert float(y.abs().max()) == 0.0
    y.backward(torch.randn_like(y))
    assert torch.isfinite(xin.grad).all() and float(xin.grad.abs().max()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f_64,b,r,d_0.5,f_13", "f_64,b,r,d_0.5", "f_64,r,d_0.3,f_13",
                                    "f_64,d_0.3,f_13", "f_13,b,r,d_0.5,f_7"])
@pytest.mark.parametrize("M", [300, 2600])
def test_dense_token_runs_with_dropout_vs_oracle(dev, config, M):
    """f/b/r/d runs of GraphNetwork (tensor-core rows at M=2600, SIMT rows at M=300; odd widths on the scalar
    kernels; a chain ending in the dropout) against the float64 oracle: output, input and parameter gradients."""
    from superpoint_graph_b200 import ops
    torch.manual_seed(2)
    g = _graphnet(config)
    sd = {k: v.clone().double().requires_grad_(nets_ref.is_param(k)) if v.is_floating_point() else v.clone()
          for k, v in g.state_dict().items()}
    g.to(dev).train()
    x = torch.randn(M, 32)
    xd = x.to(dev).requires_grad_(True)
    ops.dropout_manual_seed(11, dev)
    out = g(xd)
    toks = config.split(",")
    j = next(i for i, t in enumerate(toks) if t.startswith("d_"))
    p = float(toks[j][2:])
    width = int(toks[0][2:])
    xr = x.double().requires_grad_(True)
    ref = ref_dense(xr, sd, toks, True, masks={j: _mask(11, 0, M, width, p)})
    _close(out, ref, 1e-4)
    gy = torch.randn(ref.shape)
    ref.backward(gy.double())
    out.backward(gy.to(dev))
    _close(xd.grad, xr.grad, 1e-4)
    for k, prm in g.named_parameters():
        if k == "0.bias" and "b" in toks:
            continue  # feeds a batch-statistics BatchNorm: analytically zero, rounding noise in both
        _close(prm.grad, sd[k].grad, 3e-4, 1e-6)
    _check_running_stats(g, sd)


@pytest.mark.gpu
def test_p0_leaves_launch_counts_unchanged(dev):
    """A model with `d_0` and one without a Dropout module launch exactly the same kernels; no dropout
    kernel runs."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    batch = make_batch(n_nodes=200, seed=11)
    counts = []
    for cfg in ("gru_3_1_1_1_0,f_64,b,r,f_13", "gru_3_1_1_1_0,f_64,b,r,d_0,f_13"):
        args = make_args(model_config=cfg, ptn_prelast_do=0)
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        tr.train_step(db)
        torch.cuda.synchronize()
        ops.prof_reset()
        tr.train_step(db)
        torch.cuda.synchronize()
        counts.append({k: v[0] for k, v in ops.prof_collect().items()})
    assert counts[0] == counts[1]
    assert not any(k.startswith("dropout") for k in counts[0])


@pytest.mark.gpu
def test_local_cloud_embedder_with_dropout(dev):
    """Learned-partition shapes (20-point clouds, external STN, global features + T, L2 normalisation) with
    ptn_prelast_do=0.5: forward and backward, incl. the input gradient through the external STN."""
    from types import SimpleNamespace
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_pointnet import LocalCloudEmbedder, PointNet, STNkD
    torch.manual_seed(4)
    model = torch.nn.Module()
    model.stn = STNkD(2, [16, 64], [32, 16])
    model.ptn = PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, prelast_do=0.5, nfeat_global=11 + 4)
    with torch.no_grad():
        model.stn.proj.weight.normal_(0, 0.1)
    sd_s = {k: v.clone().double().requires_grad_(nets_ref.is_param(k)) if v.is_floating_point() else v.clone()
            for k, v in model.stn.state_dict().items()}
    sd_p = {k: v.clone().double().requires_grad_(nets_ref.is_param(k)) if v.is_floating_point() else v.clone()
            for k, v in model.ptn.state_dict().items()}
    B, L = 700, 20
    clouds, glob = torch.randn(B, 6, L) * 0.5, torch.randn(B, 11)
    model.to(dev).train()
    ops.dropout_manual_seed(5, dev)
    emb = LocalCloudEmbedder(SimpleNamespace(ptn_nfeat_stn=2, stn_as_global=1))
    out = emb.run_batch(model, clouds.to(dev), glob.to(dev))
    c = clouds.double()
    T = nets_ref.stn_forward(c[:, :2], sd_s, "", 2, 2, True)
    xy = torch.bmm(c[:, :2].transpose(1, 2), T).transpose(1, 2)
    pcfg = dict(n_conv=2, n_fc=4, n_conv_stn=0, n_fc_stn=0, nfeat_stn=0)
    ref = torch.nn.functional.normalize(ref_pointnet(
        torch.cat([xy, c[:, 2:]], 1), torch.cat([glob.double(), T.view(-1, 4)], 1), sd_p, pcfg, True,
        masks={2: (_mask(5, 0, B, 32, 0.5), 0.5)}))
    _close(out, ref, 2e-4)
    gy = torch.randn(B, 4)
    ref.backward(gy.double())
    model.zero_grad()
    out.backward(gy.to(dev))
    for name, mod, sd in (("stn", model.stn, sd_s), ("ptn", model.ptn, sd_p)):
        want = {k: v.grad for k, v in sd.items() if isinstance(v, torch.Tensor) and v.requires_grad}
        floor = 1e-5 * max(float(v.abs().max()) for v in want.values())
        for k, prm in mod.named_parameters():
            _close(prm.grad, want[k], 2e-3, floor)
