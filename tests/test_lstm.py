"""`lstm_*` model configs (LSTMCellEx and the recurrent LSTM-ECC, ref: learning/modules.py:128-183, 262-316).

CPU: the oracle against lstm.npz, lstm_plain.npz and graphnet_lstm.npz (made by the unmodified reference),
the model's state-dict layout, the drop-in name and the rejected use_pyg=1 path.
GPU: the cell kernels against the golden, GraphNetwork against the golden (fused and per-step recurrence),
and the Trainer's steps, replays and inference graphs.  The cell kernels at every width, tiling and option
against float64 are tested for both cells in test_recurrent_widths.py, the fused recurrence against the
per-step kernels, bit for bit, in test_gpu_parity.py.
"""
import os

import numpy as np
import pytest
import torch

from oracle import lstm_ref, nets_ref

GOLDEN = "graphnet_lstm.npz"
N_CONFIGS = 4


def load(golden_dir, name=GOLDEN):
    z = np.load(os.path.join(golden_dir, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


def t(a, dev=None):
    x = torch.from_numpy(np.asarray(a))
    return x.to(dev) if dev is not None else x


def sub(d, prefix):
    return {k[len(prefix):]: t(v).clone() for k, v in d.items() if k.startswith(prefix)}


def f64(d):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in d.items()}


def close(a, b, rtol, atol=0.0):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all(), "non-finite values"
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= atol + rtol * scale, "max err %g vs scale %g (rel %g)" % (err, scale, err / max(scale, 1e-30))


def close_grads(got, want, rtol):
    floor = 1e-5 * max(float(torch.as_tensor(v).abs().max()) for v in want.values())
    for k, v in want.items():
        assert got[k] is not None, "missing gradient for %s" % k
        close(got[k], v, rtol, floor)


def net_args(g):
    return [int(w) for w in g["fnet_widths"]], int(g["bnidx"])


def _cell_oracle(sd, x, h, c, g, gc, ln, ig):
    """float64 autograd through lstm_ref.lstm_cell_ex: outputs and gradients of <hy,g> + <cy,gc>."""
    sd = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    x, h, c = (v.double().clone().requires_grad_(True) for v in (x, h, c))
    hy, cy = lstm_ref.lstm_cell_ex(x, h, c, sd, "", ln, ig)
    ((hy * g.double()).sum() + (cy * gc.double()).sum()).backward()
    return hy.detach(), cy.detach(), x.grad, h.grad, c.grad, {k: v.grad for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name,ln,ig", [("lstm.npz", True, True), ("lstm_plain.npz", False, False)])
def test_oracle_matches_lstm_cell_golden(golden_dir, name, ln, ig):
    g = load(golden_dir, name)
    hy, cy, gx, gh, gcx, grads = _cell_oracle(sub(g, "sd."), t(g["x"]), t(g["h"]), t(g["c"]), t(g["g"]),
                                              t(g["g_c"]), ln, ig)
    close(hy, g["hy"], 1e-5)
    close(cy, g["cy"], 1e-5)
    close(gx, g["gx"], 1e-5)
    close(gh, g["gh"], 1e-5)
    close(gcx, g["gcx"], 1e-5)
    for k, v in sub(g, "grad.").items():
        close(grads[k], v, 1e-5, 1e-7)


def _oracle_net(g, i, training, grads, sd=None):
    config, tag = str(g["configs"][i]), "c%d." % i
    widths, bnidx = net_args(g)
    sd = f64(sub(g, tag + "sd0.")) if sd is None else sd
    if grads:
        for k, v in sd.items():
            if nets_ref.is_param(k):
                v.requires_grad_(True)
    emb = t(g[tag + "emb"]).double().requires_grad_(grads)
    out = lstm_ref.graphnet_forward_config(emb, t(g["edgefeats"]).double(), t(g["idxn"]), t(g["degs"]), sd,
                                           config, widths, bnidx, training)
    return out, emb, sd


def _loss(out, g):
    ncls = out.shape[1]
    return torch.nn.functional.cross_entropy(out, t(g["labels"], out.device),
                                             weight=t(g["cw"], out.device)[:ncls].to(out.dtype))


@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_oracle_matches_graphnet_lstm_golden(golden_dir, i):
    g = load(golden_dir)
    tag = "c%d." % i
    bwd = (tag + "loss") in g
    out, emb, sd = _oracle_net(g, i, True, bwd)
    close(out, g[tag + "out_train"], 1e-5)
    for k, v in sub(g, tag + "sd1.").items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v), k
        else:
            close(sd[k], v, 1e-6)
    if bwd:
        loss = _loss(out, g)
        close(loss, g[tag + "loss"], 1e-6)
        loss.backward()
        close(emb.grad, g[tag + "gemb"], 1e-5, 1e-8)
        for k, v in sub(g, tag + "grad.").items():
            close(sd[k].grad, v, 1e-5, 1e-8)
    with torch.no_grad():  # with the running statistics of the training forward, as the golden
        out_eval, _, _ = _oracle_net(g, i, False, False, {k: v.detach() for k, v in sd.items()})
    close(out_eval, g[tag + "out_eval"], 1e-5)


def test_graphnet_lstm_golden_covers_every_variant(golden_dir):
    g = load(golden_dir)
    assert [str(c) for c in g["configs"]] == ["lstm_3_1_1_1_0,f_13", "lstm_2,f_8", "lstm_2_1_0_0_1,f_13",
                                              "lstm_2_0,f_13"]
    assert "c3.loss" not in g and all("c%d.loss" % i in g for i in range(3))  # matrix config: forward only


@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_graphnetwork_layout_matches_golden(golden_dir, i):
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    from superpoint_graph_b200.spg_modules import LSTMCellEx, RNNGraphConvModule
    g = load(golden_dir)
    config, tag = str(g["configs"][i]), "c%d." % i
    widths, bnidx = net_args(g)
    net = GraphNetwork(config, 32, widths, True, 0, bnidx, 1e20, use_pyg=0, cuda=False)
    want = sub(g, tag + "sd0.")
    got = net.state_dict()
    assert list(got.keys()) == list(want.keys())
    for k, v in want.items():
        assert tuple(got[k].shape) == tuple(v.shape), k
    n_params = sum(v.numel() for k, v in want.items() if nets_ref.is_param(k))
    assert sum(p.numel() for p in net.parameters()) == n_params
    rnn = [m for m in net.modules() if isinstance(m, RNNGraphConvModule)]
    assert len(rnn) == 1 and isinstance(rnn[0]._cell, LSTMCellEx) and rnn[0]._isLSTM
    # initialisation: nn.LSTMCell's uniform(+-1/sqrt(H)) for the cell, as in the reference
    cell = rnn[0]._cell
    for p in (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh):
        assert float(p.detach().abs().max()) <= 32 ** -0.5
    net.load_state_dict(want)


def test_lstm_cell_signature_and_repr():
    from superpoint_graph_b200.spg_modules import LSTMCellEx
    cell = LSTMCellEx(32, 32, bias=True, layernorm=True, ingate=True)
    keys = set(cell.state_dict().keys())
    assert keys == {"weight_ih", "weight_hh", "bias_ih", "bias_hh", "ig.weight", "ig.bias"}
    assert "ini" in cell._modules and "inh" in cell._modules
    assert cell.weight_ih.shape == (128, 32) and repr(cell).endswith("(ingate layernorm)")
    plain = LSTMCellEx(32, 32, bias=False, layernorm=False, ingate=False)
    assert set(plain.state_dict().keys()) == {"weight_ih", "weight_hh"} and repr(plain).endswith("()")
    assert plain.flags() == 0 and cell.flags() == 7


def test_dropin_exposes_lstm_cell():
    from superpoint_graph_b200 import dropin, spg_modules
    try:
        dropin.install()
        from learning.modules import LSTMCellEx
        assert LSTMCellEx is spg_modules.LSTMCellEx
    finally:
        dropin.uninstall()


def test_lstm_use_pyg_still_raises():
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    with pytest.raises(NotImplementedError, match="use_pyg"):
        GraphNetwork("lstm_2,f_8", 32, [13, 32, 64], use_pyg=1)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("name,ln,ig", [("lstm.npz", True, True), ("lstm_plain.npz", False, False)])
def test_lstm_cell_golden(golden_dir, dev, name, ln, ig):
    from superpoint_graph_b200.spg_modules import LSTMCellEx
    g = load(golden_dir, name)
    cell = LSTMCellEx(32, 32, bias=True, layernorm=ln, ingate=ig)
    cell.load_state_dict(sub(g, "sd."))
    cell.to(dev)
    x, h, c = (t(g[k], dev).requires_grad_(True) for k in ("x", "h", "c"))
    hy, cy = cell(x, (h, c))
    close(hy, g["hy"], 1e-4)
    close(cy, g["cy"], 1e-4)
    ((hy * t(g["g"], dev)).sum() + (cy * t(g["g_c"], dev)).sum()).backward()
    close(x.grad, g["gx"], 3e-4)
    close(h.grad, g["gh"], 3e-4)
    close(c.grad, g["gcx"], 3e-4)
    close_grads({k: p.grad for k, p in cell.named_parameters()}, sub(g, "grad."), 3e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_graphnet_lstm_golden(golden_dir, dev, monkeypatch, i, fused):
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    monkeypatch.setattr(ops, "USE_FUSED_RNN", [fused])
    g = load(golden_dir)
    config, tag = str(g["configs"][i]), "c%d." % i
    widths, bnidx = net_args(g)
    net = GraphNetwork(config, 32, widths, True, 0, bnidx, 1e20, use_pyg=0, cuda=True)
    net.load_state_dict(sub(g, tag + "sd0."))
    net.to(dev).train()
    net.set_info([GraphConvInfo.from_arrays(g["idxn"], g["degs"], g["edgefeats"]) for _ in net.gconvs], True)
    emb = t(g[tag + "emb"], dev).requires_grad_(True)
    out = net(emb)
    close(out, g[tag + "out_train"], 1e-4)
    sd = net.state_dict()
    for k, v in sub(g, tag + "sd1.").items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v), k
        else:
            close(sd[k], v, 1e-5)
    loss = _loss(out, g)
    loss.backward()
    have = {k: p.grad for k, p in net.named_parameters()}
    if (tag + "loss") in g:
        close(loss, g[tag + "loss"], 1e-4)
        close(emb.grad, g[tag + "gemb"], 3e-4, 1e-7)
        close_grads(have, sub(g, tag + "grad."), 3e-4)
    else:  # matrix filters: the reference's backward does not run, the float64 oracle pins the gradients
        ref_out, ref_emb, ref_sd = _oracle_net(g, i, True, True)
        _loss(ref_out, g).backward()
        close(emb.grad, ref_emb.grad, 3e-4, 1e-7)
        close_grads(have, {k: v.grad for k, v in ref_sd.items() if nets_ref.is_param(k)}, 3e-4)
    net.eval()
    with torch.no_grad():
        close(net(emb.detach()), g[tag + "out_eval"], 1e-4)


TRAIN_CONFIGS = ["lstm_10_1_1_1_0,f_13", "lstm_2_0,f_13"]


def _pre_bn_bias_keys(module, prefix):
    import torch.nn as nn
    keys = set()
    for name, m in module.named_modules():
        if isinstance(m, nn.Sequential):
            mods = list(m.named_children())
            for (n0, a), (_, b) in zip(mods[:-1], mods[1:]):
                if isinstance(a, (nn.Conv1d, nn.Linear)) and isinstance(b, nn.BatchNorm1d) and a.bias is not None:
                    keys.add(prefix + (name + "." if name else "") + n0 + ".bias")
            if any(isinstance(x, nn.Conv1d) for _, x in mods):
                bns = [n for n, x in mods if isinstance(x, nn.BatchNorm1d)]
                if bns:
                    keys.add(prefix + (name + "." if name else "") + bns[-1] + ".bias")
    return keys


@pytest.mark.gpu
@pytest.mark.parametrize("config", TRAIN_CONFIGS)
def test_trainer_steps_vs_oracle(dev, config):
    """Two training steps against the float64 oracle trainer, with the bounds of the CRF configs: the first
    step at 1e-4 (>= 97 % of every parameter tensor), the second with the recurrent configs' looser bounds."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config=config)
    torch.manual_seed(3)
    model = create_model(args)
    sd_ecc = f64({k: v.clone() for k, v in model.ecc.state_dict().items()})
    sd_ptn = f64({k: v.clone() for k, v in model.ptn.state_dict().items()})
    skip = _pre_bn_bias_keys(model.ecc, "ecc.") | _pre_bn_bias_keys(model.ptn, "ptn.")
    pcfg, _ = workloads.oracle_cfg(make_args())
    mcfg = dict(config=config, fnet_widths=[args.edge_feats] + list(args.fnet_widths), bnidx=args.fnet_bnidx)
    ref = lstm_ref.RefTrainerConfig(sd_ptn, sd_ecc, pcfg, mcfg, lr=args.lr, grad_clip=args.grad_clip)
    model.to(dev)
    tr = Trainer(model, args)
    batch = make_batch(n_nodes=200, seed=4)
    db = HostBatch(batch).to_device(dev)
    b64 = f64(batch)
    loss, logits = tr.train_step(db)
    rl, ro = ref.step(b64)
    close(logits, ro, 1e-4)
    close(loss[0], rl, 1e-4)
    sd = {("ecc." + k): v for k, v in model.ecc.state_dict().items()}
    sd.update({("ptn." + k): v for k, v in model.ptn.state_dict().items()})
    for pre, rsd in (("ecc.", ref.sd_ecc), ("ptn.", ref.sd_ptn)):
        for k, v in rsd.items():
            if not nets_ref.is_param(k) or (pre + k) in skip:
                continue
            v = v.detach()
            d = (sd[pre + k].cpu().double() - v).abs()
            ok = float((d <= 1e-4 * max(float(v.abs().max()), 1e-3)).double().mean())
            assert ok >= 0.97, "%s: only %.1f %% of %d elements agree" % (pre + k, 100 * ok, v.numel())
            assert float(d.max()) <= 2.5 * args.lr, pre + k
    loss2, logits2 = tr.train_step(db)
    rl2, ro2 = ref.step(b64)
    assert abs(float(loss2[0]) - rl2) <= 5e-2 * abs(rl2)
    close(logits2, ro2, 0.15)


@pytest.mark.gpu
@pytest.mark.parametrize("config", TRAIN_CONFIGS)
def test_trainer_graph_replays_match_eager(dev, config):
    """capture()/replay() reproduces the eager training steps; capture_eval()/replay_eval() the eager
    inference forward."""
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config=config)
    batch = make_batch(n_nodes=200, seed=11)
    results = []
    for mode in ("eager", "graph"):
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        db = HostBatch(batch).to_device(dev)
        losses = []
        if mode == "eager":
            for _ in range(3):
                loss, logits = tr.train_step(db)
                losses.append(float(loss[0]))
        else:
            key = tr.capture(db, warmup=1)
            for _ in range(3):
                loss, logits = tr.replay(key)
                losses.append(float(loss[0]))
        torch.cuda.synchronize()
        results.append((losses, tr.flat.clone(), logits.clone()))
        eager_eval = tr.eval_step(db).clone()
        key = tr.capture_eval(db, key=0)
        assert torch.equal(tr.replay_eval(key), eager_eval)
    (l_e, p_e, o_e), (l_g, p_g, o_g) = results
    close(torch.tensor(l_g), torch.tensor(l_e), 1e-5)
    close(o_g, o_e, 1e-4)
    close(p_g, p_e, 1e-4, 2.1e-2 * 4)  # noise-driven (pre-BN bias) parameters random-walk by +-lr


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_side_stream_gives_identical_lstm_steps(dev, monkeypatch, graph):
    """The recurrent block's parameter gradients on the side stream: three steps bit-identical to the
    single-stream run (eager and CUDA-graph replay)."""
    from superpoint_graph_b200 import ops
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config="lstm_4_1_1_1_1,f_13")
    batch = make_batch(n_nodes=300, seed=4)
    results = []
    for side in (True, False):
        monkeypatch.setattr(ops, "USE_SIDE_STREAM", [side])
        torch.manual_seed(5)
        model = create_model(args)
        model.to(dev)
        tr = Trainer(model, args)
        assert (tr._side is not None) == side
        tr.side_in_eager = True
        db = HostBatch(batch).to_device(dev)
        losses = []
        if graph:
            key = tr.capture(db, warmup=2)
            for _ in range(3):
                loss, logits = tr.replay(key)
                losses.append(float(loss[0]))
        else:
            for _ in range(3):
                loss, logits = tr.train_step(db)
                losses.append(float(loss[0]))
        torch.cuda.synchronize()
        results.append((losses, tr.flat.clone(), logits.clone(), tr.flat_grad.clone()))
    (l_a, p_a, o_a, g_a), (l_b, p_b, o_b, g_b) = results
    assert l_a == l_b
    assert torch.equal(g_a, g_b) and torch.equal(p_a, p_b) and torch.equal(o_a, o_b)
