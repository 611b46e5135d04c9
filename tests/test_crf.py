"""`crf_<R>` model configs (ECC_CRFModule, ref: learning/modules.py:185-202).

CPU: the oracle's config-driven GraphNetwork forward against graphnet_crf.npz (made by the unmodified
reference), the model's state-dict layout, the module's construction rules and its drop-in name.
GPU: the ECC-CRF kernels against a float64 autograd restatement, GraphNetwork against the golden and the
float64 oracle (outputs, running statistics, every gradient), and the Trainer's steps, captured replays
and inference graphs against the oracle trainer and its own eager steps.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import crf_ref, ecc_ref, nets_ref

GOLDEN = "graphnet_crf.npz"
FNET_WIDTHS = [13, 32, 128, 64]
BN_KEYS = ("running_mean", "running_var", "num_batches_tracked")


def load(golden_dir):
    import os
    z = np.load(os.path.join(golden_dir, GOLDEN), allow_pickle=False)
    return {k: z[k] for k in z.files}


def t(a, dev=None):
    x = torch.from_numpy(np.asarray(a))
    return x.to(dev) if dev is not None else x


def sub(d, prefix):
    return {k[len(prefix):]: t(v).clone() for k, v in d.items() if k.startswith(prefix)}


def close(a, b, rtol, atol=0.0):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.isfinite(a).all(), "non-finite values"
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= atol + rtol * scale, "max err %g vs scale %g (rel %g)" % (err, scale, err / max(scale, 1e-30))


def configs(golden_dir):
    return [str(c) for c in load(golden_dir)["configs"]]


N_CONFIGS = 4


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_oracle_matches_crf_golden(golden_dir, i):
    g = load(golden_dir)
    config, tag = str(g["configs"][i]), "c%d." % i
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sub(g, tag + "sd0.").items()}
    emb, ef = t(g[tag + "emb"]).double(), t(g["edgefeats"]).double()
    idxn, degs = t(g["idxn"]), t(g["degs"])
    out = crf_ref.graphnet_forward_config(emb, ef, idxn, degs, sd, config, FNET_WIDTHS, 2, True)
    close(out, g[tag + "out_train"], 1e-5)
    sd1 = sub(g, tag + "sd1.")
    assert sd1, "golden holds no BatchNorm state for %s" % config
    for k, v in sd1.items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v), (k, int(sd[k]), int(v))
        else:
            close(sd[k], v, 1e-6)
    close(crf_ref.graphnet_forward_config(emb, ef, idxn, degs, sd, config, FNET_WIDTHS, 2, False),
          g[tag + "out_eval"], 1e-5)


def test_crf_running_statistics_take_one_update_per_iteration(golden_dir):
    """f_13,crf_3: the filter network's BatchNorm counted three batches; crf_0 never ran it."""
    g = load(golden_dir)
    cfgs = configs(golden_dir)
    nbt = {c: {k: int(v) for k, v in sub(g, "c%d.sd1." % i).items() if k.endswith("num_batches_tracked")}
           for i, c in enumerate(cfgs)}
    assert set(nbt["f_13,crf_3"].values()) == {3}
    assert set(nbt["f_13,crf_0"].values()) == {0}


@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_graphnetwork_layout_matches_golden(golden_dir, i):
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    from superpoint_graph_b200.spg_modules import ECC_CRFModule
    g = load(golden_dir)
    config, tag = str(g["configs"][i]), "c%d." % i
    net = GraphNetwork(config, 32, FNET_WIDTHS, True, 0, 2, 1e20, use_pyg=0, cuda=False)
    want = sub(g, tag + "sd0.")
    got = net.state_dict()
    assert list(got.keys()) == list(want.keys())
    for k, v in want.items():
        assert tuple(got[k].shape) == tuple(v.shape), k
    n_params = sum(v.numel() for k, v in want.items() if nets_ref.is_param(k))
    assert sum(p.numel() for p in net.parameters()) == n_params
    crfs = [m for m in net.modules() if isinstance(m, ECC_CRFModule)]
    assert len(crfs) == 1 and crfs[0]._propagation is net.gconvs[-1]
    assert crfs[0]._nrepeats == int(config.split("crf_")[1].split(",")[0])
    net.load_state_dict(want)


def _gconv(C, width):
    from superpoint_graph_b200.spg_ecc import GraphConvModule
    from superpoint_graph_b200.spg_graphnet import create_fnet
    return GraphConvModule(C, C, create_fnet([13, 16, width], True, 0, -1))


def test_crf_module_rejects_what_the_kernels_do_not_serve():
    from superpoint_graph_b200.spg_modules import ECC_CRFModule
    ECC_CRFModule(_gconv(13, 169), 2)  # supported: C x C matrix filters
    ECC_CRFModule(_gconv(32, 1024), 1)
    with pytest.raises(NotImplementedError, match="GraphConvModule"):
        ECC_CRFModule(nn.Linear(4, 4), 1)
    with pytest.raises(NotImplementedError, match="vector filters"):
        ECC_CRFModule(_gconv(13, 13), 1)
    with pytest.raises(NotImplementedError, match="C <= 32"):
        ECC_CRFModule(_gconv(33, 33 * 33), 1)
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    with pytest.raises(NotImplementedError, match="C <= 32"):  # crf after a cat_all GRU: C = 96
        GraphNetwork("gru_2,crf_1", 32, FNET_WIDTHS, True, 0, 2, 1e20, use_pyg=0, cuda=False)


def test_dropin_exposes_crf_module():
    from superpoint_graph_b200 import dropin, spg_modules
    try:
        dropin.install()
        from learning.ecc import GraphConvModule
        from learning.modules import ECC_CRFModule
        assert ECC_CRFModule is spg_modules.ECC_CRFModule
        m = ECC_CRFModule(GraphConvModule(8, 8, nn.Sequential(nn.Linear(13, 64))), nrepeats=2)
        assert m._nrepeats == 2 and "_propagation._fnet.0.weight" in m.state_dict()
    finally:
        dropin.uninstall()


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _graph_arrays(N, seed):
    """Target-sorted (idxn, degs): zero-degree targets, a target of degree 300, a source with no
    out-edges, N not a multiple of the 8 warps of a block."""
    rng = np.random.default_rng(seed)
    degs = rng.integers(0, 7, size=N)
    degs[[0, 5, N - 1]] = 0
    degs[N // 2] = 300
    E = int(degs.sum())
    idxn = rng.integers(0, N - 1, size=E)
    idxn[idxn == 7] = 8  # node 7 is the source of no edge
    return torch.from_numpy(idxn.astype(np.int64)), torch.from_numpy(degs.astype(np.int64))


def _crf_oracle(U, W, idxn, degs, R, g):
    """float64 autograd: out = Z_R, and the gradients of <out, g> w.r.t. U and W."""
    U = U.double().requires_grad_(True)
    W = W.double().requires_grad_(True)
    Q = torch.softmax(U, 1)
    for i in range(R):
        Q = U - ecc_ref.graph_conv_forward(Q, W, idxn, None, degs)
        if i < R - 1:
            Q = torch.softmax(Q, 1)
    Q.backward(g.double())
    return Q.detach(), U.grad, W.grad


@pytest.mark.gpu
@pytest.mark.parametrize("R", [0, 1, 3])
@pytest.mark.parametrize("C", [1, 8, 13, 16, 32])
def test_crf_kernels_vs_float64(dev, C, R):
    from superpoint_graph_b200 import ops
    N = 333
    idxn, degs = _graph_arrays(N, 100 + C)
    graph = ops.EccGraph(idxn, None, degs, n_in=N)
    E = idxn.numel()
    torch.manual_seed(C * 10 + R)
    U, W, g = torch.randn(N, C) * 2, torch.randn(E, C, C) * 0.5, torch.randn(N, C)
    out_ref, gu_ref, gw_ref = _crf_oracle(U, W, idxn, degs, R, g)
    Ud, Wd, gd = U.to(dev), W.to(dev), g.to(dev)
    nan = float("nan")
    qs = torch.full((max(R, 1), N, C), nan, device=dev)
    out = torch.full((N, C), nan, device=dev)
    if R == 0:
        ops.crf_softmax(Ud, out=out)
    else:
        ops.crf_softmax(Ud, out=qs[0])
        for r in range(1, R + 1):
            ops.crf_fwd_step(Ud, qs[r - 1], Wd, graph, out if r == R else qs[r], softmax=r < R)
    close(out, out_ref, 1e-5)
    gu = torch.full((N, C), nan, device=dev)
    if R == 0:
        ops.crf_softmax(out, gd, out=gu)
        assert gw_ref is None
    else:
        gps = torch.full((R, N, C), nan, device=dev)
        gps[R - 1] = -gd
        du_in = gd
        for r in range(R, 0, -1):
            ops.crf_bwd_step(Wd, gps[r - 1], qs[r - 1], du_in, gu, gps[r - 2] if r > 1 else None, graph)
            du_in = gu
        gw = ops.ecc_bwd_w(qs, gps, graph, (E, C, C), n_iter=R)
        close(gw, gw_ref, 1e-5)
    close(gu, gu_ref, 1e-5)


@pytest.mark.gpu
def test_crf_kernels_reject_wide_filters(dev):
    from superpoint_graph_b200 import ops
    x = torch.randn(4, 33, device=dev)
    with pytest.raises(RuntimeError, match="not supported"):
        ops.crf_softmax(x)


def _oracle_grads(g, i, emb, labels, cw):
    config, tag = str(g["configs"][i]), "c%d." % i
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sub(g, tag + "sd0.").items()}
    for k, v in sd.items():
        if nets_ref.is_param(k):
            v.requires_grad_(True)
    e = emb.double().requires_grad_(True)
    out = crf_ref.graphnet_forward_config(e, t(g["edgefeats"]).double(), t(g["idxn"]), t(g["degs"]), sd,
                                           config, FNET_WIDTHS, 2, True)
    torch.nn.functional.cross_entropy(out, labels, weight=cw.double()).backward()
    return e.grad, {k: v.grad for k, v in sd.items() if nets_ref.is_param(k)}


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_CONFIGS))
def test_graphnet_crf_golden(golden_dir, dev, i):
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    g = load(golden_dir)
    config, tag = str(g["configs"][i]), "c%d." % i
    net = GraphNetwork(config, 32, FNET_WIDTHS, True, 0, 2, 1e20, use_pyg=0, cuda=True)
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
    ncls = out.shape[1]
    rng = np.random.default_rng(i)
    labels = torch.from_numpy(rng.integers(0, ncls, size=out.shape[0]).astype(np.int64))
    labels[[3, 4]] = -100
    cw = torch.from_numpy(rng.uniform(0.5, 2.0, size=ncls).astype(np.float32))
    torch.nn.functional.cross_entropy(out, labels.to(dev), weight=cw.to(dev)).backward()
    ge, want = _oracle_grads(g, i, t(g[tag + "emb"]), labels, cw)
    close(emb.grad, ge, 3e-4, 1e-7)
    have = {k: p.grad for k, p in net.named_parameters()}
    floor = 1e-5 * max(float(v.abs().max()) for v in want.values() if v is not None)
    for k, v in want.items():
        if v is None:  # crf_0: the filter network never ran
            assert have[k] is None, k
        else:
            assert have[k] is not None, "missing gradient for %s" % k
            close(have[k], v, 3e-4, floor)
    net.eval()
    with torch.no_grad():
        close(net(emb.detach()), g[tag + "out_eval"], 1e-4)
    with pytest.raises(RuntimeError, match="eval-mode"):
        net(emb).sum().backward()


def _pre_bn_bias_keys(module, prefix):
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


TRAIN_CONFIGS = ["f_13,crf_3", "gru_3_1_1_1_0,f_13,crf_2"]


@pytest.mark.gpu
@pytest.mark.parametrize("config", TRAIN_CONFIGS)
def test_trainer_steps_vs_oracle(dev, config):
    """Two training steps against the float64 oracle trainer: loss and logits, and the parameters after
    each Adam step (>= 97 % of every tensor within 1e-4 of its scale; elements whose gradient is rounding
    noise around zero may step the other way)."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    args = make_args(model_config=config)
    torch.manual_seed(3)
    model = create_model(args)
    f64 = lambda d: {k: (v.double() if v.is_floating_point() else v) for k, v in d.items()}  # noqa: E731
    sd_ecc = f64({k: v.clone() for k, v in model.ecc.state_dict().items()})
    sd_ptn = f64({k: v.clone() for k, v in model.ptn.state_dict().items()})
    skip = _pre_bn_bias_keys(model.ecc, "ecc.") | _pre_bn_bias_keys(model.ptn, "ptn.")
    pcfg, _ = workloads.oracle_cfg(make_args())
    mcfg = dict(config=config, fnet_widths=[args.edge_feats] + list(args.fnet_widths), bnidx=args.fnet_bnidx)
    ref = crf_ref.RefTrainerConfig(sd_ptn, sd_ecc, pcfg, mcfg, lr=args.lr, grad_clip=args.grad_clip)
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
    # The second step starts from parameters that differ where Adam's first, sign-like step flipped on a
    # gradient at rounding-noise level (up to 3 % of the elements, 2*lr each): the bounds of the recurrent
    # configs' second step (tests/test_gpu_shapes.py) apply.
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
        bufs = torch.cat([b.double().reshape(-1) for k, b in model.ecc.state_dict().items()
                          if k.endswith(("running_mean", "running_var", "num_batches_tracked"))])
        results.append((losses, tr.flat.clone(), logits.clone(), bufs))
        eager_eval = tr.eval_step(db).clone()
        key = tr.capture_eval(db, key=0)
        assert torch.equal(tr.replay_eval(key), eager_eval)
    (l_e, p_e, o_e, b_e), (l_g, p_g, o_g, b_g) = results
    close(torch.tensor(l_g), torch.tensor(l_e), 1e-5)
    close(o_g, o_e, 1e-4)
    close(p_g, p_e, 1e-4, 2.1e-2 * 4)  # noise-driven (pre-BN bias) parameters random-walk by +-lr
    close(b_g, b_e, 1e-4)
