"""GPU parity at the BENCHMARKED and BASELINE shapes (VERDICT r1, "What's weak" 1-3): full steps of
the configurations bench.py times — not miniatures of them — against the pinned oracle, through the
same Trainer / CloudEmbedder / C-ABI path the bench uses.

Tolerances: logits and loss 1e-4 relative (north_star).  The oracle runs in float64 here.
Gradients (against that float64 truth):
  * everything that is not a point-wise-layer parameter agrees to <= 1e-5 of the tensor's largest
    gradient (bound here: 3e-3; 1e-2 below the filter network's BatchNorm at 1e5 edges);
  * the point-wise layers sit UNDER a max-pool over 128 points: a cloud/channel pair whose two largest
    activations differ by less than float32 rounding (~1 pair in 2.4e5 at this size) sends its pooled
    gradient to a different point row than the float64 oracle does — a discrete, legitimate difference
    that changes one row of the top layer's weight gradient by a few percent of the tensor's maximum
    and trickles down the chain.  torch's own float32 CPU kernels show the same effect on other tensors
    (1.4e-3).  Bound: 5e-2 of the maximum and 2e-2 in relative Frobenius norm.
Parameters with an analytically ZERO gradient are excluded BY NAME from gradient and parameter checks
(both sides hold rounding noise there, and Adam turns the SIGN of noise into a +-lr step; no output
depends on them):
  * a bias that feeds a batch-statistics BatchNorm (the mean subtraction cancels it);
  * the BatchNorm bias right before a max-pool that is followed by a batch-statistics BatchNorm FC
    layer: d/dbeta = sum_b g_pool[b,c] = sum_j W[j,c] sum_b dY_fc[b,j] = 0 (all ReLU masks active).
After one Adam step the parameters are compared element-wise: an element whose gradient is within
rounding noise of zero may step the other way (2*lr apart); at least 97 % of every tensor's elements
must agree to 1e-4 of the tensor's scale.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ecc_ref, nets_ref  # noqa: E402  (checker only)
from test_gpu_parity import close, load, sub, t  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def pre_bn_bias_keys(module, prefix=""):
    """Names of Conv1d/Linear biases immediately followed by a BatchNorm1d inside nn.Sequential
    containers of `module` (analytically zero gradient in training mode)."""
    keys = set()
    for name, m in module.named_modules():
        if isinstance(m, torch.nn.Sequential):
            mods = list(m.named_children())
            for (n0, a), (_, b) in zip(mods[:-1], mods[1:]):
                if isinstance(a, (torch.nn.Conv1d, torch.nn.Linear)) and isinstance(b, torch.nn.BatchNorm1d) \
                        and a.bias is not None:
                    keys.add(prefix + (name + "." if name else "") + n0 + ".bias")
            # BatchNorm bias of the last Conv1d block (the one the max-pool reads)
            if any(isinstance(x, torch.nn.Conv1d) for _, x in mods):
                bns = [n for n, x in mods if isinstance(x, torch.nn.BatchNorm1d)]
                if bns:
                    keys.add(prefix + (name + "." if name else "") + bns[-1] + ".bias")
    return keys


def _f64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


def _model_and_oracle(w, dev):
    """(model on the GPU, its Trainer, float64 oracle trainer on the same initial state, keys to skip);
    feed the oracle `_f64(batch)`."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import Trainer, create_model
    margs = w["margs"]
    torch.manual_seed(1)
    model = create_model(margs)
    sd_ecc = _f64({k: v.clone() for k, v in model.ecc.state_dict().items()})
    sd_ptn = _f64({k: v.clone() for k, v in model.ptn.state_dict().items()})
    skip = pre_bn_bias_keys(model.ecc, "ecc.") | pre_bn_bias_keys(model.ptn, "ptn.")
    model.to(dev)
    pcfg, mcfg = workloads.oracle_cfg(margs)
    ref = nets_ref.RefTrainer(sd_ptn, sd_ecc, pcfg, mcfg, lr=margs.lr, grad_clip=margs.grad_clip, ecc_mode="vec")
    return model, Trainer(model, margs), ref, skip


def _ref_grads(ref):
    g = {}
    for pre, sd in (("ecc.", ref.sd_ecc), ("ptn.", ref.sd_ptn)):
        for k, v in sd.items():
            if nets_ref.is_param(k):
                g[pre + k] = v.grad
    return g


def _check_grads(model, ref_grads, skip, rtol=3e-3, rtol_pointwise=5e-2, rtol_fnet=1e-2):
    n = 0
    for k, p in model.named_parameters():
        if k in skip:
            continue
        want = ref_grads[k]
        assert p.grad is not None, k
        got = p.grad.cpu().double()
        scale = max(float(want.abs().max()), 1e-12)
        err = float((got - want).abs().max())
        pointwise = k.startswith("ptn.convs.") or k.startswith("ptn.stn.")
        tol = rtol_pointwise if pointwise else (rtol_fnet if "._fnet." in k else rtol)
        assert err <= tol * scale + 1e-7, "%s: grad err %g vs scale %g (rel %g)" % (k, err, scale, err / scale)
        if pointwise and float(want.norm()) > 0:
            fro = float((got - want).norm() / want.norm())
            assert fro <= 2e-2, "%s: relative Frobenius error %g" % (k, fro)
        n += 1
    assert n > 20


def _check_params_after_adam(model, ref, skip, min_frac=0.97):
    """Element-wise agreement of the parameters after an Adam step (see the module docstring)."""
    sd = {("ecc." + k): v for k, v in model.ecc.state_dict().items()}
    sd.update({("ptn." + k): v for k, v in model.ptn.state_dict().items()})
    for pre, rsd in (("ecc.", ref.sd_ecc), ("ptn.", ref.sd_ptn)):
        for k, v in rsd.items():
            if not nets_ref.is_param(k) or (pre + k) in skip:
                continue
            d = (sd[pre + k].cpu().double() - v.detach().double()).abs()
            ok = float((d <= 1e-4 * max(float(v.abs().max()), 1e-3)).double().mean())
            assert ok >= min_frac, "%s: only %.1f %% of %d elements agree" % (pre + k, 100 * ok, v.numel())
            assert float(d.max()) <= 2.5 * ref.opt.param_groups[0]["lr"], pre + k  # never more than a flipped step


@pytest.mark.parametrize("graph", [False, True])
def test_bench_config_train_step_vs_oracle(dev, graph):
    """configs[1] exactly as bench.py runs it: 1024 superpoints, gru_10_1_1_1_0,f_13, S3DIS widths,
    fused recurrence, eager and CUDA-graph replay; loss, logits, every gradient, second-step logits."""
    from superpoint_graph_b200 import ops, workloads
    from superpoint_graph_b200.trainer import HostBatch
    w = workloads.get("s3dis_train")
    assert w["nodes"] == 1024 and w["margs"].model_config == "gru_10_1_1_1_0,f_13"
    batch = workloads.batch(w, 1)
    model, tr, ref, skip = _model_and_oracle(w, dev)
    db = HostBatch(batch).to_device(dev)
    assert ops.rnn_vv_supported(torch.empty(1, 32, device=dev), db.gi.graph(), 1024, 32)
    if graph:
        key = tr.capture(db, warmup=1)
        step = lambda: tr.replay(key)
    else:
        step = lambda: tr.train_step(db)
    loss, logits = step()
    ref_loss, ref_logits = ref.step(_f64(batch))
    grads = _ref_grads(ref)
    close(logits, ref_logits, 1e-4)
    assert abs(float(loss[0]) - ref_loss) <= 1e-4 * abs(ref_loss)
    _check_grads(model, grads, skip)
    _check_params_after_adam(model, ref, skip)
    loss2, logits2 = step()
    ref_loss2, ref_logits2 = ref.step(_f64(batch))
    # second step from (slightly different: flipped noise-level Adam steps) parameters: same regime
    assert abs(float(loss2[0]) - ref_loss2) <= 5e-2 * abs(ref_loss2)
    assert float((logits2.cpu().double() - ref_logits2).abs().max()) <= 0.15 * float(ref_logits2.abs().max())


def test_two_step_golden_tight(golden_dir, dev):
    """The reference's own two training steps (train_steps.npz) with the blanket tolerances of
    test_two_training_steps_golden replaced by 1e-4 on everything except the pre-BN biases."""
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model, make_args
    g = load(golden_dir, "train_steps.npz")
    args = make_args(model_config="gru_3_1_1_1_0,f_13", ptn_widths=[[16, 16, 32], [32, 16, 8]],
                     ptn_widths_stn=[[8, 16], [16, 8]], ptn_nfeat_stn=6, node_feats=6, fnet_widths=[16, 32, 16])
    model = create_model(args)
    model.ecc.load_state_dict(sub(g, "ecc0."))
    model.ptn.load_state_dict(sub(g, "ptn0."))
    skip = pre_bn_bias_keys(model.ecc, "ecc.") | pre_bn_bias_keys(model.ptn, "ptn.")
    assert "ecc.0._fnet.4.bias" in skip and "ptn.convs.0.bias" in skip and "ptn.fcs.6.bias" not in skip
    assert "ptn.convs.7.bias" in skip and "ptn.stn.convs.4.bias" in skip and "ptn.convs.4.bias" not in skip
    # The STN's projection is zero-initialised (pointnet.py:52): in step 1 every parameter INSIDE the STN
    # has an exactly zero gradient, in step 2 one of the order of Adam's eps (1e-8), where the update
    # lr*m/(sqrt(v)+eps) is ill-conditioned in any implementation.  Those tensors (not the projection
    # itself) are compared at the old blanket tolerance only.
    loose = {"ptn." + k for k, _ in model.ptn.named_parameters()
             if k.startswith("stn.convs.") or k.startswith("stn.fcs.")}
    model.to(dev)
    tr = Trainer(model, args)
    batch = dict(clouds=t(g["clouds"]), clouds_global=t(g["cglob"]), clouds_flag=t(g["flag"]),
                 edgefeats=t(g["edgefeats"]), idxn=t(g["idxn"]), degs=t(g["degs"]), labels=t(g["labels"]))
    db = HostBatch(batch).to_device(dev)
    l0, o0 = tr.train_step(db)
    l1, o1 = tr.train_step(db)
    close(o0, g["out0"], 1e-4)
    close(torch.stack([l0[0], l1[0]]), g["losses"], 1e-4)
    close(o1, g["out1"], 1e-4, 1e-4 * float(np.abs(g["out1"]).max()))
    for pre, mod in (("ecc", model.ecc), ("ptn", model.ptn)):
        sd = mod.state_dict()
        for k, v in sub(g, pre + "2.").items():
            if not nets_ref.is_param(k) or (pre + "." + k) in skip:
                continue
            d = (sd[k].cpu() - v).abs()
            if (pre + "." + k) in loose:
                assert float(d.max()) <= 5e-3 * float(v.abs().max()) + 1e-3, k
                continue
            bad = int((d > 1e-4 * max(float(v.abs().max()), 1e-3)).sum())
            assert bad <= max(1, v.numel() // 100), "%s.%s: %d of %d elements differ (max %g)" % (
                pre, k, bad, v.numel(), float(d.max()))


def test_cloud_embedder_run_golden(golden_dir, dev):
    """CloudEmbedder.run (host tensors in, as main.py:202 calls it) + GraphNetwork against the
    reference's first training step in train_steps.npz — not against this repo's other path."""
    from types import SimpleNamespace
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_pointnet import CloudEmbedder
    from superpoint_graph_b200.trainer import create_model, make_args
    g = load(golden_dir, "train_steps.npz")
    args = make_args(model_config="gru_3_1_1_1_0,f_13", ptn_widths=[[16, 16, 32], [32, 16, 8]],
                     ptn_widths_stn=[[8, 16], [16, 8]], ptn_nfeat_stn=6, node_feats=6, fnet_widths=[16, 32, 16])
    for monger in (0, 1):
        model = create_model(args)
        model.ecc.load_state_dict(sub(g, "ecc0."))
        model.ptn.load_state_dict(sub(g, "ptn0."))
        model.to(dev).train()
        emb = CloudEmbedder(SimpleNamespace(cuda=1, ptn_mem_monger=monger))
        gi = GraphConvInfo.from_arrays(g["idxn"], g["degs"], g["edgefeats"])
        model.ecc.set_info([gi], True)
        e = emb.run(model, None, t(g["flag"]), t(g["clouds"]), t(g["cglob"]))
        assert e.shape == (g["flag"].shape[0], 8)
        assert torch.all(e[torch.from_numpy(g["flag"]) == -1] == 0)  # pointnet.py:156-157
        out = model.ecc(e)
        close(out, g["out0"], 1e-4)
        loss = torch.nn.functional.cross_entropy(out, t(g["labels"], dev))
        loss.backward()
        emb.bw_hook()
        close(loss, g["losses"][0], 1e-4)
        # the gradients drive the reference's second-step logits: check them through one Adam step
        opt = torch.optim.Adam(model.parameters(), lr=1e-2)
        for p in model.parameters():
            p.grad.data.clamp_(-1, 1)
        opt.step()
        opt.zero_grad()
        e = emb.run(model, None, t(g["flag"]), t(g["clouds"]), t(g["cglob"]))
        close(model.ecc(e), g["out1"], 1e-4, 1e-4 * float(np.abs(g["out1"]).max()))


def test_sema3d_eval_chunked_vs_oracle(dev, monkeypatch):
    """configs[2]: gru_10,f_8 (cat_all, 352 -> 8), F=11, eval mode, PointNet chunked."""
    from superpoint_graph_b200 import spg_pointnet, workloads
    from superpoint_graph_b200.trainer import HostBatch
    w = workloads.get("sema3d_eval", nodes=3000)
    batch = workloads.batch(w, 7)
    model, tr, ref, _ = _model_and_oracle(w, dev)
    with torch.no_grad():  # non-trivial running statistics and STN (zero-initialised in a fresh model)
        torch.manual_seed(2)
        for m in list(model.ptn.modules()) + list(model.ecc.modules()):
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.6, 1.4)
        model.ptn.stn.proj.weight.normal_(0, 0.05)
    sd_ptn = _f64({k: v.detach().cpu().clone() for k, v in model.ptn.state_dict().items()})
    sd_ecc = _f64({k: v.detach().cpu().clone() for k, v in model.ecc.state_dict().items()})
    pcfg, mcfg = workloads.oracle_cfg(w["margs"])
    assert mcfg["cat_all"] and mcfg["fnet_widths"][-1] == 32 and pcfg["nfeat_stn"] == 11
    with torch.no_grad():
        want = nets_ref.spg_forward(_f64(batch), sd_ptn, sd_ecc, pcfg, mcfg, False)
    monkeypatch.setattr(spg_pointnet, "_EVAL_CHUNK", 1024)
    hb = HostBatch(batch)
    got = tr.eval_step(hb.to_device(dev))
    assert got.shape == (3000, 8)
    close(got, want, 1e-4)
    # the pipelined upload (chunks on a copy stream, PointNet per chunk, filter networks underneath) is the
    # same forward; thresholds lowered so that this 15 MB batch takes it, in 3 chunks
    monkeypatch.setattr(spg_pointnet.CloudEmbedder, "PIPELINE_MIN_BYTES", 1 << 20)
    monkeypatch.setattr(spg_pointnet.CloudEmbedder, "PIPELINE_CHUNK_BYTES", 4 << 20)
    assert hb.clouds.numel() * 4 >= 3 * spg_pointnet.CloudEmbedder.PIPELINE_CHUNK_BYTES
    for _ in range(2):  # second call: the copy stream and the allocator's blocks are reused
        piped = tr.eval_step_host(hb)
        close(piped, want, 1e-4)
        close(piped, got, 1e-5)


def test_vkitti_widths_train_step_vs_oracle(dev):
    """configs[3] shapes in fp32: F=9, ptn_widths [[64,64,128],[64,32,32]], STN [[32,64],[32,16]],
    minpts 15 (the bf16 variant is checked against this same oracle in test_bf16.py)."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch
    w = workloads.get("vkitti_train")
    batch = workloads.batch(w, 3)
    assert batch["clouds"].shape[1] == 9
    model, tr, ref, skip = _model_and_oracle(w, dev)
    loss, logits = tr.train_step(HostBatch(batch).to_device(dev))
    ref_loss, ref_logits = ref.step(_f64(batch))
    close(logits, ref_logits, 1e-4)
    assert abs(float(loss[0]) - ref_loss) <= 1e-4 * abs(ref_loss)
    _check_grads(model, _ref_grads(ref), skip)


def test_matrix_filters_10k_nodes_train_step_vs_oracle(dev):
    """configs[4], gru_10_0 (matrix filters [E,32,32]) at 10 000 superpoints: per-step kernels."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch
    w = workloads.get("sweep_mat", nodes=10000)
    batch = workloads.batch(w, 5)
    model, tr, ref, skip = _model_and_oracle(w, dev)
    loss, logits = tr.train_step(HostBatch(batch).to_device(dev))
    ref_loss, ref_logits = ref.step(_f64(batch))
    close(logits, ref_logits, 1e-4)
    assert abs(float(loss[0]) - ref_loss) <= 1e-4 * abs(ref_loss)
    # gradients here are float32 sums over 9e4 edges x 10 iterations of 1024-wide filter rows and over 9e3
    # clouds behind BatchNorm layers; measured 1e-5..9e-3 of the tensor maximum against the float64 truth
    _check_grads(model, _ref_grads(ref), skip, rtol=2e-2, rtol_fnet=2e-2)


def test_vector_filters_12k_nodes_fused_vs_oracle(dev, monkeypatch):
    """The fused recurrence beyond the old 9.5 k-node limit (grid-strided nodes, cooperative launch):
    against the per-step kernels and against the oracle."""
    from superpoint_graph_b200 import ops, synthetic
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    from superpoint_graph_b200.spg_graphnet import create_fnet
    from superpoint_graph_b200.spg_modules import GRUCellEx, RNNGraphConvModule
    torch.manual_seed(3)
    n = 12000
    b = synthetic.make_batch(n, k=8, seed=12, npts=8, minpts=4)
    gi = GraphConvInfo.from_arrays(b["idxn"].numpy(), b["degs"].numpy(), b["edgefeats"].numpy())
    gi.cuda()
    fnet = create_fnet([13, 32, 128, 64, 32], True, 0, 2)
    mod = RNNGraphConvModule(GRUCellEx(32, 32, bias=True, layernorm=True, ingate=True), fnet, 32, vv=True,
                             gc_info=gi, nrepeats=10, cat_all=False, use_pyg=False, cuda=True)
    sd = {k: v.clone().requires_grad_(nets_ref.is_param(k)) for k, v in mod.state_dict().items()}
    mod.to(dev).train()
    x0 = torch.randn(n, 32)
    res = []
    for fused in (True, False):
        monkeypatch.setattr(ops, "USE_FUSED_RNN", [fused])
        assert ops.rnn_vv_supported(torch.empty(1, 32, device=dev), gi.graph(), n, 32) == fused
        mod.zero_grad()
        x = x0.to(dev).requires_grad_(True)
        y = mod(x)
        (y * torch.linspace(-1, 1, y.numel(), device=dev).view_as(y)).sum().backward()
        res.append([y.detach(), x.grad.clone()] + [p.grad.clone() for p in mod.parameters()])
    for a, c in zip(*res):
        close(a, c, 1e-5, 1e-7)
    mcfg = dict(fnet_widths=[13, 32, 128, 64, 32], bnidx=2, nrepeats=10, layernorm=True, ingate=True, cat_all=False)
    xr = x0.clone().requires_grad_(True)
    yr = nets_ref.rnn_ecc_forward(xr, b["edgefeats"], b["idxn"], b["degs"], {"0." + k: v for k, v in sd.items()},
                                  "0.", mcfg, True)
    (yr * torch.linspace(-1, 1, yr.numel()).view_as(yr)).sum().backward()
    close(res[0][0], yr, 1e-4)
    close(res[0][1], xr.grad, 3e-4, 1e-6)


def test_fused_recurrence_survives_a_busy_gpu(dev):
    """The grid barrier of the fused recurrence is a cooperative launch: with another stream keeping
    the SMs busy it must still complete (the driver schedules the whole grid or nothing)."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch
    w = workloads.get("s3dis_train", nodes=512)
    batch = workloads.batch(w, 9)
    model, tr, ref, _ = _model_and_oracle(w, dev)
    db = HostBatch(batch).to_device(dev)
    loss_quiet, logits_quiet = tr.train_step(db)
    tr2_model, tr2, _, _ = _model_and_oracle(w, dev)
    noise = torch.cuda.Stream()
    a = torch.randn(8192, 8192, device=dev)
    with torch.cuda.stream(noise):
        for _ in range(30):
            a = torch.nn.functional.relu(a @ a) * 1e-4
    loss_busy, logits_busy = tr2.train_step(db)
    torch.cuda.synchronize()
    assert torch.equal(logits_busy, logits_quiet)
    close(loss_busy, loss_quiet, 1e-6)


def test_all_ignored_batch_has_nan_loss_and_zero_gradients(dev):
    """torch's cross_entropy on a batch whose labels are all -100: NaN loss, zero gradients; the
    clamp must not turn a NaN gradient into -clip (ADVICE r1)."""
    from superpoint_graph_b200 import ops
    logits = torch.randn(50, 13, device=dev)
    labels = torch.full((50,), -100, dtype=torch.int64, device=dev)
    loss, d = ops.ce_loss(logits, labels, None, -100)
    assert torch.isnan(loss).all() and torch.all(d == 0)
    p = torch.ones(8, device=dev)
    g = torch.tensor([float("nan"), 2.0, -3.0, 0.5, 0, 0, 0, 0], device=dev)
    m, v = torch.zeros(8, device=dev), torch.zeros(8, device=dev)
    ops.clamp_adam_(p, g, m, v, 1, lr=1e-2, grad_clip=1.0)
    assert torch.isnan(p[0]) and torch.isfinite(p[1:]).all()
    assert abs(float(m[1]) - 0.1) < 1e-7 and abs(float(m[2]) + 0.1) < 1e-7  # clamped to +-1, then (1-b1)*g


def test_optimizer_state_dict_matches_torch_adam(dev):
    """Trainer.optimizer_state_dict() is torch.optim.Adam's state after the same steps (checkpoint
    format of main.py:342-346), and load_optimizer_state_dict resumes bit-identically."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    w = workloads.get("s3dis_train", nodes=128)
    w["margs"].model_config = "gru_2_1_1_1_0,f_13"
    batch = workloads.batch(w, 4)
    torch.manual_seed(1)
    model = create_model(w["margs"]).to(dev)
    tr = Trainer(model, w["margs"])
    db = HostBatch(batch).to_device(dev)
    opt = torch.optim.Adam([p.detach().clone().requires_grad_(True) for p in tr.params], lr=w["margs"].lr)
    for _ in range(2):
        tr.compute_gradients(db)
        off = 0
        for q in opt.param_groups[0]["params"]:
            q.grad = tr.flat_grad[off:off + q.numel()].view(q.shape).clamp(-1, 1).clone()
            off += q.numel()
        tr.apply_update()
        opt.step()
    mine, ref = tr.optimizer_state_dict(), opt.state_dict()
    assert set(mine["state"].keys()) == set(ref["state"].keys())
    for i, st in ref["state"].items():
        assert float(mine["state"][i]["step"]) == float(st["step"]) == 2.0
        close(mine["state"][i]["exp_avg"], st["exp_avg"], 1e-5, 1e-9)
        close(mine["state"][i]["exp_avg_sq"], st["exp_avg_sq"], 1e-4, 1e-12)
    torch.manual_seed(1)
    model2 = create_model(w["margs"]).to(dev)
    tr2 = Trainer(model2, w["margs"])
    tr2.flat.copy_(tr.flat)
    for b2, b1 in zip(model2.buffers(), model.buffers()):
        b2.copy_(b1)
    tr2.load_optimizer_state_dict(mine)
    l1, o1 = tr.train_step(db)
    l2, o2 = tr2.train_step(db)
    assert torch.equal(o1, o2) and torch.equal(tr.flat, tr2.flat)


@pytest.mark.parametrize("name,nodes", [("room_fwd", 700), ("vkitti_eval", 1200)])
def test_eval_graph_replay_matches_eager(dev, name, nodes):
    """Trainer.capture_eval / replay_eval: the captured inference forward (fp32 and bf16 trunk) returns the
    eager forward's bits, also after the static inputs were refreshed from the host (HostBatch.copy_into
    re-uploads and rebuilds the graph views in place)."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    w = workloads.get(name, nodes=nodes)
    torch.manual_seed(1)
    model = create_model(w["margs"]).to(dev)
    tr = Trainer(model, w["margs"], dtype=w["dtype"])
    hb = HostBatch(workloads.batch(w, 11))
    db = hb.to_device(dev)
    eager = tr.eval_step(db).clone()
    key = tr.capture_eval(db, key=0)
    assert torch.equal(tr.replay_eval(key), eager)
    db.clouds.zero_()
    db.idxn.zero_()
    hb.copy_into(db)
    assert torch.equal(tr.replay_eval(key), eager)
    # and a training-capable Trainer still trains after an eval capture (fp32 only)
    if w["dtype"] == "f32":
        loss, _ = tr.train_step(db)
        assert torch.isfinite(loss).all()
