"""bf16 arithmetic of the PointNet trunk (BASELINE configs[3]: "bf16"): wgmma on bf16 operands,
fp32 accumulation, activations rounded to bf16 between layers.  Checked against the fp32 oracle with a
STATED tolerance: five layers of bf16 rounding (2^-9 relative per operand) give ~1e-2 of the output scale;
the bound is 3e-2 on the PointNet outputs and on the logits of a whole inference step.  The fp32 (3xTF32)
path at the same vKITTI widths — including the 32-wide STN layer — holds 1e-4."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nets_ref  # noqa: E402  (checker only)
from test_gpu_parity import close  # noqa: E402

BF16_TOL = 3e-2


@pytest.fixture(scope="module")
def dev():
    from superpoint_graph_b200 import _lib
    _lib.lib()
    return torch.device("cuda:0")


def _net(F, conv, fc, conv_stn, fc_stn, seed):
    from superpoint_graph_b200 import spg_pointnet
    net = spg_pointnet.PointNet(conv, fc, conv_stn, fc_stn, F, F, prelast_do=0)
    torch.manual_seed(seed)
    with torch.no_grad():
        net.stn.proj.weight.normal_(0, 0.05)
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 1.5)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    return net


@pytest.mark.parametrize("name,F,conv,fc,conv_stn,fc_stn", [
    ("s3dis", 14, [64, 64, 128, 128, 256], [256, 64, 32], [64, 64, 128], [128, 64]),
    ("vkitti", 9, [64, 64, 128], [64, 32, 32], [32, 64], [32, 16]),
])
def test_pointnet_trunk_bf16_and_fp32_vs_oracle(dev, name, F, conv, fc, conv_stn, fc_stn):
    from superpoint_graph_b200 import ops
    net = _net(F, conv, fc, conv_stn, fc_stn, 11)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    B = 333
    x, xg = torch.randn(B, F, 128) * 0.4, torch.rand(B) * 3
    pcfg = dict(n_conv=len(conv), n_fc=len(fc), n_conv_stn=len(conv_stn), n_fc_stn=len(fc_stn), nfeat_stn=F)
    ref = nets_ref.pointnet_forward(x, xg, sd, pcfg, False)
    net.to(dev).eval()
    with torch.no_grad():
        ops.prof_reset()
        out32 = net(x.to(dev), xg.to(dev))
        assert ops.prof_collect().get("pointnet_fused_eval", (0, 0))[0] == 2  # fused, incl. the 32-wide STN layer
        close(out32, ref, 1e-4)
        ops.EVAL_BF16[0] = True
        try:
            out16 = net(x.to(dev), xg.to(dev))
        finally:
            ops.EVAL_BF16[0] = False
    err = float((out16.cpu() - ref).abs().max() / ref.abs().max())
    assert 1e-5 < err <= BF16_TOL, err  # really a different arithmetic, within the stated bound


def test_vkitti_inference_step_bf16_vs_fp32_oracle(dev):
    """configs[3] shapes through Trainer(dtype="bf16").eval_step against the fp32 oracle."""
    from superpoint_graph_b200 import workloads
    from superpoint_graph_b200.trainer import HostBatch, Trainer, create_model
    w = workloads.get("vkitti_eval", nodes=1500)
    assert w["dtype"] == "bf16" and w["margs"].ptn_widths_stn == [[32, 64], [32, 16]]
    batch = workloads.batch(w, 2)
    torch.manual_seed(1)
    model = create_model(w["margs"])
    with torch.no_grad():
        torch.manual_seed(5)
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.6, 1.4)
        model.ptn.stn.proj.weight.normal_(0, 0.05)
    sd_ptn = {k: v.clone() for k, v in model.ptn.state_dict().items()}
    sd_ecc = {k: v.clone() for k, v in model.ecc.state_dict().items()}
    pcfg, mcfg = workloads.oracle_cfg(w["margs"])
    with torch.no_grad():
        want = nets_ref.spg_forward(batch, sd_ptn, sd_ecc, pcfg, mcfg, False)
    model.to(dev)
    db = HostBatch(batch).to_device(dev)
    got16 = Trainer(model, w["margs"], dtype="bf16").eval_step(db)
    got32 = Trainer(model, w["margs"], dtype="f32").eval_step(db)
    close(got32, want, 1e-4)
    err = float((got16.cpu() - want).abs().max() / want.abs().max())
    assert err <= BF16_TOL, err
    with pytest.raises(NotImplementedError):
        Trainer(model, w["margs"], dtype="bf16").train_step(db)
