"""Generates tests/golden/pointnet_gn.npz by running the UNMODIFIED reference's STNkD / PointNet with
norm='layer' and norm='group' on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_gn.py

Two set-ups, each with norm='layer', norm='group' (n_group 2) and, where every width divides by it,
norm='group' (n_group 4):
  * lp_*: the learned-partition embedder (supervized_partition.py defaults: STN [[16, 64], [32, 16]] on the
    first 2 of 6 features, PointNet [[32, 128], [34, 32, 32, 4]], stn_as_global, 20 points per cloud).  The
    34-wide FC layer does not divide into 4 groups, so this set-up has no n_group 4 case.
  * spg_*: an SPG-shaped PointNet with its internal STN (14 features, 128 points, small widths).
For each: the initial state dict, the training-mode output and every parameter gradient for a fixed
output gradient, the input gradient (lp: through the external STN), and the eval-mode output.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import npy, pointnet, save, sd_np  # noqa: E402  (imports the reference)


def _perturb(*mods):
    """Non-trivial GroupNorm affine parameters and STN projection (it is zero-initialised)."""
    torch.manual_seed(5)
    with torch.no_grad():
        for mod in mods:
            for m in mod.modules():
                if isinstance(m, torch.nn.GroupNorm):
                    m.weight.uniform_(0.5, 1.5)
                    m.bias.normal_(0, 0.2)
            if hasattr(mod, "proj"):
                mod.proj.weight.normal_(0, 0.2)
                mod.proj.bias.normal_(0, 0.2)
            if hasattr(mod, "stn"):
                mod.stn.proj.weight.normal_(0, 0.2)
                mod.stn.proj.bias.normal_(0, 0.2)


def learned_partition(norm, n_group, arrs):
    tag = "lp_%s%d." % (norm, n_group)
    stn = pointnet.STNkD(2, [16, 64], [32, 16], norm=norm, n_group=n_group)
    ptn = pointnet.PointNet([32, 128], [34, 32, 32, 4], [], [], 6, 0, nfeat_global=11 + 4, prelast_do=0,
                            norm=norm, n_group=n_group)
    _perturb(stn, ptn)
    arrs.update({tag + "sd0.stn." + k: v for k, v in sd_np(stn).items()})
    arrs.update({tag + "sd0.ptn." + k: v for k, v in sd_np(ptn).items()})
    torch.manual_seed(6)
    B, L = 48, 20
    clouds = (torch.randn(B, 6, L) * 0.5).requires_grad_(True)
    glob = torch.randn(B, 11)

    def embed():  # LocalCloudEmbedder.run_batch, learning/pointnet.py:195-207
        T = stn(clouds[:, :2, :])
        xy = torch.bmm(clouds[:, :2, :].transpose(1, 2), T).transpose(1, 2)
        c2 = torch.cat([xy, clouds[:, 2:, :]], 1)
        return torch.nn.functional.normalize(ptn(c2, torch.cat([glob, T.view(-1, 4)], 1)))

    stn.train(), ptn.train()
    out = embed()
    g = torch.randn_like(out)
    out.backward(g)
    stn.eval(), ptn.eval()
    with torch.no_grad():
        out_eval = embed()
    arrs.update({tag + "x": npy(clouds), tag + "xg": npy(glob), tag + "g": npy(g), tag + "out_train": npy(out),
                 tag + "out_eval": npy(out_eval), tag + "grad_x": npy(clouds.grad)})
    arrs.update({tag + "grad.stn." + k: npy(p.grad) for k, p in stn.named_parameters()})
    arrs.update({tag + "grad.ptn." + k: npy(p.grad) for k, p in ptn.named_parameters()})


SPG_CFG = dict(nf_conv=[32, 32, 64], nf_fc=[64, 32, 16], nf_conv_stn=[32, 64], nf_fc_stn=[64, 32], nfeat=14,
               nfeat_stn=11)


def spg_shaped(norm, n_group, arrs):
    tag = "spg_%s%d." % (norm, n_group)
    c = SPG_CFG
    ptn = pointnet.PointNet(c["nf_conv"], c["nf_fc"], c["nf_conv_stn"], c["nf_fc_stn"], c["nfeat"], c["nfeat_stn"],
                            prelast_do=0, norm=norm, n_group=n_group)
    _perturb(ptn)
    arrs.update({tag + "sd0." + k: v for k, v in sd_np(ptn).items()})
    torch.manual_seed(7)
    B, L = 6, 128
    x = torch.randn(B, c["nfeat"], L) * 0.5
    xg = torch.rand(B) * 3
    ptn.train()
    out = ptn(x, xg)
    g = torch.randn_like(out)
    out.backward(g)
    ptn.eval()
    with torch.no_grad():
        out_eval = ptn(x, xg)
    arrs.update({tag + "x": npy(x), tag + "xg": npy(xg), tag + "g": npy(g), tag + "out_train": npy(out),
                 tag + "out_eval": npy(out_eval)})
    arrs.update({tag + "grad." + k: npy(p.grad) for k, p in ptn.named_parameters()})


def main():
    arrs = {}
    cases = {"lp": [("layer", 1), ("group", 2)], "spg": [("layer", 1), ("group", 2), ("group", 4)]}
    for norm, n_group in cases["lp"]:
        learned_partition(norm, n_group, arrs)
    for norm, n_group in cases["spg"]:
        spg_shaped(norm, n_group, arrs)
    arrs["cases"] = json.dumps(cases)
    arrs["spg_cfg"] = json.dumps(SPG_CFG)
    save("pointnet_gn.npz", **arrs)


if __name__ == "__main__":
    main()
