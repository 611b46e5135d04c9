"""Generates tests/golden/lstm.npz, lstm_plain.npz and graphnet_lstm.npz by running the reference's
LSTMCellEx and GraphNetwork on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_lstm.py

Uses the set-up and helpers of make_golden.py (igraph stub, reference import, npz writer); writes no other
file.  Every result stays under 1 MB.
"""
import numpy as np
import torch

from make_golden import graphnet, modules, npy, save, sd_np

LSTM_CONFIGS = ("lstm_3_1_1_1_0,f_13", "lstm_2,f_8", "lstm_2_1_0_0_1,f_13", "lstm_2_0,f_13")
FNET_WIDTHS, BNIDX = [13, 32, 64], 1  # narrower than graphnet_*.npz: keeps the matrix config under 1 MB


def lstm_cell():
    """LSTMCellEx (learning/modules.py:262-308) with non-zero biases and cell state; the loss weights both
    outputs, so every gradient (x, h, c and each parameter) sees hy and cy."""
    torch.manual_seed(8)
    for tag, ln, ig in (("", True, True), ("_plain", False, False)):
        cell = modules.LSTMCellEx(32, 32, bias=True, layernorm=ln, ingate=ig)
        with torch.no_grad():
            cell.bias_ih.normal_(0, 0.3)
            cell.bias_hh.normal_(0, 0.3)
        x = torch.randn(50, 32, requires_grad=True)
        h = torch.randn(50, 32, requires_grad=True)
        c = torch.randn(50, 32, requires_grad=True)
        hy, cy = cell(x, (h, c))
        g, gc = torch.randn(50, 32), torch.randn(50, 32)
        ((hy * g).sum() + (cy * gc).sum()).backward()
        arrs = dict(x=npy(x), h=npy(h), c=npy(c), hy=npy(hy), cy=npy(cy), g=npy(g), g_c=npy(gc),
                    gx=npy(x.grad), gh=npy(h.grad), gcx=npy(c.grad))
        arrs.update({"sd." + k: v for k, v in sd_np(cell).items()})
        arrs.update({"grad." + k: npy(p.grad) for k, p in cell.named_parameters()})
        save("lstm%s.npz" % tag, **arrs)


def graphnet_lstm():
    """`lstm_*` model configs through the reference's unmodified GraphNetwork and RNNGraphConvModule
    (learning/graphnet.py:66-81, modules.py:152-183, use_pyg=0).  Per config: the initial state dict, the
    training-mode output, the state after that forward (BatchNorm buffers) and the eval-mode output; for
    the vector-filter configs also the loss and every gradient.  The matrix config (`lstm_2_0`) is
    forward-only: the reference's matrix-filter backward does not run (as for graphnet_mat.npz)."""
    rng = np.random.default_rng(51)
    N = 60
    degs_np = rng.integers(0, 9, size=N)
    degs_np[[0, 31]] = 0
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn = torch.from_numpy(rng.integers(0, N, size=E).astype(np.int64))
    ef = torch.from_numpy(rng.standard_normal((E, 13)).astype(np.float32))
    labels = torch.from_numpy(rng.integers(0, 8, size=N).astype(np.int64))
    labels[[5, 6]] = -100
    cw = torch.from_numpy(rng.uniform(0.5, 2.0, size=13).astype(np.float32))

    class GI(object):  # what RNNGraphConvModule reads from a GraphConvInfo
        def get_buffers(self):
            return idxn, None, degs, None, ef

        def get_pyg_buffers(self):
            return None

    arrs = dict(idxn=npy(idxn), degs=npy(degs), edgefeats=npy(ef), labels=npy(labels), cw=npy(cw),
                configs=np.array(LSTM_CONFIGS), fnet_widths=np.array(FNET_WIDTHS), bnidx=np.array(BNIDX))
    for i, config in enumerate(LSTM_CONFIGS):
        torch.manual_seed(23 + i)
        net = graphnet.GraphNetwork(config, 32, FNET_WIDTHS, True, 0, BNIDX, 1e20, use_pyg=0, cuda=False)
        net.set_info([GI() for _ in net.gconvs], False)
        tag = "c%d." % i
        arrs.update({tag + "sd0." + k: v for k, v in sd_np(net).items()})
        emb = torch.randn(N, 32, requires_grad=True)
        net.train()
        out = net(emb)
        arrs.update({tag + "emb": npy(emb), tag + "out_train": npy(out)})
        arrs.update({tag + "sd1." + k: v for k, v in sd_np(net).items()
                     if k.endswith(("running_mean", "running_var", "num_batches_tracked"))})
        tok = config.split(",")[0].split("_")
        if len(tok) < 3 or tok[2] != "0":  # vector filters
            ncls = out.shape[1]
            loss = torch.nn.functional.cross_entropy(out, labels, weight=cw[:ncls])
            loss.backward()
            arrs.update({tag + "loss": npy(loss), tag + "gemb": npy(emb.grad)})
            arrs.update({tag + "grad." + k: npy(p.grad) for k, p in net.named_parameters()})
        net.eval()
        with torch.no_grad():
            arrs[tag + "out_eval"] = npy(net(emb.detach()))
    save("graphnet_lstm.npz", **arrs)


if __name__ == "__main__":
    torch.set_num_threads(4)
    lstm_cell()
    graphnet_lstm()
