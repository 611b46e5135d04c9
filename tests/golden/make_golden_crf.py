"""Generates tests/golden/graphnet_crf.npz by running the reference's GraphNetwork and ECC_CRFModule on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_crf.py

Uses the set-up and helpers of make_golden.py (igraph stub, reference import, npz writer); writes no other
file.  The result stays under 1 MB.
"""
import numpy as np
import torch

from make_golden import ecc, graphnet, npy, save, sd_np

CRF_CONFIGS = ("f_13,crf_3", "crf_2,f_13", "gru_2_1_1_1_0,f_8,crf_1", "f_13,crf_0")


def graphnet_crf():
    """`crf_*` model configs through the reference's unmodified GraphNetwork and ECC_CRFModule
    (learning/graphnet.py:57-64, modules.py:185-202).  Only GraphConvModule.forward is replaced: its
    legacy autograd call (learning/ecc/GraphConvModule.py:193) no longer runs, so the same body calls
    GraphConvFunction.apply, as make_golden.ecc_unit_fixture does.  Per config: the initial state dict,
    the training-mode output, the state after that forward (running statistics updated once per CRF
    iteration: its buffers) and the eval-mode output.  No gradients: the reference's matrix-filter
    backward does not run (as for graphnet_mat.npz).  Every convolution of a model gets the same graph."""

    def forward(self, input):  # learning/ecc/GraphConvModule.py:181-193 with .apply
        idxn, idxe, degs, degs_gpu, edgefeats = self._gci.get_buffers()
        weights = self._fnet(edgefeats)
        assert input.dim() == 2 and weights.dim() == 2 and (
            weights.size(1) == self._in_channels * self._out_channels or
            (self._in_channels == self._out_channels and weights.size(1) == self._in_channels))
        if weights.size(1) == self._in_channels * self._out_channels:
            weights = weights.view(-1, self._in_channels, self._out_channels)
        return ecc.GraphConvFunction.apply(input, weights, self._in_channels, self._out_channels, idxn, idxe,
                                           degs, degs_gpu, self._edge_mem_limit)

    legacy_forward, ecc.GraphConvModule.forward = ecc.GraphConvModule.forward, forward
    try:
        _graphnet_crf()
    finally:
        ecc.GraphConvModule.forward = legacy_forward


def _graphnet_crf():
    rng = np.random.default_rng(41)
    N = 50
    degs_np = rng.integers(0, 7, size=N)
    degs_np[[0, 17]] = 0
    degs_np[30] = 24  # one heavy target
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn_np = rng.integers(0, N - 1, size=E)  # node N-1 is the source of no edge
    idxn = torch.from_numpy(idxn_np.astype(np.int64))
    ef = torch.from_numpy(rng.standard_normal((E, 13)).astype(np.float32))

    class GI(object):
        def get_buffers(self):
            return idxn, None, degs, None, ef

        def get_pyg_buffers(self):
            return None

    arrs = dict(idxn=npy(idxn), degs=npy(degs), edgefeats=npy(ef), configs=np.array(CRF_CONFIGS))
    for i, config in enumerate(CRF_CONFIGS):
        torch.manual_seed(17 + i)
        net = graphnet.GraphNetwork(config, 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0, cuda=False)
        net.set_info([GI() for _ in net.gconvs], False)
        tag = "c%d." % i
        arrs.update({tag + "sd0." + k: v for k, v in sd_np(net).items()})
        emb = torch.randn(N, 32)
        net.train()
        with torch.no_grad():
            out = net(emb)
        arrs.update({tag + "emb": npy(emb), tag + "out_train": npy(out)})
        arrs.update({tag + "sd1." + k: v for k, v in sd_np(net).items()  # buffers: the parameters did not move
                     if k.endswith(("running_mean", "running_var", "num_batches_tracked"))})
        net.eval()
        with torch.no_grad():
            arrs[tag + "out_eval"] = npy(net(emb))
    save("graphnet_crf.npz", **arrs)


if __name__ == "__main__":
    torch.set_num_threads(4)
    graphnet_crf()
