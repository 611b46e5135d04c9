"""GraphNetwork / create_fnet with the reference's signatures (ref: learning/graphnet.py:17-98).

The `model_config` mini-language is parsed with the reference's semantics — including the trap
that the third `gru_` token is `vv` (graphnet.py:68) although main.py's help text calls it `mv` —
and modules are registered under the same names (`'0'`, `'1'`, ...) so state dicts interchange.
Consecutive `f`/`b`/`r`/`d` tokens run as one fused Linear/BN/ReLU chain on the sm_90a kernels.
"""
import torch.nn as nn
import torch.nn.init as init

from . import spg_ecc as ecc
from .dense import run_sequential
from .spg_modules import ECC_CRFModule, GRUCellEx, LSTMCellEx, RNNGraphConvModule


def create_fnet(widths, orthoinit, llbias, bnidx=-1):
    """Filter-generating MLP over edge features: hidden layers are Linear(+BatchNorm1d right after
    hidden layer `bnidx`)+ReLU, the output layer is a bare Linear (bias iff `llbias`; BatchNorm1d
    after it iff `bnidx` addresses it).  Orthogonal init with ReLU gain on hidden layers."""
    n_hidden = len(widths) - 2
    layers = []
    for k, (fan_in, fan_out) in enumerate(zip(widths[:-1], widths[1:])):
        last = k == n_hidden
        lin = nn.Linear(fan_in, fan_out, bias=(llbias if last else True))
        if orthoinit:
            if last:
                init.orthogonal_(lin.weight)
            else:
                init.orthogonal_(lin.weight, gain=init.calculate_gain('relu'))
        layers.append(lin)
        if (not last and bnidx == k) or (last and bnidx == len(widths) - 1):
            layers.append(nn.BatchNorm1d(fan_out))
        if not last:
            layers.append(nn.ReLU(True))
    return nn.Sequential(*layers)


def _flag(tokens, pos, default=True):
    return bool(int(tokens[pos])) if len(tokens) > pos else default


class GraphNetwork(nn.Module):
    """Sequence of layers described by comma-separated `layer_arg1_arg2...` tokens:
    f_<out> (linear), b[_0] (batch norm [non-affine]), r (ReLU), d_<p> (dropout),
    gru_<R>[_vv[_layernorm[_ingate[_catall]]]] / lstm_... (recurrent ECC), crf_<R>."""

    def __init__(self, config, nfeat, fnet_widths, fnet_orthoinit=True, fnet_llbias=True,
                 fnet_bnidx=-1, edge_mem_limit=1e20, use_pyg=True, cuda=True):
        super(GraphNetwork, self).__init__()
        self.gconvs = []
        fnet_args = (fnet_orthoinit, fnet_llbias, fnet_bnidx)
        for d, token in enumerate(config.split(',')):
            tok = token.strip().split('_')
            kind, name = tok[0], str(d)
            if kind == 'f':
                width = int(tok[1])
                self.add_module(name, nn.Linear(nfeat, width))
                nfeat = width
            elif kind == 'b':
                self.add_module(name, nn.BatchNorm1d(nfeat, eps=1e-5, affine=(len(tok) == 1)))
            elif kind == 'r':
                self.add_module(name, nn.ReLU(True))
            elif kind == 'd':
                self.add_module(name, nn.Dropout(p=float(tok[1]), inplace=False))
            elif kind in ('gru', 'lstm'):
                repeats = int(tok[1])
                vv, layernorm, ingate, cat_all = (_flag(tok, i) for i in (2, 3, 4, 5))
                fnet = create_fnet(fnet_widths + [nfeat if vv else nfeat * nfeat], *fnet_args)
                cell_cls = GRUCellEx if kind == 'gru' else LSTMCellEx
                cell = cell_cls(nfeat, nfeat, bias=True, layernorm=layernorm, ingate=ingate)
                gconv = RNNGraphConvModule(cell, fnet, nfeat, vv=vv, nrepeats=repeats,
                                           cat_all=cat_all, edge_mem_limit=edge_mem_limit,
                                           use_pyg=use_pyg, cuda=cuda)
                self.add_module(name, gconv)
                self.gconvs.append(gconv)
                nfeat = nfeat * (repeats + 1) if cat_all else nfeat
            elif kind == 'crf':
                fnet = create_fnet(fnet_widths + [nfeat * nfeat], *fnet_args)
                gconv = ecc.GraphConvModule(nfeat, nfeat, fnet, edge_mem_limit=edge_mem_limit)
                self.add_module(name, ECC_CRFModule(gconv, int(tok[1])))
                self.gconvs.append(gconv)
            elif kind:
                raise NotImplementedError('Unknown module: ' + kind)

    def set_info(self, gc_infos, cuda):
        """Hands the batch's graph structure to every convolution module (i-th info -> i-th conv)."""
        if not isinstance(gc_infos, (list, tuple)):
            gc_infos = [gc_infos]
        for i, gconv in enumerate(self.gconvs):
            info = gc_infos[i]  # IndexError when fewer infos than convolutions, as graphnet.py:91-93
            if cuda:
                info.cuda()
            gconv.set_info(info)

    def forward(self, input):
        dense_run = []  # consecutive Linear/BN/ReLU/Dropout modules, executed as one fused chain

        def flush(x):
            if dense_run:
                x = run_sequential(list(dense_run), x, self.training)
                del dense_run[:]
            return x

        for module in self._modules.values():
            if isinstance(module, (nn.Linear, nn.BatchNorm1d, nn.ReLU, nn.Dropout)):
                if not dense_run and not isinstance(module, nn.Linear):
                    raise NotImplementedError(
                        "b/r/d tokens must follow an f token on the accelerated path")
                dense_run.append(module)
            else:
                input = module(flush(input))
        return flush(input)
