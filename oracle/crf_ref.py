"""ORACLE (test infrastructure, never imported by the product path).

CPU restatement of the reference's ECC_CRFModule (`crf_<R>` model configs) and a GraphNetwork forward
driven by the model-config string, on explicit state dicts with the reference's keys, built from the
pieces of oracle/nets_ref.py.  Pinned against the reference by tests/golden/make_golden_crf.py
(graphnet_crf.npz).
"""
import torch.nn.functional as F

from . import ecc_ref, nets_ref


def _count_batches(sd, prefix):
    """num_batches_tracked += 1 for every BatchNorm under `prefix`: what a training-mode
    nn.BatchNorm1d call does besides F.batch_norm's running-statistics update."""
    for k in sd:
        if k.startswith(prefix) and k.endswith('num_batches_tracked'):
            sd[k] += 1


def crf_forward(U, edgefeats, idxn, degs, sd, prefix, fnet_widths, bnidx, nrepeats, training):
    """ECC_CRFModule.forward, learning/modules.py:195-202, with propagation = GraphConvModule(C, C, fnet)
    (graphnet.py:57-64).  As in the reference the filter network runs inside the loop, once per
    iteration, so its BatchNorm takes `nrepeats` running-statistics updates.  fnet_widths include the
    input and output widths (the output is C*C)."""
    C = U.size(1)
    fprefix = prefix + '_propagation._fnet.'
    Q = F.softmax(U, dim=1)                                                                   # :196
    for i in range(nrepeats):                                                                 # :197
        w = nets_ref.fnet_forward(edgefeats, sd, fprefix, fnet_widths, bnidx, training)       # ecc :187-191
        w = w.view(-1, C, C)
        if training:
            _count_batches(sd, fprefix)
        Q = ecc_ref.graph_conv_forward(Q, w, idxn, None, degs)                                # :198
        Q = U - Q                                                                             # :199
        if i < nrepeats - 1:
            Q = F.softmax(Q, dim=1)                                                           # :200-201
    return Q


def graphnet_forward_config(x, edgefeats, idxn, degs, sd, config, fnet_widths, bnidx, training, prefix='',
                            ecc_mode='vec'):
    """GraphNetwork(config, ...).forward (learning/graphnet.py:40-98) for `f`, `b`, `r`, `gru` and `crf`
    tokens; `fnet_widths` as given to GraphNetwork (without the output width).  Every convolution sees the
    same graph.  Training-mode dropout is random and not restated: `d_<p>` tokens must have p = 0 or run
    in eval mode."""
    def flag(tok, i):
        return bool(int(tok[i])) if len(tok) > i else True

    for d, token in enumerate(config.split(',')):
        tok = token.strip().split('_')
        kind, p = tok[0], '%s%d.' % (prefix, d)
        C = x.size(1)
        if kind == 'f':
            x = F.linear(x, sd[p + 'weight'], sd[p + 'bias'])
        elif kind == 'b':
            x = F.batch_norm(x, sd[p + 'running_mean'], sd[p + 'running_var'], sd.get(p + 'weight'),
                             sd.get(p + 'bias'), training, 0.1, 1e-5)
            if training:
                _count_batches(sd, p)
        elif kind == 'r':
            x = F.relu(x)
        elif kind == 'd':
            if training and float(tok[1]) > 0:
                raise NotImplementedError("training-mode dropout is not restated by the oracle")
        elif kind == 'gru':
            vv = flag(tok, 2)
            mcfg = dict(fnet_widths=list(fnet_widths) + [C if vv else C * C], bnidx=bnidx, nrepeats=int(tok[1]),
                        layernorm=flag(tok, 3), ingate=flag(tok, 4), cat_all=flag(tok, 5))
            x = nets_ref.rnn_ecc_forward(x, edgefeats, idxn, degs, sd, p, mcfg, training, ecc_mode)
            if training:
                _count_batches(sd, p + '_fnet.')
        elif kind == 'crf':
            x = crf_forward(x, edgefeats, idxn, degs, sd, p, list(fnet_widths) + [C * C], bnidx, int(tok[1]),
                            training)
        elif kind:
            raise NotImplementedError('Unknown module: ' + kind)
    return x


def spg_forward_config(batch, sd_ptn, sd_ecc, pcfg, mcfg, training, ecc_mode='vec'):
    """nets_ref.spg_forward with model.ecc given by mcfg = dict(config, fnet_widths, bnidx)."""
    emb = nets_ref.cloud_embed(batch['clouds'], batch['clouds_global'], batch['clouds_flag'], sd_ptn, pcfg,
                               training)
    return graphnet_forward_config(emb, batch['edgefeats'], batch['idxn'], batch['degs'], sd_ecc,
                                   mcfg['config'], mcfg['fnet_widths'], mcfg['bnidx'], training,
                                   ecc_mode=ecc_mode)


class RefTrainerConfig(nets_ref.RefTrainer):
    """nets_ref.RefTrainer (forward, weighted CE, backward, gradient clamp, Adam; learning/main.py:199-213)
    with model.ecc run by graphnet_forward_config: mcfg = dict(config=<model config string>,
    fnet_widths=<without the output width>, bnidx=...)."""

    def step(self, batch):
        self.opt.zero_grad()
        out = spg_forward_config(batch, self.sd_ptn, self.sd_ecc, self.pcfg, self.mcfg, True, self.ecc_mode)
        loss = F.cross_entropy(out, batch['labels'], weight=self.class_weights)
        loss.backward()
        if self.grad_clip > 0:
            for p in self.params:
                p.grad.clamp_(-self.grad_clip, self.grad_clip)
        self.opt.step()
        return float(loss.detach()), out.detach()
