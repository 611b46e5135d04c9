"""ORACLE (test infrastructure, never imported by the product path).

CPU restatement of the reference's LSTMCellEx, the recurrent ECC module with either cell and a
GraphNetwork forward driven by a model config that may hold `lstm` tokens, on explicit state dicts with
the reference's keys, built from the pieces of oracle/nets_ref.py and oracle/crf_ref.py.  Pinned against
the reference by tests/golden/make_golden_lstm.py (lstm.npz, lstm_plain.npz, graphnet_lstm.npz).
"""
import torch
import torch.nn.functional as F

from . import crf_ref, ecc_ref, nets_ref


def lstm_cell_ex(x, h, c, sd, prefix, layernorm=True, ingate=True):
    """LSTMCellEx.forward, learning/modules.py:281-308 (the torch-0.x branch :286-294 never runs on a
    current torch).  Returns (hy, cy)."""
    if ingate:
        x = torch.sigmoid(F.linear(h, sd[prefix + 'ig.weight'], sd[prefix + 'ig.bias'])) * x  # :282-283
    gi = F.linear(x, sd[prefix + 'weight_ih'], sd.get(prefix + 'bias_ih'))                    # :296
    gh = F.linear(h, sd[prefix + 'weight_hh'], sd.get(prefix + 'bias_hh'))                    # :297
    if layernorm:                                                                             # :298, :275-279
        gi = F.instance_norm(gi.unsqueeze(1), eps=1e-5).squeeze(1)
        gh = F.instance_norm(gh.unsqueeze(1), eps=1e-5).squeeze(1)
    ingate_, forgetgate, cellgate, outgate = (gi + gh).chunk(4, 1)                            # :300
    ingate_ = torch.sigmoid(ingate_)                                                          # :301
    forgetgate = torch.sigmoid(forgetgate)                                                    # :302
    cellgate = torch.tanh(cellgate)                                                           # :303
    outgate = torch.sigmoid(outgate)                                                          # :304
    cy = (forgetgate * c) + (ingate_ * cellgate)                                              # :306
    hy = outgate * torch.tanh(cy)                                                             # :307
    return hy, cy


def rnn_ecc_forward(hx, edgefeats, idxn, degs, sd, prefix, mcfg, training, ecc_mode='vec', cell='gru'):
    """RNNGraphConvModule.forward, learning/modules.py:152-183, with cell = 'gru' (nets_ref.rnn_ecc_forward)
    or 'lstm' (the `_isLSTM` branch: c_0 = 0, only the h states are collected)."""
    if cell == 'gru':
        return nets_ref.rnn_ecc_forward(hx, edgefeats, idxn, degs, sd, prefix, mcfg, training, ecc_mode)
    w = nets_ref.fnet_forward(edgefeats, sd, prefix + '_fnet.', mcfg['fnet_widths'], mcfg['bnidx'], training)
    nc = hx.size(1)
    if w.size(1) != nc:
        w = w.view(-1, nc, nc)                                                                # :164
    hxs = [hx]
    cx = torch.zeros_like(hx)                                                                 # :168-169
    for _ in range(mcfg['nrepeats']):                                                         # :171
        if ecc_mode == 'loop':
            inp = ecc_ref.GraphConvLoop.apply(hx, w, idxn, degs)
        else:
            inp = ecc_ref.graph_conv_forward(hx, w, idxn, None, degs)                         # :175
        hx, cx = lstm_cell_ex(inp, hx, cx, sd, prefix + '_cell.', mcfg['layernorm'], mcfg['ingate'])  # :178
        hxs.append(hx)
    return torch.cat(hxs, 1) if mcfg['cat_all'] else hx                                      # :183


def graphnet_forward_config(x, edgefeats, idxn, degs, sd, config, fnet_widths, bnidx, training, prefix='',
                            ecc_mode='vec'):
    """crf_ref.graphnet_forward_config (learning/graphnet.py:40-98) that also takes `lstm` tokens
    (graphnet.py:66-81, the same arguments as `gru`).  Every other token is run by crf_ref on a view of
    the state dict (the tensors are shared, so running statistics are updated in place)."""
    def flag(tok, i):
        return bool(int(tok[i])) if len(tok) > i else True

    for d, token in enumerate(config.split(',')):
        tok = token.strip().split('_')
        p = '%s%d.' % (prefix, d)
        if tok[0] == 'lstm':
            C = x.size(1)
            vv = flag(tok, 2)
            mcfg = dict(fnet_widths=list(fnet_widths) + [C if vv else C * C], bnidx=bnidx, nrepeats=int(tok[1]),
                        layernorm=flag(tok, 3), ingate=flag(tok, 4), cat_all=flag(tok, 5))
            x = rnn_ecc_forward(x, edgefeats, idxn, degs, sd, p, mcfg, training, ecc_mode, cell='lstm')
            if training:
                crf_ref._count_batches(sd, p + '_fnet.')
        else:
            view = {'0.' + k[len(p):]: v for k, v in sd.items() if k.startswith(p)}
            x = crf_ref.graphnet_forward_config(x, edgefeats, idxn, degs, view, token, fnet_widths, bnidx,
                                                training, ecc_mode=ecc_mode)
    return x


def spg_forward_config(batch, sd_ptn, sd_ecc, pcfg, mcfg, training, ecc_mode='vec'):
    """crf_ref.spg_forward_config with `lstm` tokens."""
    emb = nets_ref.cloud_embed(batch['clouds'], batch['clouds_global'], batch['clouds_flag'], sd_ptn, pcfg,
                               training)
    return graphnet_forward_config(emb, batch['edgefeats'], batch['idxn'], batch['degs'], sd_ecc,
                                   mcfg['config'], mcfg['fnet_widths'], mcfg['bnidx'], training,
                                   ecc_mode=ecc_mode)


class RefTrainerConfig(crf_ref.RefTrainerConfig):
    """crf_ref.RefTrainerConfig (forward, weighted CE, backward, gradient clamp, Adam; learning/main.py:
    199-213) with model.ecc run by this module's graphnet_forward_config."""

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
