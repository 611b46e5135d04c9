"""ORACLE (test infrastructure, never imported by the product path).

Functional CPU restatement of the reference's STNkD / PointNet with norm='layer' (nn.GroupNorm(1, C)) or
norm='group' (nn.GroupNorm(n_group, C)), learning/pointnet.py:24-47,75-133, on the reference's state-dict
keys: Conv1d|Linear, GroupNorm, ReLU at indices 3i, 3i+1, 3i+2, and in a PointNet's `fcs` a Dropout after
the second-to-last layer when prelast_do > 0 (which shifts the last Linear by one).  GroupNorm keeps no
running statistics, so training and eval differ only by that dropout.  Pinned against the reference by
tests/golden/make_golden_gn.py.
"""
import torch
import torch.nn.functional as F


def _gn_relu(x, sd, key, groups, eps=1e-5):
    return F.relu(F.group_norm(x, groups, sd[key + '.weight'], sd[key + '.bias'], eps))


def conv_stack(x, sd, prefix, n_layers, groups):
    """[Conv1d(k=1), GroupNorm, ReLU] * n; x is [B, C, L]: statistics per cloud and group."""
    for i in range(n_layers):
        x = F.conv1d(x, sd['%s%d.weight' % (prefix, 3 * i)], sd['%s%d.bias' % (prefix, 3 * i)])
        x = _gn_relu(x, sd, '%s%d' % (prefix, 3 * i + 1), groups)
    return x


def fc_stack(x, sd, prefix, n_layers, groups, last_ac=True, drop=None):
    """[Linear, GroupNorm, ReLU] * n with the activation of the last layer optional.  drop = (p, mask): the
    Dropout(p) after layer n-2 (PointNet's prelast_do) with the keep mask [B, C] it applies, or None."""
    k = 0
    for i in range(n_layers):
        x = F.linear(x, sd['%s%d.weight' % (prefix, k)], sd['%s%d.bias' % (prefix, k)])
        if i < n_layers - 1 or last_ac:
            x = _gn_relu(x, sd, '%s%d' % (prefix, k + 1), groups)
            k += 3
        else:
            k += 1
        if i == n_layers - 2 and drop is not None:
            p, mask = drop
            if mask is not None:
                x = x * mask.to(x.dtype) / (1.0 - p)
            k += 1
    return x


def stn_forward(x, sd, prefix, n_conv, n_fc, groups, K=2):
    """STNkD.forward (learning/pointnet.py:55-61): convs, max over points, fcs, proj, + identity."""
    x = conv_stack(x, sd, prefix + 'convs.', n_conv, groups)
    x = F.max_pool1d(x, x.size(2)).squeeze(2)
    x = fc_stack(x, sd, prefix + 'fcs.', n_fc, groups, last_ac=True)
    x = F.linear(x, sd[prefix + 'proj.weight'], sd[prefix + 'proj.bias'])
    return x.view(-1, K, K) + torch.eye(K, dtype=x.dtype).unsqueeze(0)


def _xy_transform(x, T):
    xy = torch.bmm(x[:, :2, :].transpose(1, 2), T).transpose(1, 2)          # :123
    return torch.cat([xy, x[:, 2:, :]], 1)                                  # :124


def pointnet_forward(x, x_global, sd, cfg, groups, prefix='', drop_mask=None):
    """PointNet.forward (learning/pointnet.py:120-133).  cfg: dict(n_conv, n_fc, n_conv_stn, n_fc_stn,
    nfeat_stn, prelast_do); drop_mask: the keep mask [B, nf_fc[-2]] of the prelast dropout in training mode,
    None in eval mode."""
    if cfg['nfeat_stn'] > 0:
        T = stn_forward(x[:, :cfg['nfeat_stn'], :], sd, prefix + 'stn.', cfg['n_conv_stn'], cfg['n_fc_stn'], groups)
        x = _xy_transform(x, T)
    x = conv_stack(x, sd, prefix + 'convs.', cfg['n_conv'], groups)
    x = F.max_pool1d(x, x.size(2)).squeeze(2)                               # :127
    if x_global is not None:
        x = torch.cat([x, x_global.view(x.shape[0], -1)], 1)                # :128-132
    drop = (cfg['prelast_do'], drop_mask) if cfg.get('prelast_do', 0) > 0 else None
    return fc_stack(x, sd, prefix + 'fcs.', cfg['n_fc'], groups, last_ac=False, drop=drop)


def pointnet_forward_ragged(points, offsets, x_global, sd, cfg, groups, prefix='', drop_mask=None):
    """PointNet.forward on ragged superpoints: `points` [P, F] of all B superpoints back to back, `offsets`
    [B+1].  GroupNorm normalises every superpoint over its own points, so each superpoint runs through the
    point-wise layers on its own as a [1, F, n_b] cloud; an empty superpoint pools to 0."""
    B = len(offsets) - 1
    C = sd[prefix + 'convs.%d.weight' % (3 * (cfg['n_conv'] - 1))].shape[0]
    pooled = []
    for b in range(B):
        o0, o1 = int(offsets[b]), int(offsets[b + 1])
        if o1 == o0:
            pooled.append(points.new_zeros(C))
            continue
        x = points[o0:o1].t().unsqueeze(0)
        if cfg['nfeat_stn'] > 0:
            T = stn_forward(x[:, :cfg['nfeat_stn'], :], sd, prefix + 'stn.', cfg['n_conv_stn'], cfg['n_fc_stn'],
                            groups)
            x = _xy_transform(x, T)
        pooled.append(conv_stack(x, sd, prefix + 'convs.', cfg['n_conv'], groups).max(2)[0][0])
    h = torch.stack(pooled)
    if x_global is not None:
        h = torch.cat([h, x_global.view(B, -1)], 1)
    drop = (cfg['prelast_do'], drop_mask) if cfg.get('prelast_do', 0) > 0 else None
    return fc_stack(h, sd, prefix + 'fcs.', cfg['n_fc'], groups, last_ac=False, drop=drop)


def is_param(key):
    """GroupNorm layers hold parameters only (no buffers)."""
    return key.endswith('.weight') or key.endswith('.bias')
