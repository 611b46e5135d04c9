"""PointNet / STNkD / CloudEmbedder with the reference's operator signatures on top of the
sm_90a kernels.

Drop-in for `learning/pointnet.py` (ref: learning/pointnet.py:16-218): same class names,
constructor arguments, attribute names (`stn`, `convs`, `fcs`, `proj`, `nfeat_stn`), parameter
initialisation order (so `torch.manual_seed(0)` in `PointNet.__init__` yields the same initial
weights) and state-dict keys.  The nn.Sequential containers only *hold* parameters and buffers;
`forward` never calls them — it runs one hand-written forward/backward over the C-ABI
(superpoint_graph_b200.dense + csrc/pointnet.cu).
"""
import torch
import torch.nn as nn

from . import ops
from .dense import Deferred, chain_backward, chain_forward, parse_sequential


def _conv_stack(nfeat, widths, norm, n_group):
    mods = []
    for i, w in enumerate(widths):
        mods.append(nn.Conv1d(widths[i - 1] if i > 0 else nfeat, w, 1))
        if norm == 'batch':
            mods.append(nn.BatchNorm1d(w))
        elif norm == 'layer':
            mods.append(nn.GroupNorm(1, w))
        elif norm == 'group':
            mods.append(nn.GroupNorm(n_group, w))
        mods.append(nn.ReLU(True))
    return nn.Sequential(*mods)


def _round4(n):
    return (n + 3) // 4 * 4


def _row_ld(nfeat):
    """Leading dimension of the point-major input rows: zero-padded to 32 floats (one 128-byte
    swizzle row) so that the first layer runs on the tensor-core path as well."""
    return 32 if nfeat <= 32 else _round4(nfeat)


class STNkD(nn.Module):
    """Spatial transformer producing a KxK matrix per cloud (ref: learning/pointnet.py:16-61)."""

    def __init__(self, nfeat, nf_conv, nf_fc, K=2, norm='batch', affine=True, n_group=1):
        super(STNkD, self).__init__()
        self.convs = _conv_stack(nfeat, nf_conv, norm, n_group)
        mods = []
        for i, w in enumerate(nf_fc):
            mods.append(nn.Linear(nf_fc[i - 1] if i > 0 else nf_conv[-1], w))
            if norm == 'batch':
                mods.append(nn.BatchNorm1d(w))
            elif norm == 'layer':
                mods.append(nn.GroupNorm(1, w))
            elif norm == 'group':
                mods.append(nn.GroupNorm(n_group, w))
            mods.append(nn.ReLU(True))
        self.fcs = nn.Sequential(*mods)
        self.proj = nn.Linear(nf_fc[-1], K * K)
        nn.init.constant_(self.proj.weight, 0)
        nn.init.constant_(self.proj.bias, 0)
        self.eye = torch.eye(K).unsqueeze(0)
        self._K = K
        self._nfeat = nfeat

    def forward(self, input):
        """input [B, nfeat, L] -> [B, K, K] (= proj(...) + I)."""
        if self.eye.device != input.device:
            self.eye = self.eye.to(input.device)
        T = _StnFunction.apply(input, self, self.training, *_stn_params(self, self.training)[1])
        return T.view(-1, self._K, self._K) + self.eye


def _stn_params(stn, training):
    """(spec groups, flat parameter list) for convs | fcs+proj of an STNkD."""
    cs, cp = parse_sequential(stn.convs, training)
    fs, fp = parse_sequential(list(stn.fcs.children()) + [stn.proj], training)
    off = len(cp)
    for sp in fs:
        sp.w += off
        if sp.b is not None:
            sp.b += off
        if sp.gamma is not None:
            sp.gamma += off
            sp.beta += off
    return (cs, fs), cp + fp


def _stn_forward(rows, ld, B, L, groups, params, training, saved):
    """rows: raw point rows [B*L, ld]; returns flat T [B, K*K] (without the identity)."""
    cs, fs = groups
    M = B * L
    nfeat = cs[0].cin
    sv_c = [] if saved is not None else None
    out = chain_forward(Deferred(rows, ld, nfeat), M, cs, params, training, sv_c)
    Cs = out.C
    pooled = torch.empty((B, Cs), dtype=torch.float32, device=rows.device)
    argmax = ops.segmax_fwd(out.raw, out.ld, B, L, Cs, out.scale, out.shift, out.relu, pooled, Cs)
    sv_f = [] if saved is not None else None
    t = chain_forward(Deferred(pooled, Cs, Cs), B, fs, params, training, sv_f)
    T = t.materialise(B)
    if saved is not None:
        saved.update(stn_c=sv_c, stn_f=sv_f, stn_argmax=argmax, stn_Cs=Cs)
    return T


def _stn_backward(dT, B, L, groups, params, saved, grads):
    cs, fs = groups
    Cs = saved["stn_Cs"]
    g_pool = chain_backward(dT, dT.shape[1], B, fs, params, saved["stn_f"], True, grads)
    chain_backward(None, Cs, B * L, cs, params, saved["stn_c"], False, grads,
                   pooled=(g_pool, Cs, saved["stn_argmax"], B, L))


class _StnFunction(torch.autograd.Function):
    """Stand-alone STN (used by STNkD.forward and LocalCloudEmbedder)."""

    @staticmethod
    def forward(ctx, clouds, stn, training, *params):
        clouds = clouds.contiguous()
        B, F, L = clouds.shape
        groups, _ = _stn_params(stn, training)
        ld = _row_ld(F)
        rows = ops.cloud_rows(clouds, None, ld)
        saved = {} if training else None
        T = _stn_forward(rows, ld, B, L, groups, params, training, saved)
        ctx.saved, ctx.groups, ctx.params, ctx.dims = saved, groups, params, (B, L)
        return T

    @staticmethod
    def backward(ctx, dT):
        if ctx.saved is None:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        grads = [None] * len(ctx.params)
        B, L = ctx.dims
        _stn_backward(dT.contiguous(), B, L, ctx.groups, ctx.params, ctx.saved, grads)
        ctx.saved = None
        return (None, None, None) + tuple(grads)


class PointNet(nn.Module):
    """PointNet with one spatial transformer and a "global" input concatenated after the max-pool
    (ref: learning/pointnet.py:63-133)."""

    def __init__(self, nf_conv, nf_fc, nf_conv_stn, nf_fc_stn, nfeat, nfeat_stn=2, nfeat_global=1,
                 prelast_do=0.5, last_ac=False, is_res=False, norm='batch', affine=True, n_group=1,
                 last_bn=False):
        super(PointNet, self).__init__()
        torch.manual_seed(0)  # ref: learning/pointnet.py:78 (part of the observable behaviour)
        if nfeat_stn > 0:
            self.stn = STNkD(nfeat_stn, nf_conv_stn, nf_fc_stn, norm=norm, n_group=n_group)
        self.nfeat_stn = nfeat_stn
        self.convs = _conv_stack(nfeat, nf_conv, norm, n_group)
        mods = []
        for i, w in enumerate(nf_fc):
            mods.append(nn.Linear(nf_fc[i - 1] if i > 0 else nf_conv[-1] + nfeat_global, w))
            if i < len(nf_fc) - 1 or last_ac:
                if norm == 'batch':
                    mods.append(nn.BatchNorm1d(w))
                elif norm == 'layer':
                    mods.append(nn.GroupNorm(1, w))
                elif norm == 'group':
                    mods.append(nn.GroupNorm(n_group, w))
                mods.append(nn.ReLU(True))
            if i == len(nf_fc) - 2 and prelast_do > 0:
                mods.append(nn.Dropout(prelast_do))
        if is_res:
            nn.init.normal_(mods[-1].weight, mean=0, std=1e-2)
            nn.init.normal_(mods[-1].bias, mean=0, std=1e-2)
        self.fcs = nn.Sequential(*mods)
        self._nfeat = nfeat
        self._nfeat_global = nfeat_global

    def _groups(self, training):
        """Spec groups and the flat parameter list: [stn convs | stn fcs+proj | convs | fcs]."""
        params = []
        stn_groups = None
        if self.nfeat_stn > 0:
            stn_groups, params = _stn_params(self.stn, training)
            params = list(params)
        groups = []
        for seq in (self.convs, self.fcs):
            sp, pp = parse_sequential(seq, training)
            off = len(params)
            for s in sp:
                s.w += off
                if s.b is not None:
                    s.b += off
                if s.gamma is not None:
                    s.gamma += off
                    s.beta += off
            params += pp
            groups.append(sp)
        return stn_groups, groups[0], groups[1], params

    def forward(self, input, input_global):
        """input [B, nfeat, L], input_global [B] | [B, G] | None -> [B, nf_fc[-1]]."""
        training = self.training
        stn_g, conv_g, fc_g, params = self._groups(training)
        if input_global is not None:
            input_global = input_global.reshape(input.shape[0], -1).float()
        if not training and input.shape[0] > _EVAL_CHUNK:
            outs = []
            for i in range(0, input.shape[0], _EVAL_CHUNK):
                gl = None if input_global is None else input_global[i:i + _EVAL_CHUNK]
                outs.append(_PointNetFunction.apply(input[i:i + _EVAL_CHUNK], gl, self.nfeat_stn,
                                                    (stn_g, conv_g, fc_g), training, *params))
            return torch.cat(outs, 0)
        return _PointNetFunction.apply(input, input_global, self.nfeat_stn, (stn_g, conv_g, fc_g),
                                       training, *params)


    def forward_ragged(self, points, offsets, input_global):
        """Ragged superpoints (north_star; no counterpart in the reference, whose loader resamples every
        superpoint to ptn_npts points, spg.py:209-214): `points` [P, nfeat] float32 holds the points of all
        B superpoints back to back, `offsets` int64 [B+1] is the CSR boundary array, `input_global` [B] |
        [B,G] | None.  Same network, same parameters, same BatchNorm semantics (statistics over all P
        points); the max-pool runs over each superpoint's own points.  With equal-length segments the
        result equals `forward` on the [B, nfeat, L] layout."""
        training = self.training
        stn_g, conv_g, fc_g, params = self._groups(training)
        B = offsets.numel() - 1
        if input_global is not None:
            input_global = input_global.reshape(B, -1).float()
        return _PointNetRaggedFunction.apply(points, offsets, input_global, self.nfeat_stn,
                                             (stn_g, conv_g, fc_g), training, *params)


def prepack_weights(ptn, n_clouds, n_points, extra=()):
    """One launch that builds every tensor-core weight image the next training forward+backward of
    `ptn` on [n_clouds, F, n_points] will use (called by the Trainer at the start of a step).
    `extra`: further (W, ldw, transpose, N, K, k_valid) jobs, e.g. the ones a previous step had to
    pack on demand (small FC layers, filter net, classifier)."""
    from .dense import pack_jobs

    M = n_clouds * n_points
    stn_g, conv_g, fc_g, params = ptn._groups(True)
    ld = _row_ld(ptn._nfeat)
    jobs = pack_jobs(conv_g, params, M, ld, ptn.nfeat_stn > 0)
    if stn_g is not None:
        jobs += pack_jobs(stn_g[0], params, M, ld, False)
    seen = set((j[0].data_ptr(),) + tuple(int(v) for v in j[1:]) for j in jobs)
    jobs += [j for j in extra if ((j[0].data_ptr(),) + tuple(int(v) for v in j[1:])) not in seen]
    ops.prepack(jobs)


_EVAL_CHUNK = 16384  # clouds per eval-mode slice (bounds the [B*L, 256] activation to 2 GB)


class _PointNetFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, clouds, glob, nfeat_stn, groups, training, *params):
        stn_g, conv_g, fc_g = groups
        clouds = clouds.contiguous()
        if clouds.dtype != torch.float32:
            raise TypeError("PointNet kernels are float32")
        B, F, L = clouds.shape
        M = B * L
        ld = _row_ld(F)
        if not training and _fused_eval_ok(groups, params, F, L, nfeat_stn):
            ctx.saved = None
            return _fused_eval_forward(clouds, glob, nfeat_stn, groups, params)
        saved = {} if training else None
        T = None
        if nfeat_stn > 0:
            rows0 = ops.cloud_rows(clouds, None, ld)
            T = _stn_forward(rows0, ld, B, L, stn_g, params, training, saved)
            rows = ops.cloud_rows(clouds, T, ld, add_eye=True)
            del rows0
        else:
            rows = ops.cloud_rows(clouds, None, ld)
        sv_c = [] if training else None
        out = chain_forward(Deferred(rows, ld, F), M, conv_g, params, training, sv_c)
        Ct = out.C
        G = 0 if glob is None else glob.shape[1]
        ldp = _round4(Ct + G)
        pooled = torch.empty((B, ldp), dtype=torch.float32, device=clouds.device)
        argmax = ops.segmax_fwd(out.raw, out.ld, B, L, Ct, out.scale, out.shift, out.relu, pooled,
                                ldp)
        if G > 0:
            glob = glob.contiguous()
            ops.affine_act(glob, G, B, G, out=pooled[:, Ct:], ldo=ldp)
        sv_f = [] if training else None
        y = chain_forward(Deferred(pooled, ldp, Ct + G), B, fc_g, params, training, sv_f)
        res = y.materialise(B)
        if training:
            saved.update(conv=sv_c, fc=sv_f, argmax=argmax, Ct=Ct, G=G, ld=ld)
        ctx.saved, ctx.groups, ctx.params = saved, groups, params
        ctx.dims = (B, F, L, nfeat_stn)
        ctx.clouds = clouds if (training and nfeat_stn > 0) else None
        return res

    @staticmethod
    def backward(ctx, gy):
        if ctx.saved is None:
            raise RuntimeError("backward through an eval-mode forward is not supported "
                               "(the reference never does it: learning/main.py:229-311)")
        stn_g, conv_g, fc_g = ctx.groups
        params, saved = ctx.params, ctx.saved
        B, F, L, nfeat_stn = ctx.dims
        grads = [None] * len(params)
        gy = gy.contiguous()
        Ct, ld = saved["Ct"], saved["ld"]
        want_clouds, want_glob = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if want_clouds and nfeat_stn > 0:
            raise NotImplementedError("input gradient of a PointNet with an internal STN is not implemented "
                                      "(the reference's callers never ask for it: the clouds are data)")
        g_pool = chain_backward(gy, gy.shape[1], B, fc_g, params, saved["fc"], True, grads)
        # gradient w.r.t. the "global" inputs: the tail columns of the pooled row (pointnet.py:128-132)
        g_glob = g_pool[:, Ct:Ct + saved["G"]].contiguous() if (want_glob and saved["G"] > 0) else None
        g_rows = chain_backward(None, Ct, B * L, conv_g, params, saved["conv"], nfeat_stn > 0 or want_clouds, grads,
                                pooled=(g_pool, g_pool.shape[1], saved["argmax"], B, L))
        del g_pool
        g_clouds = None
        if nfeat_stn > 0:
            dT = ops.stn_apply_bwd(ctx.clouds, g_rows, g_rows.shape[1])
            del g_rows
            _stn_backward(dT, B, L, stn_g, params, saved, grads)
        elif want_clouds:  # external transformer (LocalCloudEmbedder): hand the gradient back as [B, F, L]
            g_clouds = ops.rows_to_clouds(g_rows, g_rows.shape[1], B, F, L)
        ctx.saved = None
        ctx.clouds = None
        return (g_clouds, g_glob, None, None, None) + tuple(grads)


def _conv_layers(specs, params):
    """[(W2d, bias, bn)] of a parsed Conv1d(k=1)+BatchNorm+ReLU chain, or None if it is not of that form."""
    out = []
    for sp in specs:
        if sp.bn is None or not sp.relu or not sp.bn.track_running_stats or sp.bn.running_mean is None:
            return None
        W = params[sp.w]
        W = W.view(W.shape[0], W.shape[1]) if W.dim() == 3 else W
        out.append((W, params[sp.b] if sp.b is not None else None, sp.bn))
    return out


def _fused_eval_ok(groups, params, F, L, nfeat_stn):
    stn_g, conv_g, fc_g = groups
    if not conv_g or _conv_layers(conv_g, params) is None:
        return False
    if not ops.pointnet_fused_supported(F, L, [sp.cout for sp in conv_g]):
        return False
    if nfeat_stn > 0:
        if nfeat_stn != F or _conv_layers(stn_g[0], params) is None:
            return False
        if not ops.pointnet_fused_supported(F, L, [sp.cout for sp in stn_g[0]]):
            return False
    return True


def _fused_eval_forward(clouds, glob, nfeat_stn, groups, params):
    """Eval-mode PointNet with both point-wise chains fused (ops.pointnet_fused_eval: input tile to pooled row
    on chip); only the [B, C] pooled rows and the small FC chains touch HBM.  ref: pointnet.py:120-133."""
    stn_g, conv_g, fc_g = groups
    B, F, L = clouds.shape
    dev = clouds.device
    T = None
    if nfeat_stn > 0:
        cs, fs = stn_g
        img, bias, widths = ops.pointnet_fused_image(_conv_layers(cs, params), F, bf16=ops.EVAL_BF16[0])
        Cs = cs[-1].cout
        pooled_s = torch.empty((B, Cs), dtype=torch.float32, device=dev)
        ops.pointnet_fused_eval(clouds, None, img, bias, widths, pooled_s, Cs)
        T = chain_forward(Deferred(pooled_s, Cs, Cs), B, fs, params, False, None).materialise(B)
    img, bias, widths = ops.pointnet_fused_image(_conv_layers(conv_g, params), F, bf16=ops.EVAL_BF16[0])
    Ct = conv_g[-1].cout
    G = 0 if glob is None else glob.shape[1]
    ldp = _round4(Ct + G)
    pooled = torch.empty((B, ldp), dtype=torch.float32, device=dev)
    ops.pointnet_fused_eval(clouds, T, img, bias, widths, pooled, ldp)
    if G > 0:
        ops.affine_act(glob.contiguous(), G, B, G, out=pooled[:, Ct:], ldo=ldp)
    return chain_forward(Deferred(pooled, ldp, Ct + G), B, fc_g, params, False, None).materialise(B)


class _PointNetRaggedFunction(torch.autograd.Function):
    """PointNet over CSR segments: the dense chains of _PointNetFunction with segmax_csr_* /
    rows_xy_transform* in place of the constant-L kernels."""

    @staticmethod
    def forward(ctx, points, offsets, glob, nfeat_stn, groups, training, *params):
        stn_g, conv_g, fc_g = groups
        if points.dtype != torch.float32 or points.dim() != 2:
            raise TypeError("ragged PointNet input must be float32 [P, nfeat]")
        offsets = offsets.to(torch.int64).contiguous()
        P, F = points.shape
        B = offsets.numel() - 1
        ld = _row_ld(F)
        rows0 = torch.empty((P, ld), dtype=torch.float32, device=points.device)
        ops.zero_(rows0)
        ops.affine_act(points.contiguous(), F, P, F, out=rows0, ldo=ld)
        row_seg = torch.repeat_interleave(torch.arange(B, device=points.device, dtype=torch.int32),
                                          (offsets[1:] - offsets[:-1]))
        saved = {} if training else None
        T = None
        rows = rows0
        if nfeat_stn > 0:
            cs, fs = stn_g
            sv_c = [] if training else None
            o = chain_forward(Deferred(rows0, ld, cs[0].cin), P, cs, params, training, sv_c)
            Cs = o.C
            pooled_s = torch.empty((B, Cs), dtype=torch.float32, device=points.device)
            am_s = ops.segmax_csr_fwd(o.raw, o.ld, offsets, Cs, o.scale, o.shift, o.relu, pooled_s, Cs)
            sv_f = [] if training else None
            t = chain_forward(Deferred(pooled_s, Cs, Cs), B, fs, params, training, sv_f)
            T = t.materialise(B)
            rows = ops.rows_xy_transform(rows0, T, row_seg, add_eye=True)
            if training:
                saved.update(stn_c=sv_c, stn_f=sv_f, stn_am=am_s, stn_Cs=Cs)
        sv_c = [] if training else None
        out = chain_forward(Deferred(rows, ld, F), P, conv_g, params, training, sv_c)
        Ct = out.C
        G = 0 if glob is None else glob.shape[1]
        ldp = _round4(Ct + G)
        pooled = torch.empty((B, ldp), dtype=torch.float32, device=points.device)
        am = ops.segmax_csr_fwd(out.raw, out.ld, offsets, Ct, out.scale, out.shift, out.relu, pooled, ldp)
        if G > 0:
            ops.affine_act(glob.contiguous(), G, B, G, out=pooled[:, Ct:], ldo=ldp)
        sv_f = [] if training else None
        y = chain_forward(Deferred(pooled, ldp, Ct + G), B, fc_g, params, training, sv_f)
        res = y.materialise(B)
        if training:
            saved.update(conv=sv_c, fc=sv_f, am=am, Ct=Ct)
        ctx.saved, ctx.groups, ctx.params = saved, groups, params
        ctx.dims = (B, P, nfeat_stn)
        ctx.aux = (offsets, rows0) if (training and nfeat_stn > 0) else None
        return res

    @staticmethod
    def backward(ctx, gy):
        if ctx.saved is None:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        stn_g, conv_g, fc_g = ctx.groups
        params, saved = ctx.params, ctx.saved
        B, P, nfeat_stn = ctx.dims
        grads = [None] * len(params)
        Ct = saved["Ct"]
        g_pool = chain_backward(gy.contiguous(), gy.shape[1], B, fc_g, params, saved["fc"], True, grads)
        G = ops.segmax_csr_bwd(g_pool, g_pool.shape[1], saved["am"], P, Ct)
        g_rows = chain_backward(G, Ct, P, conv_g, params, saved["conv"], nfeat_stn > 0, grads, own_g=True)
        if nfeat_stn > 0:
            offsets, rows0 = ctx.aux
            cs, fs = stn_g
            dT = ops.rows_xy_transform_bwd(rows0, g_rows, offsets)
            g_ps = chain_backward(dT, 4, B, fs, params, saved["stn_f"], True, grads)
            Gs = ops.segmax_csr_bwd(g_ps, g_ps.shape[1], saved["stn_am"], P, saved["stn_Cs"])
            chain_backward(Gs, saved["stn_Cs"], P, cs, params, saved["stn_c"], False, grads, own_g=True)
        ctx.saved = ctx.aux = None
        return (None, None, None, None, None, None) + tuple(grads)


class CloudEmbedder():
    """Evaluates PointNet on the superpoints that have a cloud and scatters the result into
    zero-filled descriptors (ref: learning/pointnet.py:138-180)."""

    def __init__(self, args):
        self.args = args
        self.bw_hook = lambda: None
        self.run = self.run_full_monger if args.ptn_mem_monger else self.run_full

    def _prep(self, clouds_flag, clouds, clouds_global):
        idx_valid = torch.nonzero(clouds_flag.eq(0)).reshape(-1)
        if not self.args.cuda:
            raise RuntimeError("superpoint_graph_b200 runs on CUDA only (args.cuda must be 1)")
        dev = torch.device("cuda", torch.cuda.current_device())
        return (clouds.to(dev, non_blocking=True), clouds_global.to(dev, non_blocking=True),
                idx_valid.to(dev, non_blocking=True))

    def run_full(self, model, clouds_meta, clouds_flag, clouds, clouds_global):
        if (not model.training and not clouds.is_cuda and clouds.is_pinned() and clouds_global.is_pinned()
                and clouds.numel() * clouds.element_size() >= self.PIPELINE_MIN_BYTES and self.args.cuda):
            dev = torch.device("cuda", torch.cuda.current_device())
            idx_valid = torch.nonzero(clouds_flag.eq(0)).reshape(-1).to(dev, non_blocking=True)
            return self.run_pipelined(model, clouds, clouds_global, idx_valid, clouds_flag.size(0))
        clouds, clouds_global, idx_valid = self._prep(clouds_flag, clouds, clouds_global)
        return self._embed_full(model, clouds, clouds_global, idx_valid, clouds_flag.size(0))

    def run_full_monger(self, model, clouds_meta, clouds_flag, clouds, clouds_global):
        clouds, clouds_global, idx_valid = self._prep(clouds_flag, clouds, clouds_global)
        return self._embed_monger(model, clouds, clouds_global, idx_valid, clouds_flag.size(0))

    # Large uploads go in a few chunks so that the forward of chunk i overlaps the copy of chunk i+1; more
    # chunks make the step issue-bound on the host (every chunk is ~25 launches)
    PIPELINE_MIN_BYTES = 16 << 20
    PIPELINE_CHUNK_BYTES = 14 << 20
    PIPELINE_CHUNKS = 4

    @torch.no_grad()
    def run_pipelined(self, model, clouds, clouds_global, idx_valid, n_rows, overlap=None):
        """Inference from PINNED host clouds: the upload (the dominant cost of a whole-scene batch: 115 MB
        for 20 000 superpoints against 3.9 ms of compute) is cut into chunks on a copy stream and PointNet
        starts on chunk k while chunk k+1 is in flight — eval-mode PointNet is independent per superpoint
        (BatchNorm uses running statistics), so chunking does not change the result.  `overlap` (a
        callable) is run on the compute stream after the copies are queued: work that does not need the
        clouds (the ECC filter networks).  idx_valid is a device tensor."""
        assert not model.training, "the pipelined path is for eval-mode forwards"
        dev = idx_valid.device
        nv = clouds.size(0)
        main = torch.cuda.current_stream(dev)
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        cs = self._copy_stream
        nbytes = clouds.numel() * clouds.element_size()
        nchunk = max(1, min(self.PIPELINE_CHUNKS, nbytes // self.PIPELINE_CHUNK_BYTES, nv // 512))
        bounds = [(nv * k) // nchunk for k in range(nchunk + 1)]
        d_clouds = torch.empty(clouds.shape, dtype=clouds.dtype, device=dev)
        d_glob = torch.empty(clouds_global.shape, dtype=clouds_global.dtype, device=dev)
        cs.wait_stream(main)  # the allocator may hand out blocks whose last use is still queued on `main`
        events = []
        with torch.cuda.stream(cs):
            d_glob.copy_(clouds_global, non_blocking=True)
            for k in range(nchunk):
                a, b = bounds[k], bounds[k + 1]
                d_clouds[a:b].copy_(clouds[a:b], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(cs)
                events.append(ev)
        if overlap is not None:
            overlap()
        out = None
        for k in range(nchunk):
            a, b = bounds[k], bounds[k + 1]
            main.wait_event(events[k])
            o = model.ptn(d_clouds[a:b], d_glob[a:b])
            if out is None:
                out = torch.empty((nv, o.shape[1]), dtype=o.dtype, device=dev)
            out[a:b] = o
        if out is None:
            out = model.ptn(d_clouds, d_glob)
        return ops.rows_scatter(out, idx_valid, n_rows)

    def run_resident(self, model, clouds, clouds_global, idx_valid, n_rows):
        """`run` for a batch that already lives on the device (Trainer / CUDA-graph path): same
        embedding code as run_full / run_full_monger minus the H2D copies and the host-side
        `nonzero` of the flags (done once when the batch was collated)."""
        fn = self._embed_monger if self.args.ptn_mem_monger else self._embed_full
        return fn(model, clouds, clouds_global, idx_valid, n_rows)

    def _embed_full(self, model, clouds, clouds_global, idx_valid, n_rows):
        out = model.ptn(clouds, clouds_global)
        return _ScatterRows.apply(out, idx_valid, n_rows)

    def _embed_monger(self, model, clouds, clouds_global, idx_valid, n_rows):
        """Memory mongering (ref: learning/pointnet.py:160-180): forward without saving, full
        recomputation in `bw_hook`.  As in the reference, a training step therefore runs the
        training-mode forward twice and the BatchNorm running statistics see two updates."""
        was_training = model.training
        with torch.no_grad():
            out = model.ptn(clouds, clouds_global)
        out = out.detach().requires_grad_(was_training)

        def bw_hook():
            out_v2 = model.ptn(clouds, clouds_global)
            out_v2.backward(out.grad)

        self.bw_hook = bw_hook
        return _ScatterRows.apply(out, idx_valid, n_rows)


class _ScatterRows(torch.autograd.Function):
    """descriptors = zeros[N, C]; descriptors[idx] = out (ref: learning/pointnet.py:156-157)."""

    @staticmethod
    def forward(ctx, out, idx, n_rows):
        ctx.save_for_backward(idx)
        return ops.rows_scatter(out, idx, n_rows)

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        return ops.rows_gather(g.contiguous(), idx), None, None


class LocalCloudEmbedder():
    """Learned-partition embedder: external STN, xy transform, tiny PointNet, L2 normalisation
    (ref: learning/pointnet.py:182-218).  Signature kept; the PointNet/STN run on the fused path,
    the 65535-cloud chunking of the reference (a cuDNN limit) is unnecessary here."""

    def __init__(self, args):
        self.nfeat_stn = args.ptn_nfeat_stn
        self.stn_as_global = args.stn_as_global

    def run_batch(self, model, clouds, clouds_global, *excess):
        if self.nfeat_stn > 0:
            T = model.stn(clouds[:, :self.nfeat_stn, :])
            xy_transf = torch.bmm(clouds[:, :2, :].transpose(1, 2), T).transpose(1, 2)
            clouds = torch.cat([xy_transf, clouds[:, 2:, :]], 1)
            if self.stn_as_global:
                clouds_global = torch.cat([clouds_global, T.view(-1, 4)], 1)
        out = model.ptn(clouds, clouds_global)
        return nn.functional.normalize(out)

    def run_batch_cpu(self, model, clouds, clouds_global, *excess):
        batch_size = 2 ** 10 - 1
        outs = []
        for i in range(0, clouds.shape[0], batch_size):
            outs.append(self.run_batch(model, clouds[i:i + batch_size], clouds_global[i:i + batch_size]).cpu())
        return torch.cat(outs)
