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


def _norm_relu(norm, w, n_group):
    """The normalisation the reference's `norm` argument selects for a layer of width w, then its ReLU."""
    mods = []
    if norm == 'batch':
        mods.append(nn.BatchNorm1d(w))
    elif norm == 'layer':
        mods.append(nn.GroupNorm(1, w))
    elif norm == 'group':
        mods.append(nn.GroupNorm(n_group, w))
    return mods + [nn.ReLU(True)]


def _stack(layer, nin, widths, norm, n_group):
    """nn.Sequential of layer(nin, widths[0]), norm, ReLU, layer(widths[0], widths[1]), norm, ReLU, ..."""
    mods = []
    for w in widths:
        mods += [layer(nin, w)] + _norm_relu(norm, w, n_group)
        nin = w
    return nn.Sequential(*mods)


def _conv1x1(nin, nout):
    return nn.Conv1d(nin, nout, 1)


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
        self.convs = _stack(_conv1x1, nfeat, nf_conv, norm, n_group)
        self.fcs = _stack(nn.Linear, nf_conv[-1], nf_fc, norm, n_group)
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
        params = []
        groups = _stn_groups(self, self.training, params)
        T = _StnFunction.apply(input, groups, self.training, *params)
        return T.view(-1, self._K, self._K) + self.eye


def _stn_groups(stn, training, params):
    """Spec groups (convs, fcs+proj) of an STNkD; its parameters are appended to `params`."""
    cs, _ = parse_sequential(stn.convs, training, params)
    fs, _ = parse_sequential(list(stn.fcs.children()) + [stn.proj], training, params)
    return cs, fs


# Segment layouts: everything of the PointNet forward/backward that depends on how the points of a
# cloud are laid out.  Point rows are [M, ld] (one point per row, features zero-padded to ld); `seg` =
# (B, L, offsets, row_seg) describes the segments to the pooling kernels (ops.segmax_fwd).
class _Layout(object):
    def segmax(self, out, pooled):
        """Max over each segment of the Deferred point rows `out` into pooled[:, :out.C]; returns argmax."""
        return ops.segmax_fwd(out.raw, out.ld, self.seg, out.C, out.scale, out.shift, out.relu, pooled,
                              pooled.shape[1])

    def segmax_backward(self, g_pool, specs, params, record, need_input_grad, grads):
        """Backward of segmax and of the point-wise chain `specs` before it; returns the point-row gradient."""
        saved, argmax = record
        # chain_backward fuses the pool backward into the last layer's BatchNorm backward
        return chain_backward(None, specs[-1].cout, self.M, specs, params, saved, need_input_grad, grads,
                              pooled=(g_pool, g_pool.shape[1], argmax, self.seg), seg=self.seg)


class _Clouds(_Layout):
    """Fixed-length clouds [B, F, L] (the reference's layout); point row b*L + l is point l of cloud b."""

    has_input_grad = True

    def __init__(self, clouds):
        self.clouds = clouds.contiguous()
        self.device = clouds.device
        self.B, self.F, self.L = self.clouds.shape
        self.M = self.B * self.L
        self.ld = _row_ld(self.F)
        self.seg = (self.B, self.L, None, None)

    def rows(self, T=None):
        """The point rows; with T [B, 4] the xy columns are transformed by T + I."""
        return ops.cloud_rows(self.clouds, T, self.ld, add_eye=T is not None)

    def xy_transform_backward(self, g_rows):
        """dT [B, 4] from the gradient w.r.t. the transformed point rows."""
        return ops.stn_apply_bwd(self.clouds, g_rows, g_rows.shape[1])

    def input_grad(self, g_rows):
        """The point-row gradient as [B, F, L]."""
        return ops.rows_to_clouds(g_rows, g_rows.shape[1], self.B, self.F, self.L)

    def fused_eval_ok(self, groups, params, nfeat_stn):
        """Whether an eval-mode forward can run each point-wise chain as one fused trunk kernel."""
        stn_g, conv_g, _ = groups
        if not conv_g or (nfeat_stn > 0 and nfeat_stn != self.F):
            return False
        chains = [conv_g] + ([stn_g[0]] if nfeat_stn > 0 else [])
        return all(_conv_layers(specs, params) is not None
                   and ops.pointnet_fused_supported(self.F, self.L, [sp.cout for sp in specs]) for specs in chains)

    def fused_pool(self, specs, params, T, pooled):
        """Eval-mode segmax of the chain `specs` over the (T-transformed) clouds in one kernel
        (csrc/pointnet_fused.cu: input tile to pooled row on chip, activations never in HBM)."""
        img, bias, widths = ops.pointnet_fused_image(_conv_layers(specs, params), self.F, bf16=ops.EVAL_BF16[0])
        ops.pointnet_fused_eval(self.clouds, T, img, bias, widths, pooled, pooled.shape[1])


class _Segments(_Layout):
    """Ragged superpoints as CSR segments: `points` [P, F] of all B superpoints back to back, int64
    `offsets` [B+1]; point row p is points[p]."""

    has_input_grad = False  # the points are data: no caller asks for their gradient

    def __init__(self, points, offsets):
        self.offsets = offsets.to(torch.int64).contiguous()
        self.device = points.device
        self.M, self.F = points.shape
        self.B = self.offsets.numel() - 1
        self.ld = _row_ld(self.F)
        self.rows0 = torch.empty((self.M, self.ld), dtype=torch.float32, device=self.device)
        ops.zero_(self.rows0)
        ops.affine_act(points.contiguous(), self.F, self.M, self.F, out=self.rows0, ldo=self.ld)
        # segment of every point row; built before any chain is queued, as it waits for the device
        self.row_seg = torch.repeat_interleave(torch.arange(self.B, device=self.device, dtype=torch.int32),
                                               self.offsets[1:] - self.offsets[:-1])
        self.seg = (self.B, 0, self.offsets, self.row_seg)

    def rows(self, T=None):
        if T is None:
            return self.rows0
        return ops.rows_xy_transform(self.rows0, T, self.row_seg, add_eye=True)

    def xy_transform_backward(self, g_rows):
        return ops.rows_xy_transform_bwd(self.rows0, g_rows, self.offsets)

    def fused_eval_ok(self, groups, params, nfeat_stn):
        return False  # the fused trunk kernel reads fixed-length clouds


def _conv_layers(specs, params):
    """[(W [N,K,1], bias, bn)] of a parsed Conv1d(k=1)+BatchNorm+ReLU chain, or None if it is not of that form.
    The parameters themselves, not views of them: ops.pointnet_fused_image caches on the tensors' identity."""
    out = []
    for sp in specs:
        if sp.bn is None or not sp.relu or not sp.bn.track_running_stats or sp.bn.running_mean is None:
            return None
        out.append((params[sp.w], params[sp.b] if sp.b is not None else None, sp.bn))
    return out


def _pool(layout, T, specs, params, training, fused, pooled):
    """Point-wise chain `specs` over the layout's point rows (xy-transformed by T + I if T is given),
    max-pooled per cloud into pooled[:, :C]; a GroupNorm layer of the chain normalises over each cloud.  Returns what its backward needs, (layer records, argmax),
    in training mode."""
    if fused:
        layout.fused_pool(specs, params, T, pooled)
        return None
    sv = [] if training else None
    out = chain_forward(Deferred(layout.rows(T), layout.ld, specs[0].cin), layout.M, specs, params, training, sv,
                        seg=layout.seg)
    argmax = layout.segmax(out, pooled)
    return (sv, argmax) if training else None


def _stn_forward(layout, groups, params, training, fused, saved):
    """STN conv chain, max-pool, FC chain + proj; returns flat T [B, K*K] (without the identity)."""
    cs, fs = groups
    B, Cs = layout.B, cs[-1].cout
    pooled = torch.empty((B, Cs), dtype=torch.float32, device=layout.device)
    conv = _pool(layout, None, cs, params, training, fused, pooled)
    sv_f = [] if training else None
    T = chain_forward(Deferred(pooled, Cs, Cs), B, fs, params, training, sv_f).materialise(B)
    if training:
        saved.update(stn_c=conv, stn_f=sv_f)
    return T


def _stn_backward(layout, dT, groups, params, saved, grads):
    cs, fs = groups
    g_pool = chain_backward(dT, dT.shape[1], layout.B, fs, params, saved["stn_f"], True, grads)
    layout.segmax_backward(g_pool, cs, params, saved["stn_c"], False, grads)


class _StnFunction(torch.autograd.Function):
    """Stand-alone STN (used by STNkD.forward and LocalCloudEmbedder)."""

    @staticmethod
    def forward(ctx, clouds, groups, training, *params):
        layout = _Clouds(clouds)
        saved = {} if training else None
        T = _stn_forward(layout, groups, params, training, False, saved)
        ctx.saved, ctx.groups, ctx.params, ctx.layout = saved, groups, params, layout
        return T

    @staticmethod
    def backward(ctx, dT):
        if ctx.saved is None:
            raise RuntimeError("backward through an eval-mode forward is not supported")
        grads = [None] * len(ctx.params)
        _stn_backward(ctx.layout, dT.contiguous(), ctx.groups, ctx.params, ctx.saved, grads)
        ctx.saved = ctx.layout = None
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
        self.convs = _stack(_conv1x1, nfeat, nf_conv, norm, n_group)
        mods = []
        for i, w in enumerate(nf_fc):
            mods.append(nn.Linear(nf_fc[i - 1] if i > 0 else nf_conv[-1] + nfeat_global, w))
            if i < len(nf_fc) - 1 or last_ac:
                mods += _norm_relu(norm, w, n_group)
            if i == len(nf_fc) - 2 and prelast_do > 0:
                mods.append(nn.Dropout(prelast_do))
        if is_res:
            nn.init.normal_(mods[-1].weight, mean=0, std=1e-2)
            nn.init.normal_(mods[-1].bias, mean=0, std=1e-2)
        self.fcs = nn.Sequential(*mods)
        self._nfeat = nfeat
        self._nfeat_global = nfeat_global

    def _groups(self, training):
        """Spec groups (stn groups | None, convs, fcs) and the flat parameter list:
        [stn convs | stn fcs+proj | convs | fcs]."""
        params = []
        stn_g = _stn_groups(self.stn, training, params) if self.nfeat_stn > 0 else None
        conv_g, _ = parse_sequential(self.convs, training, params)
        fc_g, _ = parse_sequential(self.fcs, training, params)
        return (stn_g, conv_g, fc_g), params

    def _run(self, x, layout, glob, groups, params):
        return _PointNetFunction.apply(x, layout, glob, self.nfeat_stn, groups, self.training, *params)

    def forward(self, input, input_global):
        """input [B, nfeat, L], input_global [B] | [B, G] | None -> [B, nf_fc[-1]]."""
        groups, params = self._groups(self.training)
        if input.dtype != torch.float32:
            raise TypeError("PointNet kernels are float32")
        if input_global is not None:
            input_global = input_global.reshape(input.shape[0], -1).float()
        if not self.training and input.shape[0] > _EVAL_CHUNK:
            outs = []
            for i in range(0, input.shape[0], _EVAL_CHUNK):
                x = input[i:i + _EVAL_CHUNK]
                gl = None if input_global is None else input_global[i:i + _EVAL_CHUNK]
                outs.append(self._run(x, _Clouds(x), gl, groups, params))
            return torch.cat(outs, 0)
        return self._run(input, _Clouds(input), input_global, groups, params)

    def forward_ragged(self, points, offsets, input_global):
        """Ragged superpoints (north_star; no counterpart in the reference, whose loader resamples every
        superpoint to ptn_npts points, spg.py:209-214): `points` [P, nfeat] float32 holds the points of all
        B superpoints back to back, `offsets` int64 [B+1] is the CSR boundary array, `input_global` [B] |
        [B,G] | None.  Same network, same parameters, same BatchNorm semantics (statistics over all P
        points); the max-pool runs over each superpoint's own points.  With equal-length segments the
        result equals `forward` on the [B, nfeat, L] layout."""
        groups, params = self._groups(self.training)
        if points.dtype != torch.float32 or points.dim() != 2:
            raise TypeError("ragged PointNet input must be float32 [P, nfeat]")
        B = offsets.numel() - 1
        if input_global is not None:
            input_global = input_global.reshape(B, -1).float()
        return self._run(points, _Segments(points, offsets), input_global, groups, params)


def prepack_weights(ptn, n_clouds, n_points, extra=()):
    """One launch that builds every tensor-core weight image the next training forward+backward of
    `ptn` on [n_clouds, F, n_points] will use (called by the Trainer at the start of a step).
    `extra`: further (W, ldw, transpose, N, K, k_valid) jobs, e.g. the ones a previous step had to
    pack on demand (small FC layers, filter net, classifier)."""
    from .dense import pack_jobs

    M = n_clouds * n_points
    (stn_g, conv_g, _), params = ptn._groups(True)
    ld = _row_ld(ptn._nfeat)
    jobs = pack_jobs(conv_g, params, M, ld, ptn.nfeat_stn > 0)
    if stn_g is not None:
        jobs += pack_jobs(stn_g[0], params, M, ld, False)
    seen = set((j[0].data_ptr(),) + tuple(int(v) for v in j[1:]) for j in jobs)
    jobs += [j for j in extra if ((j[0].data_ptr(),) + tuple(int(v) for v in j[1:])) not in seen]
    ops.prepack(jobs)


_EVAL_CHUNK = 16384  # clouds per eval-mode slice (bounds the [B*L, 256] activation to 2 GB)


class _PointNetFunction(torch.autograd.Function):
    """PointNet forward and backward over a segment layout (_Clouds or _Segments).  `x` is the
    layout's input tensor; it is an argument so that autograd can route its gradient."""

    @staticmethod
    def forward(ctx, x, layout, glob, nfeat_stn, groups, training, *params):
        stn_g, conv_g, fc_g = groups
        B = layout.B
        fused = not training and layout.fused_eval_ok(groups, params, nfeat_stn)
        saved = {} if training else None
        T = _stn_forward(layout, stn_g, params, training, fused, saved) if nfeat_stn > 0 else None
        Ct = conv_g[-1].cout
        G = 0 if glob is None else glob.shape[1]
        ldp = _round4(Ct + G)
        pooled = torch.empty((B, ldp), dtype=torch.float32, device=layout.device)
        conv = _pool(layout, T, conv_g, params, training, fused, pooled)
        if G > 0:
            ops.affine_act(glob.contiguous(), G, B, G, out=pooled[:, Ct:], ldo=ldp)
        sv_f = [] if training else None
        res = chain_forward(Deferred(pooled, ldp, Ct + G), B, fc_g, params, training, sv_f).materialise(B)
        if training:
            saved.update(conv=conv, fc=sv_f, Ct=Ct, G=G)
        ctx.saved, ctx.groups, ctx.params, ctx.nfeat_stn = saved, groups, params, nfeat_stn
        ctx.layout = layout if training else None
        return res

    @staticmethod
    def backward(ctx, gy):
        if ctx.saved is None:
            raise RuntimeError("backward through an eval-mode forward is not supported "
                               "(the reference never does it: learning/main.py:229-311)")
        stn_g, conv_g, fc_g = ctx.groups
        layout, params, saved, has_stn = ctx.layout, ctx.params, ctx.saved, ctx.nfeat_stn > 0
        grads = [None] * len(params)
        gy = gy.contiguous()
        want_input = ctx.needs_input_grad[0] and layout.has_input_grad
        if want_input and has_stn:
            raise NotImplementedError("input gradient of a PointNet with an internal STN is not implemented "
                                      "(the reference's callers never ask for it: the clouds are data)")
        g_pool = chain_backward(gy, gy.shape[1], layout.B, fc_g, params, saved["fc"], True, grads)
        # gradient w.r.t. the "global" inputs: the tail columns of the pooled row (pointnet.py:128-132)
        Ct, G = saved["Ct"], saved["G"]
        g_glob = g_pool[:, Ct:Ct + G].contiguous() if (ctx.needs_input_grad[2] and G > 0) else None
        g_rows = layout.segmax_backward(g_pool, conv_g, params, saved["conv"], has_stn or want_input, grads)
        del g_pool
        g_input = None
        if has_stn:
            dT = layout.xy_transform_backward(g_rows)
            del g_rows
            _stn_backward(layout, dT, stn_g, params, saved, grads)
        elif want_input:  # external transformer (LocalCloudEmbedder): hand the gradient back as [B, F, L]
            g_input = layout.input_grad(g_rows)
        ctx.saved = ctx.layout = None
        return (g_input, None, g_glob, None, None, None) + tuple(grads)


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
        training-mode forward twice and the BatchNorm running statistics see two updates.  Unlike the
        reference, the recomputation reuses the forward's dropout masks (the device counter is rewound to
        its value before the forward, then restored), so the gradient is the true gradient of the
        forward whose output was used."""
        was_training = model.training
        rng = None
        if was_training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in model.ptn.modules()):
            rng = ops.dropout_rng_state(clouds.device)
            ctr0 = rng[1].clone()
        with torch.no_grad():
            out = model.ptn(clouds, clouds_global)
        out = out.detach().requires_grad_(was_training)

        def bw_hook():
            if rng is not None:
                ctr1 = rng[1].clone()
                rng[1].copy_(ctr0)
            out_v2 = model.ptn(clouds, clouds_global)
            if rng is not None:
                rng[1].copy_(ctr1)
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
