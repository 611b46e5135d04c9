"""The learned partition's objective and evaluation on the device: a mirror of supervized_partition/losses.py
(same function names, argument order and `args` fields) plus the boundary metrics of learning/metrics.py:87-92
and provider.py's perfect_prediction (partition/provider.py:689-695).

    from superpoint_graph_b200.spg_partition import compute_dist, compute_loss, compute_weight_loss

A training step of supervized_partition.py:218-230 then runs after the embedding without leaving the device:

    diff = compute_dist(embeddings, edg_source, edg_target, args.dist_type)
    weights_loss, pred_comp, in_comp = compute_weight_loss(args, embeddings, objects, edg_source, edg_target,
                                                           is_transition, diff, True, xyz,
                                                           partition=(pred_comp, in_comp))
    loss1, loss2 = compute_loss(args, diff, is_transition, weights_loss)

Edge arrays may be numpy int64 (what graph_collate gives) or CUDA tensors; `is_transition` and `objects` may be
CPU or CUDA tensors or numpy arrays.  Everything comes back as CUDA tensors.  Cut pursuit (`libcp`) stays on the
host: without `partition=` the schemes that need a partition call `compute_partition`, which computes cut pursuit's
edge weights on the device and then needs the reference's `libcp` module.

Differences from the reference (DESIGN.md §4): `seal` works on CUDA `objects` (the reference's np.unique fails on
them); `perfect_prediction` returns an int64 CUDA tensor (the reference: uint32 numpy);
`relax_edge_binary` returns a CUDA tensor and reproduces the reference's indexing of losses.py:184.
"""
import numpy as np
import torch

from . import ops
from ._inputs import device_of

__all__ = ["compute_dist", "compute_loss", "compute_partition", "compute_weight_loss", "compute_weights_SEAL",
           "compute_weights_XPART", "relax_edge_binary", "compute_boundary_recall", "compute_boundary_precision",
           "perfect_prediction", "partition_edge_weight", "boundary_counts", "loss_kinds"]


def _edges(edg, n_ver, dev):
    """int64 CUDA copy of an edge array; numpy arrays are range-checked on the host (IndexError, as numpy)."""
    if torch.is_tensor(edg):
        return edg.to(device=dev, dtype=torch.int64).contiguous()
    a = np.asarray(edg)
    if a.size and (int(a.min()) < 0 or int(a.max()) >= n_ver):
        raise IndexError("edge endpoint out of bounds for %d vertices" % n_ver)
    return torch.from_numpy(a.astype(np.int64, copy=False)).to(dev)


def _mask(x, dev):
    """uint8 CUDA copy of a 0/1 mask (bool, uint8 or integer; tensor or numpy)."""
    if torch.is_tensor(x):
        return x.to(device=dev).to(torch.uint8).contiguous()
    return torch.from_numpy(np.asarray(x).astype(np.uint8)).to(dev)


def _int64(x, dev):
    if torch.is_tensor(x):
        return x.to(device=dev, dtype=torch.int64).contiguous()
    return torch.from_numpy(np.asarray(x).astype(np.int64)).to(dev)


# ------------------------------------------------------------------------------------------- distance
class _DistFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, embeddings, src, tgt, dist_type):
        emb = embeddings.detach().contiguous()
        diff, coef = ops.lp_dist_fwd(emb, src, tgt, dist_type)
        ctx.dist_type = dist_type
        if ctx.needs_input_grad[0]:
            ctx.incidence = ops.lp_incidence(src, tgt, emb.shape[0])
            ctx.save_for_backward(emb, src, tgt, coef)
        return diff

    @staticmethod
    def backward(ctx, gdiff):
        emb, src, tgt, coef = ctx.saved_tensors
        return ops.lp_dist_bwd(emb, src, tgt, ctx.dist_type, coef, gdiff, ctx.incidence), None, None, None


def compute_dist(embeddings, edg_source, edg_target, dist_type):
    """diff [E] (float32 CUDA, autograd to `embeddings` [V, D]) — ref: supervized_partition/losses.py:31-42."""
    if dist_type not in ops.LP_DIST:
        raise ValueError(" %s is an unknown argument of parameter --dist_type" % (dist_type))
    if not (torch.is_tensor(embeddings) and embeddings.is_cuda and embeddings.dtype == torch.float32
            and embeddings.dim() == 2):
        raise TypeError("compute_dist takes float32 CUDA embeddings [V, D]")
    dev, V = embeddings.device, embeddings.shape[0]
    return _DistFunction.apply(embeddings, _edges(edg_source, V, dev), _edges(edg_target, V, dev), dist_type)


# ------------------------------------------------------------------------------------------- loss
class _LossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, diff, weights, is_tr, intra, inter, dist_type):
        diff = diff.detach().contiguous()
        weights = weights.detach().contiguous()
        ctx.kinds = (intra, inter, dist_type)
        ctx.save_for_backward(diff, weights, is_tr)
        return ops.lp_loss_fwd(diff, weights, is_tr, intra, inter, dist_type)

    @staticmethod
    def backward(ctx, gloss):
        diff, weights, is_tr = ctx.saved_tensors
        gdiff = ops.lp_loss_bwd(diff, weights, is_tr, *ctx.kinds, gloss.to(torch.float32).contiguous())
        return gdiff, None, None, None, None, None


def loss_kinds(loss):
    """(intra, inter) terms of --loss, by the reference's case-sensitive substring tests in its order
    ('tv' in 'TVH_zhang' is false)."""
    if "tv" in loss:
        intra = "tv"
    elif "laplacian" in loss:
        intra = "laplacian"
    elif "TVH" in loss:
        intra = "TVH"
    else:
        raise ValueError(" %s is an unknown argument of parameter --loss" % (loss))
    inter = "zhang" if "zhang" in loss else ("TVminus" if "TVminus" in loss else None)
    return intra, inter


def compute_loss(args, diff, is_transition, weights_loss):
    """(loss1, loss2): 0-dim float32 CUDA tensors with autograd to `diff`, sums accumulated in fp64 in a fixed
    order — ref: supervized_partition/losses.py:44-64 (zhang: :24-29)."""
    intra, inter = loss_kinds(args.loss)
    if inter is None:  # the reference leaves loss2 unbound
        raise UnboundLocalError("cannot access local variable 'loss2' where it is not associated with a value")
    dev = diff.device
    w = weights_loss if torch.is_tensor(weights_loss) else torch.from_numpy(np.asarray(weights_loss))
    w = w.to(device=dev, dtype=torch.float32)
    if w.numel() != diff.numel():
        raise IndexError("weights_loss has %d entries for %d edges" % (w.numel(), diff.numel()))
    loss = _LossFunction.apply(diff, w, _mask(is_transition, dev), intra, inter, args.dist_type)
    return loss[0], loss[1]


# ------------------------------------------------------------------------------------------- weights
def partition_edge_weight(args, diff):
    """Cut pursuit's edge weights (losses.py:68-72) computed on the device: float32 numpy for
    edge_weight_threshold >= 0, float64 for < 0 (exp(diff * t) / np.exp(t) promotes under numpy >= 2)."""
    w = ops.lp_edge_weight(diff.detach().to(torch.float32), args.edge_weight_threshold).cpu().numpy()
    return w if args.edge_weight_threshold < 0 else w.astype("f4")


def compute_partition(args, embeddings, edg_source, edg_target, diff, xyz=0):
    """(pred_components, pred_in_component) by cut pursuit on the host — ref: losses.py:67-89.  The edge weights
    come from the device; cut pursuit is the reference's `libcp`, which has to be importable."""
    try:
        import libcp
    except ImportError:
        raise RuntimeError("compute_partition needs the reference's cut pursuit module `libcp` "
                           "(partition/cut-pursuit); build it, or pass partition=(pred_components, "
                           "pred_in_component) to compute_weight_loss")
    edge_weight = partition_edge_weight(args, diff)
    ver_value = embeddings.detach().cpu().numpy().astype("f4")
    use_spatial = 0
    if args.spatial_emb > 0:
        ver_value = np.hstack((ver_value, args.spatial_emb * _host(xyz, "f4")))
        use_spatial = 1
    return libcp.cutpursuit(ver_value, _host(edg_source, "uint32"), _host(edg_target, "uint32"),
                            edge_weight, args.reg_strength / (4 * args.k_nn_adj), cutoff=args.CP_cutoff,
                            spatial=use_spatial, weight_decay=0.7)


def _host(x, dtype):
    """Host copy for libcp: tensors (CUDA ones included, e.g. a load_batch batch) are copied and cast to `dtype`;
    numpy arrays go through as before (edges cast to uint32, xyz as given)."""
    if torch.is_tensor(x):
        return x.detach().cpu().numpy().astype(dtype)
    return np.asarray(x).astype(dtype) if dtype == "uint32" else x


def compute_weights_SEAL(pred_components, pred_in_component, objects, edg_source, edg_target, is_transition,
                         transition_factor):
    """float32 CUDA [E] — ref: losses.py:119-128 (w per component = size - mode frequency, by a device sort of
    (component, object) pairs)."""
    dev = device_of(objects, is_transition, edg_source)
    pic = _int64(pred_in_component, dev)
    V = pic.numel()
    w, _ = ops.lp_seal(_edges(edg_source, V, dev), _edges(edg_target, V, dev), _mask(is_transition, dev), pic,
                       _int64(objects, dev), len(pred_components), transition_factor)
    return w


def compute_weights_XPART(pred_components, pred_in_component, objects, edg_source, edg_target, is_transition,
                          transition_factor, xyz=0):
    """float32 CUDA [E] — ref: losses.py:130-166: connected components of the edges that are neither true nor
    predicted transitions, then 1 + min(|c1|, |c2|) / #edges(c1, c2) * transition_factor on every transition edge,
    by a radix sort of the unordered component pairs instead of the reference's loop over them."""
    dev = device_of(is_transition, edg_source, pred_in_component)
    pic = _int64(pred_in_component, dev)
    V = pic.numel()
    return ops.lp_xpart(_edges(edg_source, V, dev), _edges(edg_target, V, dev), _mask(is_transition, dev), pic, V,
                        transition_factor)[0]


def compute_weight_loss(args, embeddings, objects, edg_source, edg_target, is_transition, diff, return_partition,
                        xyz=0, partition=None):
    """Loss weights (float32 CUDA [E]) — ref: losses.py:91-117.  partition=(pred_components, pred_in_component)
    skips cut pursuit; without it the schemes that need one (and return_partition) call compute_partition."""
    if partition is None and (args.loss_weight in ("seal", "crosspartition") or return_partition):
        partition = compute_partition(args, embeddings, edg_source, edg_target, diff, xyz)
    dev = device_of(diff, embeddings, is_transition)
    is_tr = _mask(is_transition, dev)
    E = is_tr.numel()
    if args.loss_weight == "none":
        weights = ops.lp_fill_weights(is_tr, 1.0, 1.0)
    elif args.loss_weight == "proportional":
        n_tr = int(ops.lp_count(is_tr)[1])
        with np.errstate(divide="ignore"):
            w_other = np.float32(np.float32(float(E)) / np.float32(E - n_tr))
        w_tr = float(E) / float(n_tr) * args.transition_factor  # ZeroDivisionError without transitions, as the reference
        weights = ops.lp_fill_weights(is_tr, float(w_other), w_tr)
    elif args.loss_weight == "seal":
        weights = compute_weights_SEAL(partition[0], partition[1], objects, edg_source, edg_target, is_tr,
                                       args.transition_factor)
    elif args.loss_weight == "crosspartition":
        weights = compute_weights_XPART(partition[0], partition[1], objects, edg_source, edg_target, is_tr,
                                        args.transition_factor * 2 * args.k_nn_adj, xyz)
    else:
        raise ValueError(" %s is an unknown argument of parameter --loss" % (args.loss_weight))
    if return_partition:
        return weights, partition[0], partition[1]
    return weights


# ------------------------------------------------------------------------------------------- evaluation
def relax_edge_binary(edg_binary, edg_source, edg_target, n_ver, tolerance):
    """What the reference computes (losses.py:175-186), as a CUDA tensor of the input's kind (bool stays bool,
    anything else uint8): each round marks the endpoints of the set edges, then sets edge 0 if some edge's
    source is unmarked and edge 1 if some edge's source is marked (losses.py:184 indexes with the uint8 marks),
    then every edge whose target is marked (:185)."""
    dev = device_of(edg_binary, edg_source)
    is_bool = (edg_binary.dtype == torch.bool) if torch.is_tensor(edg_binary) else np.asarray(edg_binary).dtype == bool
    relaxed = _mask(edg_binary, dev).clone()
    src, tgt = _edges(edg_source, n_ver, dev), _edges(edg_target, n_ver, dev)
    status = ops.lp_relax(relaxed, src, tgt, n_ver, tolerance)
    if relaxed.numel() < 2 and int(status[0]):
        raise IndexError("index 1 is out of bounds for axis 0 with size %d" % relaxed.numel())
    return relaxed.bool() if is_bool else relaxed


def boundary_counts(truth, pred):
    """(numerator, denominator) of 100 * ((truth == pred) * truth).sum() / truth.sum() for 0/1 masks, counted on
    the device; only these two integers come back."""
    dev = device_of(truth, pred)
    c = ops.lp_count(_mask(truth, dev), _mask(pred, dev)).cpu().numpy()
    return int(c[0]), int(c[1])


def _percent(num, den):
    with np.errstate(divide="ignore", invalid="ignore"):
        return 100 * np.int64(num) / np.int64(den)


def compute_boundary_recall(is_transition, pred_transitions):
    """ref: learning/metrics.py:87-88."""
    return _percent(*boundary_counts(is_transition, pred_transitions))


def compute_boundary_precision(is_transition, pred_transitions):
    """ref: learning/metrics.py:91-92 ((a == b) * b counts the same pairs as (b == a) * b)."""
    return _percent(*boundary_counts(pred_transitions, is_transition))


def perfect_prediction(components, labels):
    """Majority label of every point's component (ref: partition/provider.py:689-695): per component the int64
    sum of labels[:, 1:], the first maximum wins (numpy's argmax), scattered to the points.  int64 CUDA [V]; pass
    `.cpu().numpy()` to a host ConfusionMatrix."""
    dev = device_of(labels)
    lab = _int64(labels, dev)
    sizes = np.asarray([len(c) for c in components], dtype=np.int64)
    ptr = np.zeros(len(components) + 1, dtype=np.int64)
    np.cumsum(sizes, out=ptr[1:])
    ids = (np.concatenate([np.asarray(c, dtype=np.int64).reshape(-1) for c in components])
           if len(components) else np.zeros(0, dtype=np.int64))
    return ops.lp_perfect_prediction(torch.from_numpy(ptr).to(dev), torch.from_numpy(ids).to(dev), lab,
                                     lab.shape[0])
