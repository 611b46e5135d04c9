"""CPU restatement of the learned partition's objective and evaluation (ref: supervized_partition/losses.py,
learning/metrics.py:87-92, partition/provider.py:689-695), pinned by tests/golden/partition.npz.

Distances and losses are torch functions of whatever dtype they are given (float64 for the gradient checks).
The weights follow numpy's float32/float64 promotion as the reference meets it (numpy >= 2: a float64 scalar
added to a float32 array computes in float64 and rounds once on assignment).  `compute_weights_XPART` keeps the
reference's per-pair loop over the transition edges: `tools/bench_partition.py` times it as the host arm.
libply_c's `connected_comp` (cutoff 0) is `connected_comp` below, on scipy: both number the components by their
smallest vertex.
"""
import numpy as np
import torch

ZHANG_BETA = {"euclidian": 1.0, "scalar": 1.0, "intrinsic": 1.0471975512}
SMOOTH = 0.999


def compute_dist(embeddings, edg_source, edg_target, dist_type):
    xs, xt = embeddings[edg_source, :], embeddings[edg_target, :]
    if dist_type == "euclidian":
        return ((xs - xt) ** 2).sum(1)
    if dist_type == "intrinsic":
        a0, a1 = np.arccos(SMOOTH), np.arccos(-SMOOTH)
        return (torch.acos((xs * xt).sum(1) * SMOOTH) - a0) / (a1 - a0) * 3.141592
    if dist_type == "scalar":
        return (xs * xt).sum(1) - 1
    raise ValueError(" %s is an unknown argument of parameter --dist_type" % (dist_type))


def loss_kinds(loss):
    """(intra, inter) term names chosen by the reference's case-sensitive substring tests, in its order."""
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
    intra, inter = loss_kinds(args.loss)
    m1 = is_transition == 0
    d1, w1 = diff[m1], weights_loss[m1]
    if intra == "tv":
        loss1 = (w1 * torch.sqrt(d1 + 1e-10)).sum()
    elif intra == "laplacian":
        loss1 = (w1 * d1).sum()
    else:
        delta = 0.2
        loss1 = delta * (w1 * (torch.sqrt(1 + d1 / delta ** 2) - 1)).sum()
    m2 = is_transition == 1
    d2, w2 = diff[m2], weights_loss[m2]
    if inter == "zhang":
        x = torch.sqrt(d2 + 1e-10)
        loss2 = torch.clamp(-w2 * x + w2 * ZHANG_BETA[args.dist_type], min=0).sum()
    elif inter == "TVminus":
        loss2 = (torch.sqrt(d2 + 1e-10) * w2).sum()
    else:  # the reference leaves loss2 unbound
        raise UnboundLocalError("cannot access local variable 'loss2' where it is not associated with a value")
    return loss1, loss2


def connected_comp(n_ver, edg_source, edg_target, active, cutoff=0):
    """libply_c.connected_comp with cutoff 0: (list of member arrays, in_component), numbered by smallest vertex."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    assert cutoff == 0
    act = np.asarray(active) > 0
    s, t = np.asarray(edg_source)[act], np.asarray(edg_target)[act]
    g = coo_matrix((np.ones(len(s), dtype=np.int8), (s, t)), shape=(n_ver, n_ver))
    n, lab = connected_components(g, directed=False)
    order = np.argsort(lab, kind="stable")
    bounds = np.searchsorted(lab[order], np.arange(n + 1))
    return [order[bounds[i]:bounds[i + 1]].astype(np.uint32) for i in range(n)], lab.astype(np.uint32)


def mode_frequency(values):
    return np.unique(np.asarray(values), return_counts=True)[1].max()


def compute_weights_SEAL(pred_components, pred_in_component, objects, edg_source, edg_target, is_transition,
                         transition_factor):
    weights = np.ones((len(edg_source),), dtype="float32")
    objects = np.asarray(objects)
    w_comp = np.array([len(c) - mode_frequency(objects[c]) for c in pred_components], dtype="uint32")
    tr = np.nonzero(np.asarray(is_transition))[0]
    w = np.maximum(w_comp[pred_in_component[edg_source[tr]]], w_comp[pred_in_component[edg_target[tr]]])
    weights[tr] = weights[tr] + w * transition_factor
    return weights


def compute_weights_XPART(pred_components, pred_in_component, objects, edg_source, edg_target, is_transition,
                          transition_factor, xyz=0):
    """The reference's algorithm as it is: one boolean mask over all transition edges per component pair."""
    weights = np.ones((len(edg_source),), dtype="float32")
    is_transition = np.asarray(is_transition)
    pred_transition = pred_in_component[edg_source] != pred_in_component[edg_target]
    comps, in_comp = connected_comp(pred_in_component.shape[0], edg_source, edg_target,
                                    (is_transition + pred_transition == 0).astype("uint8"), 0)
    tr = is_transition.nonzero()[0]
    cs, ct = in_comp[edg_source[tr]], in_comp[edg_target[tr]]
    sizes = [len(c) for c in comps]
    key = np.minimum(cs, ct).astype(np.int64) * len(comps) + np.maximum(cs, ct)
    _, first, count = np.unique(key, return_index=True, return_counts=True)
    for i in range(len(first)):
        c1, c2 = cs[first[i]], ct[first[i]]
        w = min(sizes[c1], sizes[c2]) / count[i] * transition_factor
        sel = tr[((cs == c1) * (ct == c2) + (ct == c1) * (cs == c2)) > 0]
        weights[sel] = weights[sel] + w
    return weights


def compute_weights_XPART_sorted(pred_in_component, edg_source, edg_target, is_transition, transition_factor):
    """The same weights without the per-pair loop (np.unique's inverse and counts), for sizes where the loop
    would take hours; equal to compute_weights_XPART bit for bit."""
    weights = np.ones((len(edg_source),), dtype="float32")
    is_transition = np.asarray(is_transition)
    in_comp, sizes = xpart_components(pred_in_component, edg_source, edg_target, is_transition)
    tr = is_transition.nonzero()[0]
    cs, ct = in_comp[edg_source[tr]].astype(np.int64), in_comp[edg_target[tr]].astype(np.int64)
    _, inv, count = np.unique(np.minimum(cs, ct) * len(sizes) + np.maximum(cs, ct), return_inverse=True,
                              return_counts=True)
    w = np.minimum(sizes[cs], sizes[ct]) / count[inv] * transition_factor
    weights[tr] = weights[tr] + w
    return weights


def xpart_components(pred_in_component, edg_source, edg_target, is_transition):
    """(in_component_x, component sizes) of the crosspartition components."""
    pred_transition = pred_in_component[edg_source] != pred_in_component[edg_target]
    comps, in_comp = connected_comp(pred_in_component.shape[0], edg_source, edg_target,
                                    (np.asarray(is_transition) + pred_transition == 0).astype("uint8"), 0)
    return in_comp, np.array([len(c) for c in comps], dtype=np.int64)


def compute_weight_loss(args, objects, edg_source, edg_target, is_transition, partition):
    """compute_weight_loss (losses.py:91-117) with the partition given, float32 numpy out."""
    pred_components, pred_in_component = partition
    is_transition = np.asarray(is_transition)
    if args.loss_weight == "none":
        return np.ones_like(edg_target).astype("f4")
    if args.loss_weight == "proportional":
        n, n_tr = len(is_transition), int(is_transition.sum())
        w = np.float32(np.float32(float(n)) / np.float32((1 - is_transition).sum()))
        out = np.full(len(edg_target), w, dtype="f4")
        out[is_transition.nonzero()] = float(n) / float(n_tr) * args.transition_factor
        return out
    if args.loss_weight == "seal":
        return compute_weights_SEAL(pred_components, pred_in_component, objects, edg_source, edg_target,
                                    is_transition, args.transition_factor)
    if args.loss_weight == "crosspartition":
        return compute_weights_XPART(pred_components, pred_in_component, objects, edg_source, edg_target,
                                     is_transition, args.transition_factor * 2 * args.k_nn_adj)
    raise ValueError(" %s is an unknown argument of parameter --loss" % (args.loss_weight))


def partition_edge_weight(args, diff):
    """Cut pursuit's edge weights (losses.py:68-72)."""
    diff = torch.as_tensor(diff).float()
    w = np.ones(diff.shape[0], dtype="f4")
    if args.edge_weight_threshold > 0:
        w[(diff > 1).numpy()] = args.edge_weight_threshold
    if args.edge_weight_threshold < 0:
        w = torch.exp(diff * args.edge_weight_threshold).numpy() / np.exp(args.edge_weight_threshold)
    return w


def relax_edge_binary(edg_binary, edg_source, edg_target, n_ver, tolerance):
    """What the reference computes: its first relaxation line indexes with the uint8 vertex marks themselves,
    so it sets edges 0 and/or 1; only the target line relaxes the edges at marked vertices."""
    relaxed = (edg_binary.cpu().numpy() if torch.is_tensor(edg_binary) else np.asarray(edg_binary)).copy()
    mark = np.zeros((n_ver,), dtype="uint8")
    for _ in range(tolerance):
        on = relaxed.nonzero()
        mark[edg_source[on]] = 1
        mark[edg_target[on]] = 1
        relaxed[mark[edg_source]] = True
        relaxed[mark[edg_target] > 0] = True
    return relaxed


def boundary_counts(truth, pred):
    """(numerator, denominator) of 100 * ((truth == pred) * truth).sum() / truth.sum()."""
    truth, pred = np.asarray(truth), np.asarray(pred)
    return int(((truth == pred) * truth).sum()), int(truth.sum())


def perfect_prediction(components, labels):
    full = np.zeros((labels.shape[0],), dtype="uint32")
    for c in components:
        full[c] = labels[c, 1:].sum(0).argmax()
    return full
