"""float64 numpy restatement of the device cut pursuit with vertex weights (superpoint_graph_b200/csrc/cut_pursuit.cu,
spg_cut_pursuit.cutpursuit2), which restates libcp.cutpursuit2 (ref: partition/cut-pursuit/src/cutpursuit.cpp:107-128;
CutPursuit_SPG.h, CutPursuit.h), and the Semantic3D label inpainting of
supervized_partition/graph_processing.py:150-165.
Test infrastructure only.

The stages that vertex weights change (k-means, centres, capacities, component values, merge, energy) are restated
here with node_weight (float32 [n]; None weighs every vertex 1 and computes exactly what oracle/cut_pursuit_ref.py
computes); the others (draws, max flow and colouring, activation, split) are cut_pursuit_ref's.  A vertex of weight 0
adds nothing to any sum and gets no terminal capacity; a component whose weights are all 0 has the value 0 / 0 = NaN,
its merge gains are NaN and never candidates, and the energy is then NaN.
"""
import numpy as np

from . import structure_ref
from .cut_pursuit_ref import (CUTOFF_ROUNDS, FLOW_STEPS, KMEANS_ITE, KMEANS_RESAMPLING, MAX_ITE_MAIN, SINK,
                              STOPPING_RATIO, _M, activate, colour, members_of, philox4x32_10, split, unary_weights)

def _mu(node_weight, n):
    return np.ones(n) if node_weight is None else np.asarray(node_weight, np.float32).astype(np.float64)



def kmeans(obs, members, offsets, sat, root, iteration, seed, margins=None, node_weight=None):
    """init_labels with Philox draws (cut_pursuit.cu cp_kmeans_kernel); returns the labels (uint8 [n]).  margins
    (float64 [n], optional) receives |d0 - d1| / (d0 + d1) of the last assignment of the restart whose labels were
    kept, the relative decision margin of each vertex (inf where no restart was kept)."""
    if margins is not None:
        margins[:] = np.inf
    label = np.zeros(obs.shape[0], np.uint8)
    x64 = obs.astype(np.float64)
    mu = _mu(node_weight, obs.shape[0])
    for c in range(len(offsets) - 1):
        mem = members[offsets[c]:offsets[c + 1]]
        size = len(mem)
        if size <= 1 or sat[c]:
            continue
        X = x64[mem]
        M = mu[mem]
        for r in range(KMEANS_RESAMPLING):
            w = philox4x32_10(iteration & _M, int(root[c]) & _M, r, 0, seed & _M, (seed >> 32) & _M)
            first = w[0] % size
            u1 = w[1] * (1.0 / 4294967296.0)
            k0 = X[first].copy()
            e = ((X - k0) ** 2).sum(1) * M  # CutPursuit_SPG.h:160-169: mu |x - k0|^2
            e0 = e.sum()
            hit = np.flatnonzero(np.cumsum(e) > e0 * u1)
            second = int(hit[0]) if len(hit) else 0
            k1 = X[second].copy()
            for _ in range(KMEANS_ITE):
                d0, d1 = ((X - k0) ** 2).sum(1), ((X - k1) ** 2).sum(1)
                plab = d0 > d1  # SPG.h:191-200: unweighted distances
                n0, n1 = M[plab].sum(), M[~plab].sum()  # SPG.h:202-244: sums of mu x and mu
                s0, s1 = (X[plab] * M[plab, None]).sum(0), (X[~plab] * M[~plab, None]).sum(0)
                if n0 == 0 or n1 == 0:  # SPG.h:236-239: break before dividing
                    k0, k1 = s0, s1
                    break
                k0, k1 = s0 / n0, s1 / n1
            en = (np.where(plab[:, None], (X - k0) ** 2, (X - k1) ** 2) * M[:, None]).sum()  # SPG.h:247-264
            if en < e0:
                label[mem] = plab
                if margins is not None:
                    with np.errstate(invalid="ignore", divide="ignore"):
                        margins[mem] = np.abs(d0 - d1) / (d0 + d1)
    return label


def centers(obs, members, offsets, sat, value, label, spatial, node_weight=None):
    """compute_centers; returns (c0, c1) and saturates (L2) components with a side of weight 0 in place."""
    n_comp = len(offsets) - 1
    D = obs.shape[1]
    mu = _mu(node_weight, obs.shape[0])
    c0 = np.zeros((n_comp, D))
    c1 = np.zeros((n_comp, D))
    for c in range(n_comp):
        if sat[c]:
            continue
        mem = members[offsets[c]:offsets[c + 1]]
        X = obs[mem].astype(np.float64)
        M = mu[mem]
        lab = label[mem].astype(bool)
        n0, n1 = M[lab].sum(), M[~lab].sum()  # CutPursuit_SPG.h:310-334
        if n0 == 0 or n1 == 0:  # SPG.h:335-344
            c0[c] = c1[c] = value[c]
            if not spatial:
                sat[c] = 1
        else:
            c0[c] = (X[lab] * M[lab, None]).sum(0) / n0
            c1[c] = (X[~lab] * M[~lab, None]).sum(0) / n1
    return c0, c1


def capacities(obs, comp, sat, c0, c1, w, active, lam, unary, spatial, node_weight=None):
    """set_capacities' fp32 formulas (cut_pursuit.cu cp_capacities_kernel)."""
    n, D = obs.shape
    hm = 0.5 * _mu(node_weight, n)  # CutPursuit_SPG.h:396-401: 0.5 mu (c c - 2 c x)
    cb_all = c0[comp].astype(np.float32)
    cn_all = c1[comp].astype(np.float32)
    cost_b = np.zeros(n, np.float32)
    cost_n = np.zeros(n, np.float32)
    for d in range(D):
        x = obs[:, d]
        cb, cn = cb_all[:, d], cn_all[:, d]
        with np.errstate(invalid="ignore"):  # a NaN centre meets only weight-0 vertices, zeroed below
            tb = hm * (cb.astype(np.float64) * cb.astype(np.float64) -
                       (np.float32(2) * (cb * x)).astype(np.float64))
            tn = hm * (cn.astype(np.float64) * cn.astype(np.float64) -
                       (np.float32(2) * (cn * x)).astype(np.float64))
        cost_b = (cost_b.astype(np.float64) + tb).astype(np.float32)
        cost_n = (cost_n.astype(np.float64) + tn).astype(np.float32)
    pos = cost_b > cost_n
    cs = np.where(pos, cost_b - cost_n, np.float32(0)).astype(np.float32)
    ct = np.where(pos, np.float32(0), cost_n - cost_b).astype(np.float32)
    s = sat[comp].astype(bool) | (hm == 0)  # SPG.h:388-393: no observation, no cut
    cs[s] = 0
    ct[s] = 0
    c = (w * np.float32(lam)).astype(np.float32)
    if spatial:
        c = (c / np.float32(unary)).astype(np.float32)
    ecap = np.where(active.astype(bool), np.float32(0), c).astype(np.float32)
    return cs, ct, ecap



def comp_weights(members, offsets, node_weight=None):
    """The component weights sum mu (CutPursuit_SPG.h:449): the sizes when node_weight is None."""
    if node_weight is None:
        return np.diff(offsets).astype(np.float64)
    mu = _mu(node_weight, len(members))
    return np.array([mu[members[offsets[c]:offsets[c + 1]]].sum() for c in range(len(offsets) - 1)])


def comp_values(obs, members, offsets, node_weight=None):
    """compute_value (CutPursuit_SPG.h:439-468): sum mu x / sum mu, NaN where every weight is 0."""
    n_comp = len(offsets) - 1
    D = obs.shape[1]
    value = np.zeros((n_comp, D))
    mu = _mu(node_weight, obs.shape[0])
    wc = comp_weights(members, offsets, node_weight)
    for c in range(n_comp):
        mem = members[offsets[c]:offsets[c + 1]]
        with np.errstate(invalid="ignore"):
            value[c] = (obs[mem].astype(np.float64) * mu[mem, None]).sum(0) / wc[c]
    return value


def merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, cutoff, is_cutoff, selected=None, node_weight=None):
    """compute_reduced_graph + merge(is_cutoff); returns (value, n_merged, n_comp).  Candidates are taken by
    descending gain, ties by ascending (comp1, comp2); the component weights (CutPursuit.h:473-478, 578-619) are
    sum mu, and a NaN gain (a NaN-valued component) is never a candidate."""
    members, offsets = members_of(comp, n_comp)
    value = comp_values(obs, members, offsets, node_weight)
    size = comp_weights(members, offsets, node_weight)
    a, b = comp[eu], comp[ev]
    cross = a != b
    lo, hi = np.minimum(a, b)[cross], np.maximum(a, b)[cross]
    keys, inv = np.unique(lo.astype(np.int64) * (1 << 32) + hi, return_inverse=True)
    bw = np.zeros(len(keys))
    np.add.at(bw, inv, w[cross].astype(np.float64))
    c1, c2 = keys >> 32, keys & 0xFFFFFFFF
    w1, w2 = size[c1], size[c2]
    v1, v2 = value[c1], value[c2]
    gain = np.zeros(len(keys))
    with np.errstate(invalid="ignore"):
        for d in range(value.shape[1]):  # the device's order: dimensions in sequence, then the border term
            a1, a2 = v1[:, d], v2[:, d]
            mv = (w1 * a1 + w2 * a2) / (w1 + w2)
            gain = gain + 0.5 * (mv * mv * (w1 + w2) - a1 * a1 * w1 - a2 * a2 * w2)
    gain = gain + bw * np.float64(lam)
    gain = np.where(gain == 0, 0.0, gain)  # -0 and +0 are one gain
    cand = ((w1 <= cutoff) | (w2 <= cutoff)) & ~np.isnan(gain) if is_cutoff else gain > 0
    idx = np.flatnonzero(cand)
    idx = idx[np.argsort(-gain[idx], kind="stable")]
    partner = -np.ones(n_comp, np.int64)
    for i in idx:
        x, y = int(c1[i]), int(c2[i])
        if partner[x] >= 0 or partner[y] >= 0:
            continue
        partner[x], partner[y] = y, x
    n_merged = int((partner >= 0).sum() // 2)
    if selected is not None:
        selected.extend((x, int(partner[x])) for x in range(n_comp) if partner[x] > x)
    for x in range(n_comp):
        y = partner[x]
        if y > x:
            value[x] = (size[x] * value[x] + size[y] * value[y]) / (size[x] + size[y])
            sat[x] = 0
    pa, pb = comp[eu], comp[ev]
    active[(pa != pb) & (partner[pa] == pb)] = 0
    keep = ~((partner >= 0) & (partner < np.arange(n_comp)))
    newid = np.cumsum(keep) - 1
    target = np.where(keep, np.arange(n_comp), partner)
    m = int(keep.sum())
    root[:m] = root[:n_comp][keep]
    sat[:m] = sat[:n_comp][keep]
    comp[:] = newid[target[comp]]
    return value[keep], n_merged, m


def energy(obs, comp, value, w, active, lam, node_weight=None):
    """compute_energy (CutPursuit_SPG.h:25-34): sum 0.5 mu (x - v)^2 + lambda sum of the active edges' weights."""
    fid = 0.5 * (((obs.astype(np.float64) - value[comp]) ** 2) * _mu(node_weight, len(comp))[:, None]).sum()
    return fid + float(lam) * w[active.astype(bool)].astype(np.float64).sum()


# ------------------------------------------------------------------------------------------------ driver
def cutpursuit(obs, source, target, edge_weight, reg_strength, cutoff=0, spatial=0, weight_decay=1.0, seed=0,
               stats=None, node_weight=None):
    """(offsets, members, in_component) and the final energy, as the device computes them."""
    obs = np.ascontiguousarray(obs, np.float32)
    eu = np.asarray(source, np.int64).reshape(-1)
    ev = np.asarray(target, np.int64).reshape(-1)
    w = np.asarray(edge_weight, np.float32).reshape(-1)
    n = obs.shape[0]
    lam = np.float32(reg_strength)
    unary = unary_weights(weight_decay) if spatial else [np.float32(1)] * FLOW_STEPS
    comp = np.zeros(n, np.int64)
    root = np.zeros(n, np.int64)
    sat = np.zeros(n, np.uint8)
    active = np.zeros(len(eu), np.uint8)
    n_comp = 1
    nw = node_weight
    if nw is None:
        value = obs.astype(np.float64).sum(0, keepdims=True) / n
    else:
        value = comp_values(obs, np.arange(n), np.array([0, n]), nw)
    old = energy(obs, comp, value, w, active, lam, nw)
    ite = 0
    for ite in range(1, MAX_ITE_MAIN + 1):
        members, offsets = members_of(comp, n_comp)
        label = kmeans(obs, members, offsets, sat, root, ite, seed, node_weight=nw)
        for step in range(FLOW_STEPS):
            c0, c1 = centers(obs, members, offsets, sat, value, label, spatial, nw)
            cs, ct, ecap = capacities(obs, comp, sat, c0, c1, w, active, lam, unary[step], spatial, nw)
            col = colour(n, eu, ev, ecap, cs, ct)
            unsat = ~sat[comp].astype(bool)
            label[unsat] = col[unsat] == SINK
        saturation = activate(col, comp, offsets, sat, eu, ev, active, spatial)
        n_comp = split(comp, root, sat, eu, ev, active, n_comp)
        value, _, n_comp = merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, 0, False, node_weight=nw)
        e = energy(obs, comp, value, w, active, lam, nw)
        if saturation == n:
            break
        with np.errstate(divide="ignore", invalid="ignore"):
            if np.float64(old - e) / np.float64(old) < STOPPING_RATIO:
                break
        old = e
    if cutoff > 0:
        i = 0
        while True:
            value, n_merged, n_comp = merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, float(cutoff), True,
                                            node_weight=nw)
            i += 1
            if n_merged == 0 or i > CUTOFF_ROUNDS:
                break
    members, offsets = members_of(comp, n_comp)
    if stats is not None:
        stats.update(iterations=ite, components=n_comp, energy=energy(obs, comp, value, w, active, lam, nw))
    return offsets, members, comp


def cutpursuit2(obs, source, target, edge_weight, node_weight, reg_strength, seed=0, stats=None):
    """libcp.cutpursuit2 (cutpursuit.cpp:107-128): CutPursuit_SPG with the vertex weights node_weight, cutoff 0,
    weight_decay 1 (unary weights 1); (offsets, members, in_component) as the device computes them."""
    return cutpursuit(obs, source, target, edge_weight, reg_strength, cutoff=0, spatial=1, weight_decay=1.0, seed=seed,
                      stats=stats, node_weight=node_weight)


# ------------------------------------------------------------------------------------------------ inpainting
def inpaint_objects(labels, source, target, seed=0):
    """graph_processing.py:150-165: the objects libcp.cutpursuit2 makes of the hard labels (this oracle's
    cutpursuit2 with the device's k-means draws under `seed`), in_component int64 [n]."""
    hard, s, t, edge_weight, node_weight = structure_ref.inpainting_problem(labels, source, target)
    obs = hard.reshape(-1, 1).astype("f4")
    return cutpursuit2(obs, s, t, edge_weight, node_weight, 0.01, seed=seed)[2]


def inpainted_structure(xyz, labels, neighbors, k_nn_adj, k_nn_local, voronoi=0.0, simplices=None, plane=None,
                        seed=0):
    """structure_ref.structure for sema3d with labels, its objects inpainted (inpaint_objects over the structure's
    edges) and is_transition = objects[source] != objects[target] over every edge (:165)."""
    n = np.asarray(xyz).shape[0]
    g = structure_ref.structure("sema3d", xyz, labels, np.zeros(n, np.int64), neighbors, k_nn_adj, k_nn_local,
                                voronoi, simplices, True, plane)
    objects = inpaint_objects(labels, g["source"], g["target"], seed)
    return structure_ref.structure("sema3d", xyz, labels, objects, neighbors, k_nn_adj, k_nn_local, voronoi,
                                   simplices, True, plane)
