"""float64 numpy restatement of the device cut pursuit (superpoint_graph_b200/csrc/cut_pursuit.cu), which restates
libcp.cutpursuit at speed 4 (ref: partition/cut-pursuit/include/CutPursuit.h, CutPursuit_L2.h, CutPursuit_SPG.h).
Test infrastructure only.  It takes the same Philox4x32-10 draws, the same ascending member order and the same
2^k fixed-point capacities, and colours by the two residual reachabilities of a maximum flow from a plain Dinic.
"""
from collections import deque

import numpy as np

FLOW_STEPS, KMEANS_ITE, KMEANS_RESAMPLING, MAX_ITE_MAIN, STOPPING_RATIO, CUTOFF_ROUNDS = 3, 5, 10, 15, 0.05, 50
CAP_MAX = 1 << 61
SOURCE, FREE, SINK = 0, 1, 4

_M = 0xFFFFFFFF


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on Python ints; returns the four output words."""
    for r in range(10):
        if r:
            k0 = (k0 + 0x9E3779B9) & _M
            k1 = (k1 + 0xBB67AE85) & _M
        p0 = 0xD2511F53 * c0
        p1 = 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _M, p1 & _M, ((p0 >> 32) ^ c3 ^ k1) & _M, p0 & _M
    return c0, c1, c2, c3


def unary_weights(weight_decay):
    wd = np.float32(weight_decay)
    u = np.float32(np.power(wd, np.float32(-FLOW_STEPS)))
    out = []
    for _ in range(FLOW_STEPS):
        u = np.float32(u * wd)
        out.append(u)
    return out


# ------------------------------------------------------------------------------------------------ max flow
def shift(tmax, n):
    b = float(tmax) * float(n)
    if b == 0.0:
        return 40
    return min(40, 61 - int(np.frexp(b)[1]))


def fix(c, k):
    q = np.rint(np.ldexp(np.asarray(c, np.float64), k))
    return np.where(q >= CAP_MAX, CAP_MAX, q).astype(np.int64)


def max_flow(n, eu, ev, ecap, cs, ct):
    """Dinic on integer capacities: vertices 0..n-1, source n, sink n + 1; every listed edge is an arc pair with
    capacity ecap both ways.  Returns (flow value, residual capacities per arc, arc tails, arc heads, arc
    reverse)."""
    s, t = n, n + 1
    tails, heads, caps = [], [], []

    def add(u, v, cu, cv):
        tails.extend((u, v))
        heads.extend((v, u))
        caps.extend((int(cu), int(cv)))

    for e in range(len(eu)):
        add(int(eu[e]), int(ev[e]), ecap[e], ecap[e])
    for v in range(n):
        if cs[v] > 0:
            add(s, v, cs[v], 0)
        if ct[v] > 0:
            add(v, t, ct[v], 0)
    m = len(tails)
    adj = [[] for _ in range(n + 2)]
    for a in range(m):
        adj[tails[a]].append(a)
    res = caps[:]
    flow = 0
    while True:
        level = [-1] * (n + 2)
        level[s] = 0
        q = deque([s])
        while q:
            x = q.popleft()
            for a in adj[x]:
                y = heads[a]
                if res[a] > 0 and level[y] < 0:
                    level[y] = level[x] + 1
                    q.append(y)
        if level[t] < 0:
            break
        it = [0] * (n + 2)

        while True:
            f = _iterative_dfs(s, t, adj, heads, res, level, it)
            if f == 0:
                break
            flow += f
    return flow, np.array(res, dtype=object), np.array(tails), np.array(heads), np.array(caps, dtype=object)


def _iterative_dfs(s, t, adj, heads, res, level, it):
    """One augmenting path of the level graph (an explicit stack; Python recursion is too shallow)."""
    path = []
    x = s
    while True:
        if x == t:
            f = min(res[a] for a in path)
            for a in path:
                res[a] -= f
                res[a ^ 1] += f
            return f
        advanced = False
        while it[x] < len(adj[x]):
            a = adj[x][it[x]]
            y = heads[a]
            if res[a] > 0 and level[y] == level[x] + 1:
                path.append(a)
                x = y
                advanced = True
                break
            it[x] += 1
        if advanced:
            continue
        if not path:
            return 0
        level[x] = -1  # dead end
        a = path.pop()
        x = heads[a ^ 1]
        it[x] += 1


def residual_reach(n, res, tails, heads, start, forward):
    """Vertices reachable from `start` (forward) or reaching it (backward) along arcs of positive residual."""
    adj = [[] for _ in range(n + 2)]
    for a in range(len(tails)):
        if res[a] > 0:
            if forward:
                adj[tails[a]].append(heads[a])
            else:
                adj[heads[a]].append(tails[a])
    seen = np.zeros(n + 2, bool)
    seen[start] = True
    q = deque([start])
    while q:
        x = q.popleft()
        for y in adj[x]:
            if not seen[y]:
                seen[y] = True
                q.append(y)
    return seen[:n]


def colour(n, eu, ev, ecap_f32, cs_f32, ct_f32):
    """Boykov-Kolmogorov's colouring from any maximum flow: SINK where the sink is reachable in the residual
    graph, SOURCE where the vertex is reachable from the source, FREE elsewhere (2^k fixed point, cut_pursuit.cu)."""
    tmax = max(float(np.max(cs_f32, initial=0)), float(np.max(ct_f32, initial=0)))
    k = shift(np.float32(tmax), n)
    _, res, tails, heads, _ = max_flow(n, eu, ev, fix(ecap_f32, k), fix(cs_f32, k), fix(ct_f32, k))
    sink = residual_reach(n, res, tails, heads, n + 1, False)
    src = residual_reach(n, res, tails, heads, n, True)
    return np.where(sink, SINK, np.where(src, SOURCE, FREE)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ stages
def members_of(comp, n_comp):
    order = np.argsort(comp, kind="stable")
    offsets = np.searchsorted(comp[order], np.arange(n_comp + 1))
    return order, offsets


def kmeans(obs, members, offsets, sat, root, iteration, seed, margins=None):
    """init_labels with Philox draws (cut_pursuit.cu cp_kmeans_kernel); returns the labels (uint8 [n]).  margins
    (float64 [n], optional) receives |d0 - d1| / (d0 + d1) of the last assignment of the restart whose labels were
    kept, the relative decision margin of each vertex (inf where no restart was kept)."""
    if margins is not None:
        margins[:] = np.inf
    label = np.zeros(obs.shape[0], np.uint8)
    x64 = obs.astype(np.float64)
    for c in range(len(offsets) - 1):
        mem = members[offsets[c]:offsets[c + 1]]
        size = len(mem)
        if size <= 1 or sat[c]:
            continue
        X = x64[mem]
        for r in range(KMEANS_RESAMPLING):
            w = philox4x32_10(iteration & _M, int(root[c]) & _M, r, 0, seed & _M, (seed >> 32) & _M)
            first = w[0] % size
            u1 = w[1] * (1.0 / 4294967296.0)
            k0 = X[first].copy()
            e = ((X - k0) ** 2).sum(1)
            e0 = e.sum()
            hit = np.flatnonzero(np.cumsum(e) > e0 * u1)
            second = int(hit[0]) if len(hit) else 0
            k1 = X[second].copy()
            for _ in range(KMEANS_ITE):
                d0, d1 = ((X - k0) ** 2).sum(1), ((X - k1) ** 2).sum(1)
                plab = d0 > d1
                n0 = int(plab.sum())
                n1 = size - n0
                s0, s1 = X[plab].sum(0), X[~plab].sum(0)
                if n0 == 0 or n1 == 0:
                    k0, k1 = s0, s1
                    break
                k0, k1 = s0 / n0, s1 / n1
            en = np.where(plab[:, None], (X - k0) ** 2, (X - k1) ** 2).sum()
            if en < e0:
                label[mem] = plab
                if margins is not None:
                    with np.errstate(invalid="ignore", divide="ignore"):
                        margins[mem] = np.abs(d0 - d1) / (d0 + d1)
    return label


def centers(obs, members, offsets, sat, value, label, spatial):
    """compute_centers; returns (c0, c1) and saturates (L2) components with an empty side in place."""
    n_comp = len(offsets) - 1
    D = obs.shape[1]
    c0 = np.zeros((n_comp, D))
    c1 = np.zeros((n_comp, D))
    for c in range(n_comp):
        if sat[c]:
            continue
        mem = members[offsets[c]:offsets[c + 1]]
        X = obs[mem].astype(np.float64)
        lab = label[mem].astype(bool)
        if lab.all() or not lab.any():
            c0[c] = c1[c] = value[c]
            if not spatial:
                sat[c] = 1
        else:
            c0[c] = X[lab].sum(0) / lab.sum()
            c1[c] = X[~lab].sum(0) / (~lab).sum()
    return c0, c1


def capacities(obs, comp, sat, c0, c1, w, active, lam, unary, spatial):
    """set_capacities' fp32 formulas (cut_pursuit.cu cp_capacities_kernel)."""
    n, D = obs.shape
    cb_all = c0[comp].astype(np.float32)
    cn_all = c1[comp].astype(np.float32)
    cost_b = np.zeros(n, np.float32)
    cost_n = np.zeros(n, np.float32)
    for d in range(D):
        x = obs[:, d]
        cb, cn = cb_all[:, d], cn_all[:, d]
        tb = 0.5 * (cb.astype(np.float64) * cb.astype(np.float64) -
                    (np.float32(2) * (cb * x)).astype(np.float64))
        tn = 0.5 * (cn.astype(np.float64) * cn.astype(np.float64) -
                    (np.float32(2) * (cn * x)).astype(np.float64))
        cost_b = (cost_b.astype(np.float64) + tb).astype(np.float32)
        cost_n = (cost_n.astype(np.float64) + tn).astype(np.float32)
    pos = cost_b > cost_n
    cs = np.where(pos, cost_b - cost_n, np.float32(0)).astype(np.float32)
    ct = np.where(pos, np.float32(0), cost_n - cost_b).astype(np.float32)
    s = sat[comp].astype(bool)
    cs[s] = 0
    ct[s] = 0
    c = (w * np.float32(lam)).astype(np.float32)
    if spatial:
        c = (c / np.float32(unary)).astype(np.float32)
    ecap = np.where(active.astype(bool), np.float32(0), c).astype(np.float32)
    return cs, ct, ecap


def activate(colour_, comp, offsets, sat, eu, ev, active, spatial):
    """activate_edges; updates sat and active in place, returns the saturation (vertices in saturated
    components)."""
    n_comp = len(offsets) - 1
    if not spatial:
        nsink = np.bincount(comp[(colour_ == SINK) & ~sat[comp].astype(bool)], minlength=n_comp)
        size = np.diff(offsets)
        new = (~sat[:n_comp].astype(bool)) & ((nsink == 0) | (nsink == size))
        sat[:n_comp][new] = 1
    active[colour_[eu] != colour_[ev]] = 1
    return int(np.diff(offsets)[sat[:n_comp].astype(bool)].sum())


def split(comp, root, sat, eu, ev, active, n_comp):
    """compute_connected_components: pieces of the non-active graph inside unsaturated components; the piece
    holding a root keeps its component's index, the others are appended by smallest vertex.  Returns the new
    n_comp; comp, root, sat are updated in place (root and sat have room for n entries)."""
    n = comp.shape[0]
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    unsat = ~sat[comp].astype(bool)
    for e in np.flatnonzero(~active.astype(bool)):
        u, v = int(eu[e]), int(ev[e])
        if not (unsat[u] and unsat[v]):
            continue
        ru, rv = find(u), find(v)
        if ru != rv:
            parent[max(ru, rv)] = min(ru, rv)
    rep = np.array([find(v) for v in range(n)])
    pid = -np.ones(n, np.int64)
    for c in range(n_comp):
        if not sat[c]:
            pid[rep[root[c]]] = c
    new_roots = [v for v in range(n) if unsat[v] and rep[v] == v and pid[v] < 0]
    for i, v in enumerate(new_roots):
        pid[v] = n_comp + i
        root[n_comp + i] = v
        sat[n_comp + i] = 0
    comp[unsat] = pid[rep[unsat]]
    return n_comp + len(new_roots)


def comp_values(obs, members, offsets):
    n_comp = len(offsets) - 1
    D = obs.shape[1]
    value = np.zeros((n_comp, D))
    for c in range(n_comp):
        value[c] = obs[members[offsets[c]:offsets[c + 1]]].astype(np.float64).sum(0) / (offsets[c + 1] - offsets[c])
    return value


def merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, cutoff, is_cutoff, selected=None):
    """compute_reduced_graph + merge(is_cutoff); returns (value, n_merged, n_comp).  Candidates are taken by
    descending gain, ties by ascending (comp1, comp2)."""
    members, offsets = members_of(comp, n_comp)
    value = comp_values(obs, members, offsets)
    size = np.diff(offsets).astype(np.float64)
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
    for d in range(value.shape[1]):  # the device's order: dimensions in sequence, then the border term
        a1, a2 = v1[:, d], v2[:, d]
        mv = (w1 * a1 + w2 * a2) / (w1 + w2)
        gain = gain + 0.5 * (mv * mv * (w1 + w2) - a1 * a1 * w1 - a2 * a2 * w2)
    gain = gain + bw * np.float64(lam)
    gain = np.where(gain == 0, 0.0, gain)  # -0 and +0 are one gain
    cand = ((w1 <= cutoff) | (w2 <= cutoff)) if is_cutoff else gain > 0
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


def energy(obs, comp, value, w, active, lam):
    fid = 0.5 * ((obs.astype(np.float64) - value[comp]) ** 2).sum()
    return fid + float(lam) * w[active.astype(bool)].astype(np.float64).sum()


# ------------------------------------------------------------------------------------------------ driver
def cutpursuit(obs, source, target, edge_weight, reg_strength, cutoff=0, spatial=0, weight_decay=1.0, seed=0,
               stats=None):
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
    value = obs.astype(np.float64).sum(0, keepdims=True) / n
    old = energy(obs, comp, value, w, active, lam)
    ite = 0
    for ite in range(1, MAX_ITE_MAIN + 1):
        members, offsets = members_of(comp, n_comp)
        label = kmeans(obs, members, offsets, sat, root, ite, seed)
        for step in range(FLOW_STEPS):
            c0, c1 = centers(obs, members, offsets, sat, value, label, spatial)
            cs, ct, ecap = capacities(obs, comp, sat, c0, c1, w, active, lam, unary[step], spatial)
            col = colour(n, eu, ev, ecap, cs, ct)
            unsat = ~sat[comp].astype(bool)
            label[unsat] = col[unsat] == SINK
        saturation = activate(col, comp, offsets, sat, eu, ev, active, spatial)
        n_comp = split(comp, root, sat, eu, ev, active, n_comp)
        value, _, n_comp = merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, 0, False)
        e = energy(obs, comp, value, w, active, lam)
        if saturation == n:
            break
        with np.errstate(divide="ignore", invalid="ignore"):
            if np.float64(old - e) / np.float64(old) < STOPPING_RATIO:
                break
        old = e
    if cutoff > 0:
        i = 0
        while True:
            value, n_merged, n_comp = merge(obs, comp, root, sat, eu, ev, w, active, n_comp, lam, float(cutoff), True)
            i += 1
            if n_merged == 0 or i > CUTOFF_ROUNDS:
                break
    members, offsets = members_of(comp, n_comp)
    if stats is not None:
        stats.update(iterations=ite, components=n_comp, energy=energy(obs, comp, value, w, active, lam))
    return offsets, members, comp
