"""Numpy restatement of the superpoint graph batch's device draws (superpoint_graph_b200/csrc/batch_rng.cu,
spg_loader.load_batch(device_rng=True)) and of the batch built from them.  Test infrastructure only.

Counter layout (Philox4x32-10, key = (seed lo, seed hi)).  The 64-bit draw k of stream (a, b, purpose) is
Philox(c0 = k >> 1, c1 = a, c2 = b, c3 = purpose), words (2(k & 1), 2(k & 1) + 1) as (low, high).  Purposes:
1 permutation, 2 centres, 3 resample, 4 augmentation, 5 jitter.
  graph draws        (a, b) = (0, graph position); draw v is the sort key of vertex (new id) v
  training clouds    (a, b) = (superpoint id, graph position); resample draw j for output point j; augmentation
                     draws 0 scale, 1 angle, 2 mirror x, 3 mirror y; jitter element k = j F + f takes draws 2k, 2k + 1
  evaluation clouds  (a, b) = (low, high word of id + test_seed_offset), purpose 3 | 0x100
Distributions (learning/spg.py): random.shuffle (:135-137) -> ranks of a stable sort of the permutation keys;
random.sample(range(n), nneigh) (:117) -> the nneigh smallest keys of the centre stream; rs.choice(n, L) (:209-214)
-> the high word of draw * n, the original points first when n < L; augment_cloud (:240-253) -> u53 = (x >> 11)
2^-53, s = 1/a + (a - 1/a) u, angle 2 pi u, mirror when u < p / 2, composed as augment_matrix; jitter (:255-257)
-> float32(clip(0.01 g, +-0.05)) with g = sqrt(-2 log(1 - u53)) cos(2 pi u53) in float64.
"""
import numpy as np

from oracle import loader_ref
from oracle import spg_batch_ref as sref

PERM, CENTRES, RESAMPLE, AUGMENT, JITTER, EVAL = 1, 2, 3, 4, 5, 0x100
_M = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays (broadcast) of 32-bit words held in uint64; returns the four output words."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0) & _M, np.uint64(k1) & _M
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _M
            k1 = (k1 + np.uint64(0xBB67AE85)) & _M
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0), p1 & _M, ((p0 >> np.uint64(32)) ^ c3 ^ k1), p0 & _M
    return c0, c1, c2, c3


def draw64(seed, a, b, purpose, k):
    """The 64-bit draws k (array) of stream (a, b, purpose) under `seed`, as uint64."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    k = np.asarray(k, dtype=np.uint64)
    w = philox(k >> np.uint64(1), a, b, purpose, seed & 0xFFFFFFFF, seed >> 32)
    odd = (k & np.uint64(1)).astype(bool)
    lo, hi = np.where(odd, w[2], w[0]), np.where(odd, w[3], w[1])
    return (hi << np.uint64(32)) | lo


def u53(x):
    return (np.asarray(x, dtype=np.uint64) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def below(x, n):
    """floor(x n / 2^64): the high word of the 128-bit product, for n < 2^32."""
    x, n = np.asarray(x, dtype=np.uint64), np.uint64(n)
    return (((x >> np.uint64(32)) * n + (((x & _M) * n) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def graph_draws(n, seed, graph_pos, train, hardcutoff, nneigh):
    """(perm or None, centres or None, cut) of the graph at `graph_pos`: perm[i] = new id of vertex i (0 < hardcutoff
    < n), centres = new ids (0 < nneigh < n), cut as graph_draws of spg_loader."""
    if not train:
        return None, None, 0
    perm = centres = None
    v = np.arange(n)
    if 0 < hardcutoff < n:
        order = np.argsort(draw64(seed, 0, graph_pos, PERM, v), kind="stable")
        perm = np.empty(n, np.int64)
        perm[order] = v
    if 0 < nneigh < n:
        centres = np.argsort(draw64(seed, 0, graph_pos, CENTRES, v), kind="stable")[:nneigh]
    return perm, centres, max(hardcutoff, 0)


def _stream(sp_id, graph_pos, train, test_seed_offset):
    if train:
        return int(sp_id), int(graph_pos), RESAMPLE
    e = (int(sp_id) + int(test_seed_offset)) & 0xFFFFFFFFFFFFFFFF
    return e & 0xFFFFFFFF, e >> 32, RESAMPLE | EVAL


def sample_indices(seed, sp_id, graph_pos, n, L, train, test_seed_offset=0):
    a, b, p = _stream(sp_id, graph_pos, train, test_seed_offset)
    j = np.arange(L)
    drawn = below(draw64(seed, a, b, p, j), n)
    return np.where((n > L) | (j >= n), drawn, j).astype(np.int64)


def augment_uniforms(seed, sp_id, graph_pos):
    """(scale u, angle u, mirror x u, mirror y u) of a training cloud."""
    return u53(draw64(seed, int(sp_id), int(graph_pos), AUGMENT, np.arange(4)))


def augment_matrix(seed, sp_id, graph_pos, scale, rot, mirror_prob):
    """augment_matrix (spg.py:240-253) on the device's uniforms, composed by np.dot in the same order."""
    u = augment_uniforms(seed, sp_id, graph_pos)
    M = np.eye(3)
    if scale > 1:
        M = np.dot(np.eye(3) * (1 / scale + (scale - 1 / scale) * u[0]), M)
    if rot == 1:
        angle = 2 * np.pi * u[1]
        c, s = np.cos(angle), np.sin(angle)
        M = np.dot(np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]), M)
    if mirror_prob > 0:
        if u[2] < mirror_prob / 2:
            M = np.dot(np.diag([-1.0, 1.0, 1.0]), M)
        if u[3] < mirror_prob / 2:
            M = np.dot(np.diag([1.0, -1.0, 1.0]), M)
    return M


def jitter(seed, sp_id, graph_pos, L, F):
    """[L, F] float32: clip(0.01 g, +-0.05) (spg.py:255-257)."""
    k = np.arange(L * F, dtype=np.uint64)
    u1 = 1.0 - u53(draw64(seed, int(sp_id), int(graph_pos), JITTER, 2 * k))
    u2 = u53(draw64(seed, int(sp_id), int(graph_pos), JITTER, 2 * k + 1))
    g = np.sqrt(-2.0 * np.log(u1)) * np.cos(2 * np.pi * u2)
    return np.clip(0.01 * g, -0.05, 0.05).astype(np.float32).reshape(L, F)


def build_batch(graphs, parsed, train, args, seed, test_seed_offset=0):
    """The device_rng batch from the draws above.  graphs: per position (name, n, edges [E, 2], s [n], targets rows
    [n, T], edge features [E, F]); parsed: {name: {sp_id: [n_pts, C] float32}}.  Returns (targets, idxn, degs,
    edgefeats, edge_index, clouds_meta, clouds_flag, clouds [Nv, F, L], clouds_global [Nv], draws) with the edges in
    the stable-order collate; draws = per cloud (sample indices, matrix or None, jitter or None).  Raises as
    load_batch does."""
    hc, nn = (int(args.spg_augm_hardcutoff), int(args.spg_augm_nneigh)) if train else (0, 0)
    order = int(args.spg_augm_order) if train else 0
    L = int(args.ptn_npts)
    cols = loader_ref.attrib_columns(args.pc_attribs)
    picks = []
    for b, (name, n, edges, s, targets, feats) in enumerate(graphs):
        perm, centres, cut = graph_draws(n, seed, b, train, hc, nn)
        ids, sub, sel = sref.sample_graph(n, edges, s, perm, centres, order, int(args.ptn_minpts), cut)
        if sub.shape[0] and any(int(i) not in parsed[name] for i in ids):
            raise KeyError(name)
        picks.append((name, b, ids, sub, sel, targets, feats))
    kept = [p for p in picks if p[3].shape[0]]
    if not kept:
        raise RuntimeError("no graph has an edge")
    if not picks[0][3].shape[0]:
        raise TypeError("the first graph has no edge")
    meta, flags, clouds, diam, draws, cg = [], [], [], [], [], []
    for name, b, ids, sub, sel, targets, feats in kept:
        n_valid = 0
        for i in ids.tolist():
            meta.append("%s.%d" % (name, i))
            P = parsed[name][i]
            if P.shape[0] < args.ptn_minpts:
                flags.append(-1)
                continue
            flags.append(0)
            n_valid += 1
            ii = sample_indices(seed, i, b, P.shape[0], L, train, test_seed_offset)
            M = noise = None
            if train:
                M = augment_matrix(seed, i, b, args.pc_augm_scale, args.pc_augm_rot, args.pc_augm_mirror_prob)
                if args.pc_augm_jitter:
                    noise = jitter(seed, i, b, L, len(cols) if cols is not None else P.shape[1])
            cloud, d = loader_ref.load_superpoint(P, ii, args.pc_attribs, args.pc_xyznormalize, M, noise)
            clouds.append(cloud)
            diam.append(d)
            draws.append((ii, M, noise))
        if n_valid == 0:
            raise TypeError("a graph with edges has no cloud")
        cg.append((targets[ids], sub, feats[sel]))
    targets, idxn, degs, edgefeats, edge_index = sref.collate(cg, kind="stable")
    return (targets, idxn, degs, edgefeats, edge_index, meta, np.array(flags, np.int64),
            loader_ref.stack_clouds(clouds), np.concatenate(diam), draws)
