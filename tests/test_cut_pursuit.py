"""The device cut pursuit (superpoint_graph_b200/spg_cut_pursuit.py, csrc/cut_pursuit.cu) against its float64
restatement (oracle/cut_pursuit_ref.py).

CPU: the oracle on hand-worked cases; the oracle's max flow by certificate and its colouring by brute force; host
validation; the ABI symbols and kernel names.
GPU: end to end on piecewise-constant signals (the ground truth, the oracle's in_component bit for bit, the energy),
in both modes, with and without cutoff; a 5000-vertex cloud whose first component takes the 512-thread path (energy,
component count, connectivity, the cutoff invariant, output invariants); per stage from the same state: k-means
labels (margin rule), centres, capacities, the colouring (up to a 10^4-vertex strip of hundreds of BFS levels, with
the device's own preflow checked by certificate), split numbering and merge selection (ties included); bitwise
reproducibility; prune -> k-NN -> geof -> cut pursuit -> superpoint graph on device tensors; compute_weight_loss.
"""
import itertools
import types

import numpy as np
import pytest
import torch

from oracle import cut_pursuit_ref as R


def _grid(H=16, W=16, noise=0.01, seed=0):
    rng = np.random.default_rng(seed)
    xy = np.stack(np.meshgrid(np.arange(H), np.arange(W), indexing="ij"), -1).reshape(-1, 2)
    truth = (xy[:, 0] >= H // 2).astype(np.int64) + 2 * (xy[:, 1] >= W // 3)
    obs = (truth[:, None] * np.array([1.0, 2.0, -1.0]) + rng.normal(0, noise, (H * W, 3))).astype(np.float32)
    idx = np.arange(H * W).reshape(H, W)
    src = np.concatenate([idx[:-1].ravel(), idx[:, :-1].ravel()])
    tgt = np.concatenate([idx[1:].ravel(), idx[:, 1:].ravel()])
    return obs, src, tgt, np.ones(len(src), np.float32), truth


def _knn(n=600, k=5, pieces=3, noise=0.01, seed=1):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    truth = np.minimum((xyz[:, 0] * pieces).astype(np.int64), pieces - 1)
    obs = (truth[:, None] * np.array([1.0, -0.5]) + rng.normal(0, noise, (n, 2))).astype(np.float32)
    d = ((xyz[:, None] - xyz[None]) ** 2).sum(-1)
    nn = np.argsort(d, 1)[:, 1:k + 1]
    src = np.repeat(np.arange(n), k)
    tgt = nn.ravel()
    return obs, src, tgt, np.ones(len(src), np.float32), truth


def _same_partition(a, b):
    return len(np.unique(a)) == len(np.unique(b)) == len(np.unique(a * (b.max() + 1) + b))


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_three_vertex_chain():
    obs = np.array([[10.0, 20.0], [0.0, 1.0], [0.0, 0.0]], np.float32)
    off, mem, comp = R.cutpursuit(obs, [0, 1], [1, 2], np.ones(2, np.float32), 1)
    assert comp.tolist() == [0, 1, 1]
    assert off.tolist() == [0, 1, 3] and mem.tolist() == [0, 1, 2]


@pytest.mark.parametrize("spatial", [0, 1])
def test_oracle_recovers_pieces(spatial):
    obs, src, tgt, w, truth = _grid()
    _, _, comp = R.cutpursuit(obs, src, tgt, w, 0.05, spatial=spatial, weight_decay=0.7)
    assert _same_partition(comp, truth)


def test_oracle_huge_lambda_gives_one_component():
    obs, src, tgt, w, _ = _grid(8, 8)
    off, _, comp = R.cutpursuit(obs, src, tgt, w, 1e6)
    assert len(off) == 2 and (comp == 0).all()


def test_oracle_cutoff_merges_small_components():
    obs, src, tgt, w, truth = _grid(12, 12)
    obs[5] += 50.0  # a one-vertex outlier piece
    _, _, comp = R.cutpursuit(obs, src, tgt, w, 0.05)
    assert np.bincount(comp).min() == 1
    _, _, cut = R.cutpursuit(obs, src, tgt, w, 0.05, cutoff=3)
    assert np.bincount(cut).min() > 3


def _brute_colour(n, eu, ev, ecap, cs, ct):
    """Minimal source-side and minimal sink-side minimum cuts by enumeration of every cut."""
    k = R.shift(np.float32(max(cs.max(), ct.max())), n)
    qe, qs, qt = R.fix(ecap, k), R.fix(cs, k), R.fix(ct, k)
    best, cuts = None, []
    for bits in itertools.product([0, 1], repeat=n):
        S = np.array(bits, bool)  # True: source side
        v = int(qs[~S].sum()) + int(qt[S].sum())
        v += int(qe[S[eu] & ~S[ev]].sum()) + int(qe[S[ev] & ~S[eu]].sum())
        if best is None or v < best:
            best, cuts = v, [S]
        elif v == best:
            cuts.append(S)
    src_min = np.logical_and.reduce(cuts)
    sink_min = np.logical_and.reduce([~S for S in cuts])
    return np.where(sink_min, R.SINK, np.where(src_min, R.SOURCE, R.FREE)), best


@pytest.mark.parametrize("seed", range(6))
def test_oracle_max_flow_certificate_and_colouring(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(4, 12))
    m = int(rng.integers(n, 3 * n))
    eu, ev = rng.integers(0, n, m), rng.integers(0, n, m)
    keep = eu != ev
    eu, ev = eu[keep], ev[keep]
    ecap = rng.choice([0.0, 0.25, 0.5, 1.0], len(eu)).astype(np.float32)
    d = rng.choice([-1.0, -0.5, 0.0, 0.5, 1.0], n).astype(np.float32)
    cs, ct = np.maximum(d, 0).astype(np.float32), np.maximum(-d, 0).astype(np.float32)
    k = R.shift(np.float32(max(cs.max(), ct.max())), n)
    flow, res, tails, heads, caps = R.max_flow(n, eu, ev, R.fix(ecap, k), R.fix(cs, k), R.fix(ct, k))
    f = caps - res
    assert all(int(r) >= 0 for r in res)
    net = np.zeros(n + 2, dtype=object)
    for a in range(len(f)):
        if a % 2 == 0:
            net[tails[a]] -= f[a]
            net[heads[a]] += f[a]
    assert all(net[v] == 0 for v in range(n))
    assert int(net[n + 1]) == flow == -int(net[n])
    col = R.colour(n, eu, ev, ecap, cs, ct)
    want, best = _brute_colour(n, eu, ev, ecap, cs, ct)
    assert best == flow
    assert np.array_equal(col, want)


def test_validation_errors():
    pytest.importorskip("torch")
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs = np.zeros((3, 2), np.float32)
    e = np.array([0, 1])
    w = np.ones(2, np.float32)
    with pytest.raises(TypeError):
        cp.prepare(obs.astype(np.float64), e, e + 1, w, 1.0)
    with pytest.raises(TypeError):
        cp.prepare(obs, e.astype(np.float32), e + 1, w, 1.0)
    with pytest.raises(TypeError):
        cp.prepare(obs, e, e + 1, w.astype(np.float64), 1.0)
    with pytest.raises(ValueError):
        cp.prepare(np.zeros((3, 33), np.float32), e, e + 1, w, 1.0)
    with pytest.raises(ValueError):
        cp.prepare(np.zeros((3, 0), np.float32), e, e + 1, w, 1.0)
    with pytest.raises(ValueError):
        cp.prepare(obs, e, e + 1, w[:1], 1.0)
    with pytest.raises(ValueError):
        cp.prepare(obs, e, e + 1, w, 1.0, cutoff=-1)
    with pytest.raises(ValueError):
        cp.prepare(obs, e, e + 1, w, 1.0, spatial=2)
    with pytest.raises(ValueError):
        cp.prepare(obs, e, e + 1, w, 1.0, weight_decay=0)


def test_unary_weights_match_oracle():
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    assert [np.float32(u) for u in cp.unary_weights(0.7)] == R.unary_weights(0.7)


def test_abi_symbols_and_kernel_names():
    from superpoint_graph_b200 import _lib
    names = ["spg_cp_workspace", "spg_cp_regions", "spg_cp_setup", "spg_cp_members", "spg_cp_kmeans",
             "spg_cp_centers", "spg_cp_capacities", "spg_cp_maxflow", "spg_cp_activate", "spg_cp_split",
             "spg_cp_merge", "spg_cp_energy", "spg_cp_output"]
    protos = _lib.protos()
    lib = _lib.lib()
    for n in names:
        assert n in protos, n
        assert getattr(lib, n) is not None
    kn = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    for k in ("cp_graph", "cp_members", "cp_kmeans", "cp_centers", "cp_capacities", "cp_maxflow", "cp_colour",
              "cp_activate", "cp_split", "cp_merge", "cp_energy"):
        assert k in kn, k


# ------------------------------------------------------------------------------------------------- GPU
def _dev_run(obs, src, tgt, w, lam, **kw):
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    comps, inc = cp.cutpursuit(obs, src, tgt, w, lam, **kw)
    return comps, inc.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["grid", "knn"])
@pytest.mark.parametrize("spatial", [0, 1])
@pytest.mark.parametrize("cutoff", [0, 4])
def test_end_to_end_matches_oracle_bit_for_bit(case, spatial, cutoff):
    obs, src, tgt, w, truth = _grid() if case == "grid" else _knn()
    if cutoff:
        obs[7] += 40.0
    kw = dict(cutoff=cutoff, spatial=spatial, weight_decay=0.7)
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    st = cp.prepare(obs, src, tgt, w, 0.05, **kw)
    stats, ref = {}, {}
    with torch.cuda.device(st.dev):
        cp.run(st, 0.05, cutoff, spatial, 0.7, 0, stats=stats)
        comps, inc = st.output()
    inc = inc.cpu().numpy()
    off, mem, comp = R.cutpursuit(obs, src, tgt, w, 0.05, stats=ref, **kw)
    assert np.array_equal(inc, comp)
    assert abs(stats["energy"] - ref["energy"]) <= 1e-12 * abs(ref["energy"])
    assert np.array_equal(comps.offsets.cpu().numpy(), off)
    assert np.array_equal(comps.members.cpu().numpy(), mem)
    if not cutoff and case == "grid":
        assert _same_partition(inc, truth)


@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [0, 1])
def test_colouring_matches_oracle(spatial):
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    for n, seed in ((100, 0), (2000, 1)):
        obs, src, tgt, w, _ = _knn(n=n, k=5, pieces=4, noise=0.3, seed=seed)
        st = cp.prepare(obs, src, tgt, w, 0.05, spatial=spatial, weight_decay=0.7)
        st.members()
        st.kmeans(1, 0)
        st.centers(spatial)
        u = cp.unary_weights(0.7)[0] if spatial else 1.0
        st.capacities(np.float32(0.05), u, spatial)
        st.maxflow()
        cs = st.region("cs", torch.float32, n).cpu().numpy()
        ct = st.region("ct", torch.float32, n).cpu().numpy()
        ecap = st.region("ecap", torch.float32, len(src)).cpu().numpy()
        col = st.region("colour", torch.uint8, n).cpu().numpy()
        assert np.array_equal(col, R.colour(n, src, tgt, ecap, cs, ct))
        # the capacities are the fp32 formulas of the oracle from the device's centres
        comp = np.zeros(n, np.int64)
        c0 = st.region("c0", torch.float64, obs.shape[1]).cpu().numpy()[None]
        c1 = st.region("c1", torch.float64, obs.shape[1]).cpu().numpy()[None]
        rcs, rct, recap = R.capacities(obs, comp, np.zeros(n, np.uint8), c0, c1, w, np.zeros(len(src), np.uint8),
                                       np.float32(0.05), np.float32(u), spatial)
        assert np.array_equal(rcs.view(np.uint32), cs.view(np.uint32))
        assert np.array_equal(rct.view(np.uint32), ct.view(np.uint32))
        assert np.array_equal(recap.view(np.uint32), ecap.view(np.uint32))


def _knn_tree(xyz, k):
    from scipy.spatial import cKDTree
    d, nn = cKDTree(xyz).query(xyz, k + 1)
    return np.repeat(np.arange(len(xyz)), k), nn[:, 1:].ravel(), d[:, 1:].ravel()


def _strip(n, seed, length=200.0):
    """n points in a long thin box with their 5-NN graph: deep in breadth-first levels."""
    rng = np.random.default_rng(seed)
    xyz = (rng.uniform(0, 1, (n, 3)) * np.array([length, 1.0, 1.0])).astype(np.float32)
    src, tgt, _ = _knn_tree(xyz, 5)
    return xyz, src, tgt


@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [0, 1])
def test_large_component_end_to_end_against_oracle(spatial):
    """5000 vertices: the first iterations run k-means, centres and values on the 512-thread path (> 2048)."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    rng = np.random.default_rng(3)
    n, cutoff = 5000, 10
    xyz = rng.uniform(0, 4, (n, 3)).astype(np.float32)
    piece = (xyz[:, 0] // 1 + 4 * (xyz[:, 1] // 1)).astype(np.int64)
    emb = rng.normal(0, 1, (16, 4))[piece] + rng.normal(0, 0.3, (n, 4))
    obs = (np.concatenate([emb, 0.2 * xyz], 1) if spatial else emb).astype(np.float32)
    src, tgt, _ = _knn_tree(xyz, 5)
    w = np.ones(len(src), np.float32)
    kw = dict(cutoff=cutoff, spatial=spatial, weight_decay=0.7)
    st = cp.prepare(obs, src, tgt, w, 0.05, **kw)
    stats, ref = {}, {}
    with torch.cuda.device(st.dev):
        cp.run(st, 0.05, cutoff, spatial, 0.7, 0, stats=stats)
        comps, inc = st.output()
    R.cutpursuit(obs, src, tgt, w, 0.05, stats=ref, **kw)
    assert abs(stats["energy"] - ref["energy"]) <= 1e-3 * abs(ref["energy"])
    assert abs(stats["components"] - ref["components"]) <= max(1, 0.02 * ref["components"])
    inc = inc.cpu().numpy()
    off, mem = comps.offsets.cpu().numpy(), comps.members.cpu().numpy()
    assert len(comps) == inc.max() + 1 and set(np.unique(inc)) == set(range(len(comps)))
    for c in range(len(comps)):
        assert (inc[mem[off[c]:off[c + 1]]] == c).all()
        assert (np.diff(mem[off[c]:off[c + 1]]) > 0).all()
    import scipy.sparse as sps
    from scipy.sparse.csgraph import connected_components
    same = inc[src] == inc[tgt]
    g = sps.coo_matrix((np.ones(same.sum()), (src[same], tgt[same])), shape=(n, n))
    assert connected_components(g, directed=False)[0] == len(comps)
    # no component at or below the cutoff keeps a neighbour (51 cutoff rounds are far from needed here)
    size = np.bincount(inc)
    cross = inc[src] != inc[tgt]
    has_nb = np.zeros(len(comps), bool)
    has_nb[inc[src][cross]] = True
    has_nb[inc[tgt][cross]] = True
    assert not (has_nb & (size <= cutoff)).any()


def _put(st, name, dtype, a):
    st.region(name, dtype, a.size).copy_(torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(st.dev))


def _get(st, name, dtype, count):
    return st.region(name, dtype, count).cpu().numpy()


@pytest.mark.gpu
def test_deep_colouring_and_device_flow_certificate():
    """10^4 vertices in a strip, sources at one end and sinks at the other: the residual BFS needs many 16-level
    batches.  The colouring equals the oracle's; the device's own preflow of the reversed problem is checked by
    certificate (capacities, conservation with nonnegative excess, value = the oracle's maximum flow)."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import shortest_path
    n = 10_000
    xyz, src, tgt = _strip(n, 8)
    rng = np.random.default_rng(9)
    obs = rng.normal(0, 1, (n, 2)).astype(np.float32)
    w = rng.uniform(0.5, 1.5, len(src)).astype(np.float32)
    st = cp.prepare(obs, src, tgt, w, 1.0)
    cs = np.where(xyz[:, 0] > 120, rng.uniform(0, 1, n), 0).astype(np.float32)
    ct = np.where(xyz[:, 0] < 30, rng.uniform(0, 1, n), 0).astype(np.float32)
    ecap = (w * np.float32(0.02)).astype(np.float32)
    tmax = np.float32(max(cs.max(), ct.max()))
    words = _get(st, "words", torch.int64, 10)
    words[1] = int(tmax.view(np.uint32))
    _put(st, "words", torch.int64, words)
    for name, a in (("cs", cs), ("ct", ct), ("ecap", ecap)):
        _put(st, name, torch.float32, a)
    st.maxflow()
    seeds = np.flatnonzero(ct > 0)  # hop depth from the sink side, through one extra vertex n joined to it
    g = coo_matrix((np.ones(len(src) + len(seeds)), (np.r_[src, np.full(len(seeds), n)], np.r_[tgt, seeds])),
                   shape=(n + 1, n + 1))
    depth = shortest_path(g, directed=False, unweighted=True, indices=n)[:n] - 1
    assert depth[np.isfinite(depth)].max() > 4 * 16
    col = _get(st, "colour", torch.uint8, n)
    assert np.array_equal(col, R.colour(n, src, tgt, ecap, cs, ct))
    assert (col == R.SINK).any() and (col == R.SOURCE).any()
    k = R.shift(tmax, n)
    qe, qs, qt = R.fix(ecap, k), R.fix(cs, k), R.fix(ct, k)
    A = 2 * len(src)
    res = _get(st, "res", torch.int64, A)
    rev = _get(st, "arc_rev", torch.int32, A)
    edge = _get(st, "arc_edge", torch.int32, A)
    off = _get(st, "arc_off", torch.int32, n + 1)
    ex = _get(st, "excess", torch.int64, n)
    rt = _get(st, "rt", torch.int64, n)
    assert (res >= 0).all() and (rt >= 0).all() and (ex >= 0).all()
    assert np.array_equal(res + res[rev], 2 * qe[edge])
    out = np.add.reduceat(np.append(qe[edge] - res, 0), off[:-1].clip(max=A)) * (np.diff(off) > 0)
    assert np.array_equal(ex, qt - out - (qs - rt))  # the reversed problem: ct feeds, cs drains
    flow, *_ = R.max_flow(n, src, tgt, qe, qs, qt)
    assert int((qs - rt).sum()) == flow


@pytest.mark.gpu
@pytest.mark.parametrize("spatial", [0, 1])
def test_kmeans_centres_capacities_against_oracle(spatial):
    """Four components (4000 vertices on the 512-thread path, 1500, 499 and 1 on the warp path) with roots that
    are not their smallest vertex: k-means labels equal the oracle's wherever its decision margin exceeds 1e-6,
    centres within 1e-6, capacities bit-exact to the fp32 formulas, saturation as compute_center."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    rng = np.random.default_rng(5)
    n = 6000
    comp = np.repeat(np.arange(4), [4000, 1500, 499, 1])[rng.permutation(n)]
    blob = rng.integers(0, 2, n)
    obs = (rng.normal(0, 0.4, (n, 3)) + blob[:, None] * np.array([1.0, -1.0, 0.5])).astype(np.float32)
    xyz, src, tgt = _strip(n, 6, length=20.0)
    w = rng.uniform(0.5, 1.5, len(src)).astype(np.float32)
    st = cp.prepare(obs, src, tgt, w, 0.05, spatial=spatial, weight_decay=0.7)
    members, offsets = R.members_of(comp, 4)
    root = np.array([members[offsets[c] + (offsets[c + 1] - offsets[c]) // 2] for c in range(4)])
    sat = np.zeros(n, np.uint8)
    active = (rng.uniform(size=len(src)) < 0.2).astype(np.uint8)
    _put(st, "comp", torch.int32, comp.astype(np.int32))
    _put(st, "root", torch.int32, root.astype(np.int32))
    _put(st, "active", torch.uint8, active)
    value = R.comp_values(obs, members, offsets)
    _put(st, "value", torch.float64, value)
    st.n_comp = 4
    st.members()
    assert np.array_equal(_get(st, "members", torch.int32, n), members)
    st.kmeans(3, 11)
    label = _get(st, "label", torch.uint8, n)
    margin = np.zeros(n)
    want = R.kmeans(obs, members, offsets, sat, root, 3, 11, margins=margin)
    sure = margin > 1e-6
    assert sure.sum() > 0.9 * n
    assert np.array_equal(label[sure], want[sure])
    st.centers(spatial)
    c0 = _get(st, "c0", torch.float64, 12).reshape(4, 3)
    c1 = _get(st, "c1", torch.float64, 12).reshape(4, 3)
    rsat = sat.copy()
    r0, r1 = R.centers(obs, members, offsets, rsat, value, label, spatial)
    live = ~rsat[:4].astype(bool) | bool(spatial)
    np.testing.assert_allclose(c0[live], r0[live], rtol=0, atol=1e-6)
    np.testing.assert_allclose(c1[live], r1[live], rtol=0, atol=1e-6)
    assert np.array_equal(_get(st, "sat", torch.uint8, 4), rsat[:4])
    assert rsat[3] == (0 if spatial else 1)  # the one-vertex component has an empty side
    u = cp.unary_weights(0.7)[1] if spatial else 1.0
    st.capacities(np.float32(0.05), u, spatial)
    cs, ct, ecap = R.capacities(obs, comp, _get(st, "sat", torch.uint8, n), c0, c1, w, active, np.float32(0.05),
                                np.float32(u), spatial)
    for name, a in (("cs", cs), ("ct", ct), ("ecap", ecap)):
        assert np.array_equal(_get(st, name, torch.float32, a.size).view(np.uint32), a.view(np.uint32)), name


def _stripes(n_stripes=6, width=10, values=None, noise=0.0, seed=0):
    """A grid of n_stripes vertical stripes width x width each, stripe s valued values[s]."""
    rng = np.random.default_rng(seed)
    H, W = width, width * n_stripes
    idx = np.arange(H * W).reshape(H, W)
    stripe = (np.arange(H * W) % W) // width
    vals = np.arange(n_stripes) if values is None else np.asarray(values)
    obs = (vals[stripe][:, None] * np.array([1.0, 0.5]) + rng.normal(0, noise, (H * W, 2))).astype(np.float32)
    src = np.concatenate([idx[:-1].ravel(), idx[:, :-1].ravel()])
    tgt = np.concatenate([idx[1:].ravel(), idx[:, 1:].ravel()])
    return obs, src, tgt, stripe


def _seed_state(st, comp, root, sat, active, n_comp):
    _put(st, "comp", torch.int32, comp.astype(np.int32))
    r = np.zeros(st.n, np.int32)
    r[:len(root)] = root
    _put(st, "root", torch.int32, r)
    sfull = np.zeros(st.n, np.uint8)
    sfull[:len(sat)] = sat
    _put(st, "sat", torch.uint8, sfull)
    _put(st, "active", torch.uint8, active.astype(np.uint8))
    st.n_comp = n_comp


@pytest.mark.gpu
def test_split_numbering_bit_exact():
    """Old roots keep their index (roots chosen away from the smallest vertex), new pieces are appended by smallest
    vertex, a saturated component is left whole even with active edges inside it."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs, src, tgt, stripe = _stripes(6, 12, noise=0.1, seed=1)
    n = len(obs)
    rng = np.random.default_rng(2)
    comp = stripe // 2  # three old components of two stripes each
    cross = comp[src] != comp[tgt]
    active = (cross | (rng.uniform(size=len(src)) < 0.45)).astype(np.uint8)
    members, offsets = R.members_of(comp, 3)
    root = np.array([members[offsets[c + 1] - 1 - c] for c in range(3)])
    sat = np.array([0, 1, 0], np.uint8)
    st = cp.prepare(obs, src, tgt, np.ones(len(src), np.float32), 0.1)
    _seed_state(st, comp, root, sat, active, 3)
    st.split()
    rc, rr, rs = comp.copy(), np.zeros(n, np.int64), np.zeros(n, np.uint8)
    rr[:3], rs[:3] = root, sat
    m = R.split(rc, rr, rs, src, tgt, active, 3)
    assert m > 6 and st.n_comp == m
    assert np.array_equal(_get(st, "comp", torch.int32, n), rc)
    assert np.array_equal(_get(st, "root", torch.int32, m), rr[:m])
    assert np.array_equal(_get(st, "sat", torch.uint8, m), rs[:m])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ties", "noisy"])
@pytest.mark.parametrize("is_cutoff", [False, True])
def test_merge_selection_bit_exact(case, is_cutoff):
    """The reduced graph, gains and greedy selection from the same partition: the selected pairs, the renumbered
    components, roots, saturation and activity equal the oracle's; values within 1e-12.  "ties": six equal stripes
    valued 0 1 0 1 0 1, whose five borders all have one gain, so the (comp1, comp2) order decides."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    if case == "ties":
        obs, src, tgt, stripe = _stripes(6, 10, values=[0, 1, 0, 1, 0, 1])
        comp, lam, cutoff = stripe, 10.0, 100.0
    else:
        obs, src, tgt, stripe = _stripes(8, 10, values=[0, 0.2, 0.25, 1, 1.1, 0.3, 0.31, 2], noise=0.05, seed=4)
        comp, lam, cutoff = stripe, 1.0, 100.0
    n, n_comp = len(obs), int(comp.max()) + 1
    active = (comp[src] != comp[tgt]).astype(np.uint8)
    members, offsets = R.members_of(comp, n_comp)
    root = members[offsets[:-1] + 1]
    sat = (np.arange(n_comp) % 3 == 1).astype(np.uint8)
    w = np.ones(len(src), np.float32)
    st = cp.prepare(obs, src, tgt, w, lam)
    _seed_state(st, comp, root, sat, active, n_comp)
    n_merged = st.merge(np.float32(lam), cutoff, is_cutoff)
    rc, rr, rs, ra = comp.astype(np.int64), np.zeros(n, np.int64), np.zeros(n, np.uint8), active.copy()
    rr[:n_comp], rs[:n_comp] = root, sat
    sel = []
    value, rm, m = R.merge(obs, rc, rr, rs, src, tgt, w, ra, n_comp, np.float32(lam), cutoff, is_cutoff, selected=sel)
    partner = _get(st, "partner", torch.int32, n_comp)
    assert sorted(sel) == sorted((c, int(p)) for c, p in enumerate(partner) if p > c)
    assert n_merged == rm and st.n_comp == m and rm > 0
    if case == "ties":
        assert sorted(sel) == [(0, 1), (2, 3), (4, 5)]
    assert np.array_equal(_get(st, "comp", torch.int32, n), rc)
    assert np.array_equal(_get(st, "root", torch.int32, m), rr[:m])
    assert np.array_equal(_get(st, "sat", torch.uint8, m), rs[:m])
    assert np.array_equal(_get(st, "active", torch.uint8, len(src)), ra)
    np.testing.assert_allclose(_get(st, "value", torch.float64, m * 2).reshape(m, 2), value, rtol=1e-12, atol=0)


@pytest.mark.gpu
def test_prune_geometry_cut_pursuit_sp_graph_on_device():
    """prune -> compute_graph_nn_2 -> compute_geof -> cutpursuit -> compute_sp_graph on device tensors (features as
    partition.py:165-166, edge weights as :175)."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    from superpoint_graph_b200 import spg_geometry, spg_prune, spg_sp_graph
    rng = np.random.default_rng(7)
    m = 6000
    xyz = np.concatenate([np.c_[rng.uniform(0, 6, m), rng.uniform(0, 5, m), np.zeros(m)],
                          np.c_[np.zeros(m), rng.uniform(0, 5, m), rng.uniform(0, 3, m)],
                          np.c_[rng.uniform(0, 6, m), np.zeros(m), rng.uniform(0, 3, m)]])
    xyz = (xyz + rng.normal(0, 0.01, xyz.shape)).astype(np.float32)
    rgb = np.repeat(np.array([[200, 30, 30], [30, 200, 30], [30, 30, 200]], np.uint8), m, 0)
    pruned = spg_prune.prune(torch.from_numpy(xyz).cuda(), 0.05, torch.from_numpy(rgb).cuda(), None, None, 0, 0)
    xyz_p, rgb_p = pruned[0], pruned[1]
    graph, target2 = spg_geometry.compute_graph_nn_2(xyz_p, 10, 20)
    geof = spg_geometry.compute_geof(xyz_p, target2, 20)
    geof[:, 3] *= 2
    features = torch.cat([geof, rgb_p.float() / 255], 1).contiguous()
    d = graph["distances"]
    w = (1 / (1 + d / d.mean())).float()
    comps, inc = cp.cutpursuit(features, graph["source"], graph["target"], w, 0.1)
    assert inc.is_cuda and comps.offsets.is_cuda and comps.members.is_cuda
    assert 3 <= len(comps) < xyz_p.shape[0] // 10
    g = spg_sp_graph.compute_sp_graph(xyz_p, 1.0, inc, comps, [], 0)
    assert g["sp_point_count"].is_cuda and int(g["sp_point_count"].sum()) == xyz_p.shape[0]
    assert g["sp_centroids"].shape[0] == len(comps)


@pytest.mark.gpu
def test_two_runs_bitwise_identical():
    obs, src, tgt, w, _ = _knn(n=3000, k=5, pieces=6, noise=0.3, seed=4)
    a = _dev_run(obs, src, tgt, w, 0.05, cutoff=3, spatial=1, weight_decay=0.7, seed=7)
    b = _dev_run(obs, src, tgt, w, 0.05, cutoff=3, spatial=1, weight_decay=0.7, seed=7)
    assert np.array_equal(a[1], b[1])
    assert torch.equal(a[0].members, b[0].members)


@pytest.mark.gpu
def test_device_validation_errors():
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs = np.zeros((3, 2), np.float32)
    e = np.array([0, 1])
    w = np.ones(2, np.float32)
    with pytest.raises(IndexError):
        cp.cutpursuit(obs, e, e + 2, w, 1.0)
    bad = obs.copy()
    bad[1, 1] = np.nan
    with pytest.raises(ValueError):
        cp.cutpursuit(bad, e, e + 1, w, 1.0)
    with pytest.raises(ValueError):
        cp.cutpursuit(obs, e, e + 1, np.array([1, np.inf], np.float32), 1.0)
    comps, inc = cp.cutpursuit(obs, e, e + 1, w, 1.0)
    lists, ic = cp.to_numpy((comps, inc))
    assert ic.dtype == np.uint32 and all(a.dtype == np.uint32 for a in lists)
    assert len(comps) == 1 and comps[0].tolist() == [0, 1, 2]


@pytest.mark.gpu
def test_composition_with_sp_graph_and_weight_loss():
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    from superpoint_graph_b200 import spg_partition, spg_sp_graph
    obs, src, tgt, w, truth = _knn(n=800, k=5, pieces=4, noise=0.01, seed=5)
    rng = np.random.default_rng(0)
    xyz = torch.from_numpy(rng.uniform(0, 1, (800, 3)).astype(np.float32)).cuda()
    comps, inc = cp.cutpursuit(torch.from_numpy(obs).cuda(), torch.from_numpy(src).cuda(),
                               torch.from_numpy(tgt).cuda(), torch.from_numpy(w).cuda(), 0.05)
    g = spg_sp_graph.compute_sp_graph(xyz, 0, inc, comps, [], 0)
    assert g["sp_centroids"].shape[0] == len(comps)
    args = types.SimpleNamespace(edge_weight_threshold=-0.5, spatial_emb=0.2, reg_strength=0.4, k_nn_adj=5,
                                 CP_cutoff=4)
    emb = torch.from_numpy(obs).cuda()
    diff = torch.rand(len(src), device="cuda")
    part = cp.compute_partition(args, emb, torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda(), diff, xyz)
    is_tr = torch.from_numpy(truth[src] != truth[tgt]).cuda()
    objects = torch.from_numpy(truth).cuda()
    for scheme in ("seal", "crosspartition"):
        args.loss_weight = scheme
        args.transition_factor = 5
        wl = spg_partition.compute_weight_loss(args, emb, objects, torch.from_numpy(src).cuda(),
                                               torch.from_numpy(tgt).cuda(), is_tr, diff, False, xyz, partition=part)
        off, mem, comp = R.cutpursuit(torch.cat([emb, 0.2 * xyz], 1).cpu().numpy(), src, tgt,
                                      spg_partition.ops.lp_edge_weight(diff, -0.5).float().cpu().numpy(),
                                      np.float32(0.4 / 20), cutoff=4, spatial=1, weight_decay=0.7)
        assert np.array_equal(part[1].cpu().numpy(), comp)
        wl2 = spg_partition.compute_weight_loss(args, emb, objects, torch.from_numpy(src).cuda(),
                                                torch.from_numpy(tgt).cuda(), is_tr, diff, False, xyz,
                                                partition=([None] * len(off[:-1]), torch.from_numpy(comp).cuda()))
        assert torch.equal(wl, wl2)
