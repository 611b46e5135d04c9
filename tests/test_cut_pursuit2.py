"""The node-weighted cut pursuit, libcp.cutpursuit2 (superpoint_graph_b200/spg_cut_pursuit.py cutpursuit2,
csrc/cut_pursuit.cu), and Semantic3D's label inpainting in compute_structure, against the float64 oracle
(oracle/cut_pursuit2_ref.py: cutpursuit2, inpaint_objects, inpainted_structure).

There is no libcp to make a golden from, so the oracle is the arbiter, and metamorphic properties tie it to the
reference's weighted objective.
CPU: the weighted oracle at unit weights (and without weights) is oracle/cut_pursuit_ref.py's unweighted cut
pursuit; scaling the weights by a power of two and lambda by its inverse leaves the partition unchanged; a weight-0
vertex hanging off a component joins it; a disconnected weight-0 island becomes its own NaN-valued component and a
NaN-valued component is never merged; the oracle's inpainted structure is made of its inpainted objects; host
validation, compute_structure's inpaint= refusals, the ABI symbol and kernel names.
GPU: end to end against the oracle (in_component and the CSR bit for bit, the energy to 1e-12, NaN where the
oracle's is NaN) on dyadic weights over the grid and k-NN shapes, on an inpainting problem with a disconnected
unlabelled cluster, on all-zero weights and on n = 1; stage by stage from one state on the warp and 512-thread paths;
unit weights against the device's cutpursuit; compute_structure(sema3d, inpaint=True) against the oracle structure and
on through PartitionStore and load_batch; bitwise reproducibility.
"""
import types

import numpy as np
import pytest
import torch

from oracle import cut_pursuit2_ref as R
from oracle import cut_pursuit_ref as R0
from oracle import structure_ref

DYADIC = np.array([0.0, 0.25, 0.5, 1.0, 2.0], np.float32)


def _weights(n, seed, zeros=0.3):
    """Dyadic vertex weights, about `zeros` of them 0."""
    rng = np.random.default_rng(seed)
    p = np.r_[zeros, np.full(4, (1 - zeros) / 4)]
    return rng.choice(DYADIC, n, p=p).astype(np.float32)


def _grid(H=16, W=16, noise=0.01, seed=0):
    rng = np.random.default_rng(seed)
    xy = np.stack(np.meshgrid(np.arange(H), np.arange(W), indexing="ij"), -1).reshape(-1, 2)
    truth = (xy[:, 0] >= H // 2).astype(np.int64) + 2 * (xy[:, 1] >= W // 3)
    obs = (truth[:, None] * np.array([1.0, 2.0, -1.0]) + rng.normal(0, noise, (H * W, 3))).astype(np.float32)
    idx = np.arange(H * W).reshape(H, W)
    src = np.concatenate([idx[:-1].ravel(), idx[:, :-1].ravel()])
    tgt = np.concatenate([idx[1:].ravel(), idx[:, 1:].ravel()])
    return obs, src, tgt, np.ones(len(src), np.float32)


def _knn_tree(xyz, k):
    from scipy.spatial import cKDTree
    _, nn = cKDTree(xyz).query(xyz, k + 1)
    return np.repeat(np.arange(len(xyz)), k), nn[:, 1:].ravel()


def _knn(n=600, k=5, pieces=3, noise=0.01, seed=1):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    truth = np.minimum((xyz[:, 0] * pieces).astype(np.int64), pieces - 1)
    obs = (truth[:, None] * np.array([1.0, -0.5]) + rng.normal(0, noise, (n, 2))).astype(np.float32)
    src, tgt = _knn_tree(xyz, k)
    return obs, src, tgt, np.ones(len(src), np.float32)


def _sema_cloud(n=1500, island=30, seed=0):
    """A Semantic3D-like labelled cloud: 8 classes in blocks of a 4 x 4 m patch, label histograms [n, 9] (column 0
    counts unlabelled points), about 30 % of the points without a label, and a cluster of `island` unlabelled points
    far from the rest (its 5-NN graph stays inside it)."""
    rng = np.random.default_rng(seed)
    m = n - island
    xyz = np.concatenate([rng.uniform(0, 4, (m, 3)) * [1, 1, 0.5],
                          np.array([40.0, 40.0, 0.0]) + rng.uniform(0, 0.3, (island, 3))]).astype(np.float32)
    cls = (np.floor(xyz[:, 0]) * 2 + np.floor(xyz[:, 1] / 2)).astype(np.int64) % 8 + 1
    labels = np.zeros((n, 9), np.int64)
    labels[np.arange(n), cls] = rng.integers(1, 4, n)
    unlab = rng.uniform(size=n) < 0.3
    unlab[m:] = True
    labels[unlab, 1:] = 0
    labels[unlab, 0] = 1
    rgb = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    return xyz, rgb, labels


def _inpainting(n=1500, seed=0):
    xyz, _, labels = _sema_cloud(n, seed=seed)
    src, tgt = _knn_tree(xyz, 5)
    hard, s, t, ew, nw = structure_ref.inpainting_problem(labels, src, tgt)
    return hard.reshape(-1, 1).astype(np.float32), s, t, ew, nw


def _oracle2(obs, src, tgt, w, nw, lam, seed=0):
    stats = {}
    off, mem, comp = R.cutpursuit2(obs, src, tgt, w, nw, lam, seed=seed, stats=stats)
    return off, mem, comp, stats


def _same_energy(got, want):
    if np.isnan(want):
        return np.isnan(got)
    return abs(got - want) <= 1e-12 * abs(want)


# ------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("case", ["grid", "knn"])
def test_oracle_unit_weights_are_the_unweighted_spg(case):
    obs, src, tgt, w = _grid() if case == "grid" else _knn()
    a = R.cutpursuit2(obs, src, tgt, w, np.ones(len(obs), np.float32), 0.05, seed=3, stats=(sa := {}))
    b = R0.cutpursuit(obs, src, tgt, w, 0.05, cutoff=0, spatial=1, weight_decay=1.0, seed=3, stats=(sb := {}))
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert sa == sb


@pytest.mark.parametrize("weights", ["none", "ones"])
def test_oracle_unit_weights_change_nothing(weights):
    """The weighted oracle without weights or at unit weights is the unweighted oracle bit for bit, stage by stage."""
    obs, src, tgt, w = _knn(n=300, noise=0.3, seed=2)
    n = len(obs)
    ones = None if weights == "none" else np.ones(n, np.float32)
    comp = (np.arange(n) % 3).astype(np.int64)
    members, offsets = R.members_of(comp, 3)
    sat, root = np.zeros(n, np.uint8), members[offsets[:-1]]
    ma, mb = np.zeros(n), np.zeros(n)
    la = R0.kmeans(obs, members, offsets, sat, root, 2, 5, margins=ma)
    lb = R.kmeans(obs, members, offsets, sat, root, 2, 5, margins=mb, node_weight=ones)
    assert np.array_equal(la, lb) and np.array_equal(ma, mb)
    va, vb = R0.comp_values(obs, members, offsets), R.comp_values(obs, members, offsets, ones)
    assert np.array_equal(va, vb)
    ca, cb = R0.centers(obs, members, offsets, sat.copy(), va, la, 1), R.centers(obs, members, offsets, sat.copy(),
                                                                                 va, la, 1, ones)
    assert all(np.array_equal(x, y) for x, y in zip(ca, cb))
    act = np.zeros(len(src), np.uint8)
    pa = R0.capacities(obs, comp, sat, *ca, w, act, np.float32(0.05), np.float32(1), 1)
    pb = R.capacities(obs, comp, sat, *ca, w, act, np.float32(0.05), np.float32(1), 1, ones)
    assert all(np.array_equal(x, y) for x, y in zip(pa, pb))
    assert R0.energy(obs, comp, va, w, act, 0.05) == R.energy(obs, comp, va, w, act, 0.05, ones)


@pytest.mark.parametrize("c", [2.0, 0.25])
@pytest.mark.parametrize("case", ["grid", "knn"])
def test_oracle_power_of_two_scaling(case, c):
    """(c mu, lambda) and (mu, lambda / c): every capacity, gain and energy scales by c exactly, so the partition is
    the same."""
    obs, src, tgt, w = _grid(noise=0.2) if case == "grid" else _knn(noise=0.2)
    nw = _weights(len(obs), 4)
    a = R.cutpursuit2(obs, src, tgt, w, (nw * np.float32(c)).astype(np.float32), 0.05, seed=1)
    b = R.cutpursuit2(obs, src, tgt, w, nw, 0.05 / c, seed=1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert len(a[0]) > 2


def test_oracle_weight_zero_vertex_joins_its_neighbour():
    obs, src, tgt, w = _grid(12, 12)
    n = len(obs)
    obs = np.vstack([obs, [[50.0, -50.0, 50.0]]]).astype(np.float32)  # far from every value, but no observation
    src, tgt, w = np.r_[src, 5], np.r_[tgt, n], np.r_[w, np.float32(1)].astype(np.float32)
    nw = np.r_[np.ones(n), 0].astype(np.float32)
    _, _, comp, _ = _oracle2(obs, src, tgt, w, nw, 0.05)
    assert comp[n] == comp[5]
    assert len(np.unique(comp)) == 4


def test_oracle_zero_island_is_a_nan_component_never_merged():
    """A disconnected island of weight-0 vertices splits off with the value NaN; the energy is then NaN, so the
    main loop runs its 15 iterations.  In a merge pass a NaN component's borders are never candidates."""
    obs, src, tgt, w = _grid(10, 10)
    n = len(obs)
    isl = np.arange(n, n + 6)
    obs = np.vstack([obs, np.zeros((6, 3))]).astype(np.float32)
    src, tgt = np.r_[src, isl[:-1]], np.r_[tgt, isl[1:]]
    w = np.ones(len(src), np.float32)
    nw = np.r_[_weights(n, 7, zeros=0.1), np.zeros(6)].astype(np.float32)
    nw[:4] = 1
    off, mem, comp, stats = _oracle2(obs, src, tgt, w, nw, 0.05)
    c = comp[n]
    assert (comp[isl] == c).all() and (np.bincount(comp)[c] == 6)
    value = R.comp_values(obs, mem, off, nw)
    assert np.isnan(value[c]).all() and not np.isnan(np.delete(value, c, 0)).any()
    assert np.isnan(stats["energy"]) and stats["iterations"] == R.MAX_ITE_MAIN
    # the island joined to the grid by one edge: its border's gain is NaN, with and without is_cutoff
    n_comp = int(comp.max()) + 1
    for is_cutoff in (False, True):
        cc, rr, ss = comp.copy(), np.zeros(len(obs), np.int64), np.zeros(len(obs), np.uint8)
        s2, t2 = np.r_[src, 0], np.r_[tgt, n]
        act = (cc[s2] != cc[t2]).astype(np.uint8)
        sel = []
        R.merge(obs, cc, rr, ss, s2, t2, np.ones(len(s2), np.float32), act, n_comp, np.float32(1e3), 1e9, is_cutoff,
                selected=sel, node_weight=nw)
        assert sel and all(c not in p for p in sel)


def test_oracle_inpainted_structure():
    xyz, _, labels = _sema_cloud(300, island=10, seed=2)
    src, tgt = _knn_tree(xyz, 5)
    nb = np.asarray(_knn_tree(xyz, 10)[1]).reshape(300, 10)
    got = R.inpainted_structure(xyz, labels, nb, 5, 10, seed=1)
    assert np.array_equal(got["source"], src) and np.array_equal(got["target"], tgt)
    objects = R.inpaint_objects(labels, src, tgt, seed=1)
    assert np.array_equal(got["objects"], objects)
    assert np.array_equal(got["is_transition"], objects[src] != objects[tgt])
    assert (objects[-10:] == objects[-1]).all() and (objects == objects[-1]).sum() == 10


def test_host_validation():
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs = np.zeros((3, 2), np.float32)
    e = np.array([0, 1])
    w = np.ones(2, np.float32)
    with pytest.raises(TypeError, match="node_weight"):
        cp.prepare(obs, e, e + 1, w, 1.0, node_weight=np.ones(3))
    with pytest.raises(TypeError, match="node_weight"):
        cp.cutpursuit2(obs, e, e + 1, w, torch.ones(3, dtype=torch.float16), 1.0)
    with pytest.raises(ValueError, match="one entry per vertex"):
        cp.cutpursuit2(obs, e, e + 1, w, np.ones(4, np.float32), 1.0)
    with pytest.raises(TypeError):
        cp.cutpursuit2(obs.astype(np.float64), e, e + 1, w, np.ones(3, np.float32), 1.0)


def test_compute_structure_inpaint_refusals():
    from superpoint_graph_b200 import spg_structure as st
    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=10, use_voronoi=0.0, compute_geof=0, plane_model=0)
    xyz = np.zeros((20, 3), np.float32)
    lab = np.zeros((20, 9), np.uint32)
    with pytest.raises(NotImplementedError, match="cutpursuit2"):
        st.compute_structure(args, "sema3d", xyz, xyz, lab)
    for dataset, labels, objects in (("vkitti", lab, None), ("s3dis", lab, lab), ("sema3d", None, None),
                                     ("sema3d", lab, np.zeros(20, np.int64))):
        with pytest.raises(ValueError, match="inpaint"):
            st.compute_structure(args, dataset, xyz, xyz, labels, objects, inpaint=True)


def test_abi_symbol_and_kernel_names():
    from superpoint_graph_b200 import _lib
    assert "spg_cp_node_weights" in _lib.protos()
    lib = _lib.lib()
    assert lib.spg_cp_node_weights is not None
    kn = {lib.spg_prof_kernel_name(i).decode() for i in range(lib.spg_prof_num_kernels())}
    assert {"cp_graph", "cp_kmeans", "cp_centers", "cp_capacities", "cp_merge", "cp_energy"} <= kn


# ------------------------------------------------------------------------------------------------- GPU
def _dev2(obs, src, tgt, w, nw, lam, seed=0):
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    st = cp.prepare(obs, src, tgt, w, lam, 0, 1, 1.0, node_weight=nw)
    stats = {}
    with torch.cuda.device(st.dev):
        cp.run(st, lam, 0, 1, 1.0, seed, stats=stats)
        comps, inc = st.output()
    return comps.offsets.cpu().numpy(), comps.members.cpu().numpy(), inc.cpu().numpy(), stats


def _fixture(case):
    if case == "grid":
        obs, src, tgt, w = _grid(noise=0.05)
        return obs, src, tgt, w, _weights(len(obs), 10), 0.05
    if case == "knn":
        obs, src, tgt, w = _knn(noise=0.05)
        return obs, src, tgt, w, _weights(len(obs), 11), 0.05
    if case == "inpaint":
        return _inpainting() + (0.01,)
    if case == "zeros":
        obs, src, tgt, w = _knn(n=200, seed=3)
        return obs, src, tgt, w, np.zeros(len(obs), np.float32), 0.05
    if case in ("one0", "one1"):
        e = np.zeros(0, np.int64)
        nw = np.array([case[-1] == "1"], np.float32)
        return np.array([[3.0]], np.float32), e, e, np.zeros(0, np.float32), nw, 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["grid", "knn", "inpaint", "zeros", "one0", "one1"])
def test_end_to_end_matches_oracle(case):
    obs, src, tgt, w, nw, lam = _fixture(case)
    off, mem, inc, stats = _dev2(obs, src, tgt, w, nw, lam, seed=2)
    roff, rmem, rcomp, ref = _oracle2(obs, src, tgt, w, nw, lam, seed=2)
    assert np.array_equal(inc, rcomp)
    assert np.array_equal(off, roff) and np.array_equal(mem, rmem)
    assert _same_energy(stats["energy"], ref["energy"]), (stats["energy"], ref["energy"])
    assert stats["iterations"] == ref["iterations"]
    if case == "inpaint":  # the disconnected unlabelled cluster is one NaN-valued component
        island = np.arange(len(obs) - 30, len(obs))
        c = inc[island[0]]
        assert (inc[island] == c).all() and (inc == c).sum() == 30
        assert np.isnan(stats["energy"])
    if case == "zeros":
        assert np.isnan(stats["energy"]) and len(off) == 2


@pytest.mark.gpu
def test_public_entry_and_node_weights_state():
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs, src, tgt, w, nw, lam = _fixture("knn")
    comps, inc = cp.cutpursuit2(torch.from_numpy(obs).cuda(), src, tgt, w, torch.from_numpy(nw).cuda(), lam, seed=2)
    _, _, comp, _ = _oracle2(obs, src, tgt, w, nw, lam, seed=2)
    assert inc.is_cuda and np.array_equal(inc.cpu().numpy(), comp)
    lists, ic = cp.to_numpy((comps, inc))
    assert ic.dtype == np.uint32 and all(a.dtype == np.uint32 for a in lists)
    # spg_cp_node_weights: the weights, the one component's weight and weighted mean (NaN when all weights are 0)
    for weights in (nw, np.zeros_like(nw)):
        st = cp.prepare(obs, src, tgt, w, lam, 0, 1, 1.0, node_weight=weights)
        assert np.array_equal(st.region("nw", torch.float32, len(obs)).cpu().numpy(), weights)
        cw = st.region("cw", torch.float64, 1).item()
        value = st.region("value", torch.float64, 2).cpu().numpy()
        assert cw == weights.astype(np.float64).sum()
        want = R.comp_values(obs, np.arange(len(obs)), np.array([0, len(obs)]), weights)[0]
        np.testing.assert_allclose(value, want, rtol=1e-12, atol=0)
    for bad in (-0.5, np.nan, np.inf):
        b = nw.copy()
        b[7] = bad
        with pytest.raises(ValueError, match="node_weight"):
            cp.cutpursuit2(obs, src, tgt, w, b, lam)


def _put(st, name, dtype, a):
    st.region(name, dtype, a.size).copy_(torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(st.dev))


def _get(st, name, dtype, count):
    return st.region(name, dtype, count).cpu().numpy()


@pytest.mark.gpu
def test_kmeans_centres_capacities_against_oracle():
    """Four components (4000 vertices on the 512-thread path, 1500, 499 of weight 0 and 1 on the warp path) with
    dyadic weights: k-means labels equal the oracle's wherever its decision margin exceeds 1e-6, centres within 1e-6
    (NaN for the weight-0 component), capacities bit-exact to the fp32 formulas, 0 where the weight is 0."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    rng = np.random.default_rng(5)
    n = 6000
    comp = np.repeat(np.arange(4), [4000, 1500, 499, 1])[rng.permutation(n)]
    blob = rng.integers(0, 2, n)
    obs = (rng.normal(0, 0.4, (n, 3)) + blob[:, None] * np.array([1.0, -1.0, 0.5])).astype(np.float32)
    xyz = (rng.uniform(0, 1, (n, 3)) * np.array([20.0, 1.0, 1.0])).astype(np.float32)
    src, tgt = _knn_tree(xyz, 5)
    w = rng.uniform(0.5, 1.5, len(src)).astype(np.float32)
    nw = _weights(n, 12)
    nw[comp == 2] = 0
    st = cp.prepare(obs, src, tgt, w, 0.05, spatial=1, weight_decay=1.0, node_weight=nw)
    members, offsets = R.members_of(comp, 4)
    root = np.array([members[offsets[c] + (offsets[c + 1] - offsets[c]) // 2] for c in range(4)])
    sat = np.zeros(n, np.uint8)
    active = (rng.uniform(size=len(src)) < 0.2).astype(np.uint8)
    _put(st, "comp", torch.int32, comp.astype(np.int32))
    _put(st, "root", torch.int32, root.astype(np.int32))
    _put(st, "active", torch.uint8, active)
    value = R.comp_values(obs, members, offsets, nw)
    assert np.isnan(value[2]).all()
    _put(st, "value", torch.float64, value)
    st.n_comp = 4
    st.members()
    st.kmeans(3, 11)
    label = _get(st, "label", torch.uint8, n)
    margin = np.zeros(n)
    want = R.kmeans(obs, members, offsets, sat, root, 3, 11, margins=margin, node_weight=nw)
    sure = margin > 1e-6
    assert sure.sum() > 0.9 * n
    assert np.array_equal(label[sure], want[sure])
    assert not label[comp == 2].any()  # no restart beats a seeding energy of 0
    st.centers(1)
    c0 = _get(st, "c0", torch.float64, 12).reshape(4, 3)
    c1 = _get(st, "c1", torch.float64, 12).reshape(4, 3)
    r0, r1 = R.centers(obs, members, offsets, sat.copy(), value, label, 1, nw)
    np.testing.assert_allclose(c0, r0, rtol=0, atol=1e-6)
    np.testing.assert_allclose(c1, r1, rtol=0, atol=1e-6)
    assert np.isnan(c0[2]).all() and np.isnan(c1[2]).all()
    st.capacities(np.float32(0.05), 1.0, 1)
    cs, ct, ecap = R.capacities(obs, comp, sat, c0, c1, w, active, np.float32(0.05), np.float32(1), 1, nw)
    for name, a in (("cs", cs), ("ct", ct), ("ecap", ecap)):
        assert np.array_equal(_get(st, name, torch.float32, a.size).view(np.uint32), a.view(np.uint32)), name
    assert not cs[nw == 0].any() and not ct[nw == 0].any()


def _stripes(n_stripes, width, values, noise, seed):
    rng = np.random.default_rng(seed)
    H, W = width, width * n_stripes
    idx = np.arange(H * W).reshape(H, W)
    stripe = (np.arange(H * W) % W) // width
    obs = (np.asarray(values)[stripe][:, None] * np.array([1.0, 0.5]) + rng.normal(0, noise, (H * W, 2)))
    src = np.concatenate([idx[:-1].ravel(), idx[:, :-1].ravel()])
    tgt = np.concatenate([idx[1:].ravel(), idx[:, 1:].ravel()])
    return obs.astype(np.float32), src, tgt, stripe


@pytest.mark.gpu
@pytest.mark.parametrize("is_cutoff", [False, True])
def test_merge_selection_with_a_nan_component(is_cutoff):
    """Eight stripes, stripe 3 of weight 0 (value NaN): its borders are never selected and the others' selection,
    renumbering, roots, saturation and activity equal the oracle's; values within 1e-12, NaN kept."""
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs, src, tgt, stripe = _stripes(8, 10, [0, 0.2, 0.25, 1, 1.1, 0.3, 0.31, 2], 0.05, 4)
    n, n_comp = len(obs), 8
    nw = _weights(n, 13, zeros=0.2)
    nw[stripe == 3] = 0
    comp, lam, cutoff = stripe, 1.0, 100.0
    active = (comp[src] != comp[tgt]).astype(np.uint8)
    members, offsets = R.members_of(comp, n_comp)
    root = members[offsets[:-1] + 1]
    sat = (np.arange(n_comp) % 3 == 1).astype(np.uint8)
    w = np.ones(len(src), np.float32)
    st = cp.prepare(obs, src, tgt, w, lam, spatial=1, node_weight=nw)
    _put(st, "comp", torch.int32, comp.astype(np.int32))
    r = np.zeros(n, np.int32)
    r[:n_comp] = root
    _put(st, "root", torch.int32, r)
    s = np.zeros(n, np.uint8)
    s[:n_comp] = sat
    _put(st, "sat", torch.uint8, s)
    _put(st, "active", torch.uint8, active)
    st.n_comp = n_comp
    n_merged = st.merge(np.float32(lam), cutoff, is_cutoff)
    rc, rr, rs, ra = comp.astype(np.int64), np.zeros(n, np.int64), np.zeros(n, np.uint8), active.copy()
    rr[:n_comp], rs[:n_comp] = root, sat
    sel = []
    value, rm, m = R.merge(obs, rc, rr, rs, src, tgt, w, ra, n_comp, np.float32(lam), cutoff, is_cutoff, selected=sel,
                           node_weight=nw)
    partner = _get(st, "partner", torch.int32, n_comp)
    assert sorted(sel) == sorted((c, int(p)) for c, p in enumerate(partner) if p > c)
    assert partner[3] == -1 and rm > 0 and n_merged == rm and st.n_comp == m
    assert np.array_equal(_get(st, "comp", torch.int32, n), rc)
    assert np.array_equal(_get(st, "root", torch.int32, m), rr[:m])
    assert np.array_equal(_get(st, "sat", torch.uint8, m), rs[:m])
    assert np.array_equal(_get(st, "active", torch.uint8, len(src)), ra)
    got = _get(st, "value", torch.float64, m * 2).reshape(m, 2)
    assert np.isnan(got).any(1).sum() == 1
    np.testing.assert_allclose(got, value, rtol=1e-12, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["grid", "knn"])
def test_unit_weights_equal_device_cutpursuit(case):
    from superpoint_graph_b200 import spg_cut_pursuit as cp
    obs, src, tgt, w = _grid(noise=0.2) if case == "grid" else _knn(noise=0.2)
    off, mem, inc, stats = _dev2(obs, src, tgt, w, np.ones(len(obs), np.float32), 0.05, seed=5)
    st = cp.prepare(obs, src, tgt, w, 0.05, 0, 1, 1.0)
    ref = {}
    with torch.cuda.device(st.dev):
        cp.run(st, 0.05, 0, 1, 1.0, 5, stats=ref)
        comps, rinc = st.output()
    assert np.array_equal(inc, rinc.cpu().numpy())
    assert np.array_equal(off, comps.offsets.cpu().numpy()) and np.array_equal(mem, comps.members.cpu().numpy())
    assert stats == ref


def _np(t):
    return t.cpu().numpy()


@pytest.mark.gpu
def test_compute_structure_inpaint_against_oracle_and_loader():
    from superpoint_graph_b200 import spg_structure as st
    from superpoint_graph_b200.spg_partition_loader import PartitionStore, load_batch
    xyz, rgb, labels = _sema_cloud(1500, seed=6)
    args = types.SimpleNamespace(k_nn_adj=5, k_nn_local=10, use_voronoi=0.0, compute_geof=0, plane_model=0)
    got = st.compute_structure(args, "sema3d", xyz, rgb, labels, inpaint=True, seed=4)
    nb = _np(got["target_local_geometry"])
    want = R.inpainted_structure(xyz, labels, nb, 5, 10, seed=4)
    assert np.array_equal(_np(got["graph_nn"]["source"]), want["source"])
    assert np.array_equal(_np(got["graph_nn"]["target"]), want["target"])
    for k in ("is_transition", "objects", "xyn", "elevation"):
        assert np.array_equal(_np(got[k]), np.asarray(want[k]).astype(_np(got[k]).dtype)), k
    assert np.array_equal(_np(got["labels"]), labels)
    assert np.array_equal(nb, want["target_local_geometry"])
    objects = _np(got["objects"])
    assert 8 <= objects.max() + 1 < 200 and _np(got["is_transition"]).any()
    island = objects[-30:]
    assert (island == island[0]).all() and (objects == island[0]).sum() == 30
    host = (xyz, rgb.astype(np.float32), want["source"], want["target"], want["is_transition"].astype(np.uint8),
            nb.astype(np.uint32), labels.astype(np.int32), want["objects"].astype(np.uint32), want["elevation"],
            want["xyn"])
    bargs = types.SimpleNamespace(ver_value="ptn", k_nn_local=10, use_rgb=1, global_feat="eXYrgb", pc_augm_rot=0,
                                  pc_augm_jitter=0, max_ver_train=0, learned_embeddings_geof=0)
    outs = []
    for tup in (st.as_read_structure(got, False), host):
        store = PartitionStore()
        store.add("A/f.h5", *tup)
        store.finalize(torch.device("cuda"))
        np.random.seed(0)
        outs.append(load_batch(store, ["A/f.h5"], False, bargs))
    a, b = outs
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        xs, ys = (x, y) if isinstance(x, tuple) else ((x,), (y,))
        for u, v in zip(xs, ys):
            if torch.is_tensor(u):
                assert torch.equal(u, v)
            else:
                assert (u is None and v is None) or np.array_equal(np.asarray(u), np.asarray(v))


@pytest.mark.gpu
def test_two_runs_bitwise_identical():
    obs, src, tgt, w, nw, lam = _fixture("inpaint")
    a = _dev2(obs, src, tgt, w, nw, lam, seed=9)
    b = _dev2(obs, src, tgt, w, nw, lam, seed=9)
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)
    assert np.array_equal(np.float64(a[3]["energy"]), np.float64(b[3]["energy"]), equal_nan=True)
