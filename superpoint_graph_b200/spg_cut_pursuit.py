"""The l0 cut pursuit partition on the device: `libcp.cutpursuit` of both partition pipelines (ref:
partition/cut-pursuit/src/cutpursuit.cpp:77-105; called at partition/partition.py:177 and
supervized_partition/losses.py:82), and the node-weighted `libcp.cutpursuit2` (cutpursuit.cpp:107-128) that
supervized_partition/graph_processing.py:163 uses to inpaint Semantic3D's labels.

    from superpoint_graph_b200.spg_cut_pursuit import cutpursuit, to_numpy

    components, in_component = cutpursuit(features, source, target, edge_weight, reg_strength)
    graph_sp = compute_sp_graph(xyz, d_max, in_component, components, labels, n_labels)
    components, in_component = cutpursuit2(obs, source, target, edge_weight, node_weight, reg_strength)

Same arguments as libcp (speed 4: 3 flow steps, 10 k-means restarts of 5 iterations, at most 15 iterations, a
backward merge step, stopping ratio 0.05; every vertex weighs 1).  spatial = 0 is CutPursuit_L2, 1 is
CutPursuit_SPG.  in_component is an int64 CUDA tensor and components a `Components` CSR value (len() and indexing);
to_numpy gives libcp's types.  The k-means draws are Philox4x32-10 keyed by `seed`, so a partition is reproducible;
the minimal-cut colouring, the component numbering and the merge selection are the reference's (DESIGN.md §4).
cutpursuit2 is CutPursuit_SPG with the caller's vertex weights, cutoff 0 and weight_decay 1; a vertex of weight 0
holds no observation, and a component whose weights are all 0 has the value NaN and is never merged, as in the
reference.  The kernels are in csrc/cut_pursuit.cu.
"""
import math

import numpy as np
import torch

from . import _lib, ops
from ._inputs import check_dtype, check_ints, device_of, on_device

__all__ = ["Components", "cutpursuit", "cutpursuit2", "to_numpy", "compute_partition"]

FLOW_STEPS, MAX_ITE_MAIN, STOPPING_RATIO, CUTOFF_ROUNDS = 3, 15, 0.05, 50
REGIONS = ("obs", "comp", "root", "sat", "label", "colour", "active", "value", "c0", "c1", "cs", "ct", "ecap",
           "members", "offsets", "words", "dwords", "partner", "res", "excess", "rt", "arc_off", "arc_dst", "arc_rev",
           "arc_edge", "nw", "cw")


class Components:
    """The components of a partition as a CSR: offsets [n_com + 1] and members [n] (int64 CUDA, ascending vertex
    id within a component).  len() is the component count; components[i] is the members of component i."""

    def __init__(self, offsets, members):
        self.offsets = offsets
        self.members = members
        self._host = None

    def __len__(self):
        return self.offsets.numel() - 1

    def __getitem__(self, i):
        if self._host is None:
            self._host = self.offsets.cpu().numpy()
        n = len(self)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError("component %d out of range for %d components" % (i, n))
        return self.members[int(self._host[i]):int(self._host[i + 1])]


def unary_weights(weight_decay):
    """SPG's per-step weights (CutPursuit_SPG.h:75-79): float32 decay^-3, then times decay before each step."""
    wd = np.float32(weight_decay)
    u = np.float32(np.power(wd, np.float32(-FLOW_STEPS)))
    out = []
    for _ in range(FLOW_STEPS):
        u = np.float32(u * wd)
        out.append(float(u))
    return out


class State:
    """The device state of one cut pursuit: the workspace and the stage calls on it (csrc/cut_pursuit.cu)."""

    def __init__(self, obs, source, target, edge_weight, node_weight=None):
        self.n, self.D = obs.shape
        self.E = source.numel()
        self.dev = obs.device
        self.ws = ops._workspace("spg_cp_workspace", self.dev, self.n, self.E, self.D)
        self.out = torch.zeros(4, dtype=torch.int64)
        self.dout = torch.zeros(4, dtype=torch.float64)
        self._call("spg_cp_setup", obs, source, target, edge_weight, *self._dims(), self.out)
        self.status = int(self.out[0])
        if node_weight is not None and self.status == 0:
            self._call("spg_cp_node_weights", node_weight, *self._dims(), self.out)
            self.status = int(self.out[0])
        self.n_comp = 1

    def _dims(self):
        return self.n, self.E, self.D, self.ws, self.ws.numel()

    def _call(self, name, *args):
        _lib.call(name, *args, _lib.current_stream())

    def region(self, name, dtype, count):
        offs = torch.zeros(len(REGIONS), dtype=torch.int64)
        _lib.call("spg_cp_regions", self.n, self.E, self.D, offs)
        o = int(offs[REGIONS.index(name)])
        nb = torch.empty((), dtype=dtype).element_size() * count
        return self.ws[o:o + nb].view(dtype)

    def members(self):
        self._call("spg_cp_members", *self._dims(), self.n_comp)

    def kmeans(self, iteration, seed):
        self._call("spg_cp_kmeans", *self._dims(), self.n_comp, int(iteration), int(seed))

    def centers(self, spatial):
        self._call("spg_cp_centers", *self._dims(), self.n_comp, int(spatial))

    def capacities(self, reg_strength, unary, spatial):
        self._call("spg_cp_capacities", *self._dims(), float(reg_strength), float(unary), int(spatial))

    def maxflow(self):
        self._call("spg_cp_maxflow", *self._dims(), self.out)
        return int(self.out[0])

    def activate(self, spatial):
        self._call("spg_cp_activate", *self._dims(), self.n_comp, int(spatial), self.out)
        return int(self.out[0])

    def split(self):
        self._call("spg_cp_split", *self._dims(), self.n_comp, self.out)
        self.n_comp = int(self.out[0])

    def merge(self, reg_strength, cutoff, is_cutoff):
        self._call("spg_cp_merge", *self._dims(), self.n_comp, float(reg_strength), float(cutoff), int(is_cutoff),
                   self.out)
        self.n_comp = int(self.out[1])
        return int(self.out[0])

    def energy(self, reg_strength):
        self._call("spg_cp_energy", *self._dims(), float(reg_strength), self.dout)
        return float(self.dout[2])

    def output(self):
        in_component = torch.empty(self.n, dtype=torch.int64, device=self.dev)
        offsets = torch.empty(self.n_comp + 1, dtype=torch.int64, device=self.dev)
        members = torch.empty(self.n, dtype=torch.int64, device=self.dev)
        self._call("spg_cp_output", *self._dims(), self.n_comp, in_component, offsets, members)
        return Components(offsets, members), in_component


def _relative_drop(old, new):
    """(old - new) / old with IEEE semantics (a zero old energy gives nan or +-inf, never an exception)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(old - new) / np.float64(old))


def run(state, reg_strength, cutoff, spatial, weight_decay, seed, timer=None, stats=None):
    """CutPursuit::run (ref: CutPursuit.h:73-160) on a set-up State; `timer(stage)` brackets each stage when
    given, and `stats` collects the iteration count and the push-relabel rounds."""
    lam = float(np.float32(reg_strength))
    unary = unary_weights(weight_decay) if spatial else [1.0] * FLOW_STEPS
    tick = timer or (lambda stage: _Null())
    old = state.energy(lam)
    ite = rounds = 0
    for ite in range(1, MAX_ITE_MAIN + 1):
        with tick("kmeans"):
            state.members()
            state.kmeans(ite, seed)
        for step in range(FLOW_STEPS):
            with tick("flow"):
                state.centers(spatial)
                state.capacities(lam, unary[step], spatial)
                rounds += state.maxflow()
        with tick("colour"):
            saturation = state.activate(spatial)
        with tick("split"):
            state.split()
        with tick("merge"):
            state.merge(lam, 0, False)
        energy = state.energy(lam)
        if saturation == state.n:
            break
        if _relative_drop(old, energy) < STOPPING_RATIO:
            break
        old = energy
    if cutoff > 0:
        with tick("cutoff"):
            i = 0
            while True:
                n_merged = state.merge(lam, cutoff, True)
                i += 1
                if n_merged == 0 or i > CUTOFF_ROUNDS:
                    break
    if stats is not None:
        stats.update(iterations=ite, push_relabel_rounds=rounds, components=state.n_comp,
                     energy=state.energy(lam))


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def prepare(obs, source, target, edge_weight, reg_strength, cutoff=0, spatial=0, weight_decay=1.0, node_weight=None):
    """Host validation and the device state; see cutpursuit and cutpursuit2 (node_weight: float32 [n], every vertex
    weighs 1 when None)."""
    shape = tuple(obs.shape)
    if len(shape) != 2 or shape[0] < 1:
        raise ValueError("obs must be [n, D] with n >= 1 (got shape %s)" % (shape,))
    n, D = shape
    if not 1 <= D <= 32:
        raise ValueError("obs must have between 1 and 32 columns (got %d)" % D)
    if cutoff < 0:
        raise ValueError("cutoff must be >= 0 (got %r)" % (cutoff,))
    if spatial not in (0, 1):
        raise ValueError("spatial must be 0 or 1 (got %r)" % (spatial,))
    if not weight_decay > 0:
        raise ValueError("weight_decay must be > 0 (got %r)" % (weight_decay,))
    if not math.isfinite(float(reg_strength)):
        raise ValueError("reg_strength must be finite (got %r)" % (reg_strength,))
    check_dtype(obs, "obs", "float32")
    check_dtype(edge_weight, "edge_weight", "float32")
    check_ints(source, "source")
    check_ints(target, "target")
    sizes = [a.numel() if torch.is_tensor(a) else np.asarray(a).size for a in (source, target, edge_weight)]
    if len(set(sizes)) != 1:
        raise ValueError("source, target and edge_weight must have one entry per edge (got %d, %d, %d)"
                         % tuple(sizes))
    if node_weight is not None:
        check_dtype(node_weight, "node_weight", "float32")
        m = node_weight.numel() if torch.is_tensor(node_weight) else np.asarray(node_weight).size
        if m != n:
            raise ValueError("node_weight must have one entry per vertex (got %d for %d vertices)" % (m, n))
    dev = device_of(obs, source, target, edge_weight, node_weight)
    obs_t = on_device(obs, dev)
    w = on_device(edge_weight, dev).reshape(-1)
    src = on_device(source, dev, int64=True).reshape(-1)
    tgt = on_device(target, dev, int64=True).reshape(-1)
    nw = None if node_weight is None else on_device(node_weight, dev).reshape(-1)
    with torch.cuda.device(dev):
        state = State(obs_t, src, tgt, w, nw)
    if state.status & 4:
        raise IndexError("an edge id is outside [0, %d)" % n)
    if state.status & 1:
        raise ValueError("obs contains NaN or infinity")
    if state.status & 2:
        raise ValueError("edge_weight contains NaN or infinity")
    if state.status & 8:
        raise ValueError("node_weight contains a negative weight, NaN or infinity")
    return state


def cutpursuit(obs, source, target, edge_weight, reg_strength, cutoff=0, spatial=0, weight_decay=1.0, seed=0):
    """(components, in_component) of the l0 cut pursuit partition of obs on the graph (source, target,
    edge_weight) (ref: libcp.cutpursuit).

    TypeError: obs or edge_weight not float32, non-integer ids.  ValueError: shapes, D outside [1, 32], cutoff < 0,
    spatial not in {0, 1}, weight_decay <= 0, non-finite observations or weights.  IndexError: an edge id outside
    [0, n)."""
    state = prepare(obs, source, target, edge_weight, reg_strength, cutoff, spatial, weight_decay)
    with torch.cuda.device(state.dev):
        run(state, reg_strength, cutoff, spatial, weight_decay, seed)
        return state.output()


def cutpursuit2(obs, source, target, edge_weight, node_weight, reg_strength, seed=0):
    """(components, in_component) of libcp.cutpursuit2 (ref: cutpursuit.cpp:107-128): CutPursuit_SPG with the vertex
    weights node_weight (float32 [n], >= 0), cutoff 0, weight_decay 1 (unary weights 1), speed 4.  A vertex of weight
    0 holds no observation: it takes the component its edges lead it to, and a component whose weights are all 0 keeps
    the value NaN and is never merged (DESIGN.md §4).

    TypeError: obs, edge_weight or node_weight not float32, non-integer ids.  ValueError: shapes, D outside [1, 32],
    non-finite observations or edge weights, a negative or non-finite node weight.  IndexError: an edge id outside
    [0, n)."""
    state = prepare(obs, source, target, edge_weight, reg_strength, 0, 1, 1.0, node_weight=node_weight)
    with torch.cuda.device(state.dev):
        run(state, reg_strength, 0, 1, 1.0, seed)
        return state.output()


def to_numpy(partition):
    """libcp's types: a list of uint32 member arrays and a uint32 in_component."""
    components, in_component = partition
    off = components.offsets.cpu().numpy()
    mem = components.members.cpu().numpy().astype(np.uint32)
    return [mem[off[i]:off[i + 1]] for i in range(len(off) - 1)], in_component.cpu().numpy().astype(np.uint32)


def compute_partition(args, embeddings, edg_source, edg_target, diff, xyz=0, seed=0):
    """(pred_components, pred_in_component) on the device — ref: losses.py:67-89.  Edge weights from
    ops.lp_edge_weight (cast to float32), ver_value = [embeddings | spatial_emb * xyz], lambda = reg_strength /
    (4 k_nn_adj), cutoff = CP_cutoff, weight_decay = 0.7.  Feed the result to
    spg_partition.compute_weight_loss(..., partition=...)."""
    dev = device_of(embeddings, diff)
    d = diff if torch.is_tensor(diff) else torch.as_tensor(np.asarray(diff))
    edge_weight = ops.lp_edge_weight(d.detach().to(device=dev, dtype=torch.float32),
                                     args.edge_weight_threshold).to(torch.float32)
    ver_value = embeddings.detach().to(device=dev, dtype=torch.float32)
    use_spatial = 0
    if args.spatial_emb > 0:
        x = xyz if torch.is_tensor(xyz) else torch.as_tensor(np.asarray(xyz))
        ver_value = torch.cat([ver_value, (args.spatial_emb * x.to(device=dev, dtype=torch.float32))], 1)
        use_spatial = 1
    return cutpursuit(ver_value.contiguous(), edg_source, edg_target, edge_weight,
                      args.reg_strength / (4 * args.k_nn_adj), cutoff=args.CP_cutoff, spatial=use_spatial,
                      weight_decay=0.7, seed=seed)
