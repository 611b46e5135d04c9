"""Device-side batch builder: the per-superpoint half of the reference's data loader.

Reference: learning/spg.py:130-170 (`loader`: one `load_superpoint` per graph node, `np.stack` of
`cloud.T`), :198-236 (`load_superpoint`: resample to `ptn_npts`, centre / normalise xyz, attribute
selection), :238-260 (`augment_cloud`).  There every superpoint is one HDF5 dataset read, a handful
of numpy calls and a host->device copy of the finished [Nv, F, L] tensor (7 KB per superpoint per
step).  Here the parsed points live in HBM once (`SuperpointStore`: one packed [rows, C] array —
all of S3DIS is a few GB, an H100 has 80 GB), the host only decides WHICH rows (ids, sample
indices: 0.5 KB per superpoint) and one kernel (`spg_cloud_build`, csrc/loader.cu) emits the
tensor PointNet reads.  With the host-drawn indices the output is bit-identical to the
reference's; `device_rng=True` moves the draws onto the GPU as well (same distribution, not the
same MT19937 stream).
"""
import math
import random

import numpy as np
import torch

from . import _inputs, ops

_ATTRIBS = (("xyz", (0, 1, 2)), ("rgb", (3, 4, 5)), ("e", (6,)), ("lpsv", (7, 8, 9, 10)),
            ("XYZ", (11, 12, 13)))


def attrib_columns(pc_attribs, n_columns):
    """`--pc_attribs` -> source columns (ref: learning/spg.py:221-230)."""
    if pc_attribs == "":
        return list(range(n_columns))
    if "d" in pc_attribs:
        # same failure as the reference, which concatenates the 1-D slice P[:,14] (spg.py:228-230)
        raise ValueError("all the input arrays must have same number of dimensions (pc_attribs 'd')")
    cols = []
    for key, cc in _ATTRIBS:
        if key in pc_attribs:
            cols.extend(cc)
    return cols


class SuperpointStore(object):
    """Parsed superpoints of one or more files, packed for the device.

    `add(fname, {sp_id: ndarray [n, C]})` mirrors the reference's `parsed/<fname>.h5` layout (one
    dataset per superpoint, learning/s3dis_dataset.py:151-158); `finalize(device)` uploads once."""

    def __init__(self):
        self._chunks, self._index, self._rows = [], {}, 0
        self.points = None
        self.n_columns = None
        self._dense, self._columns = {}, {}

    def add(self, fname, superpoints):
        for sp_id, P in superpoints.items():
            P = np.ascontiguousarray(P, dtype=np.float32)
            if P.ndim != 2 or P.shape[1] < 3:
                raise ValueError("superpoint %s/%s: expected [n, >=3] points" % (fname, sp_id))
            if self.n_columns is None:
                self.n_columns = P.shape[1]
            elif self.n_columns != P.shape[1]:
                raise ValueError("superpoints with different numbers of attributes")
            self._index[(fname, int(sp_id))] = (self._rows, P.shape[0])
            self._chunks.append(P)
            self._rows += P.shape[0]

    def finalize(self, device):
        """Uploads the packed array.  Rows are padded with zeros to a multiple of 4 floats so that
        the kernel fetches a point with 128-bit loads (15 parsed columns -> 64-byte rows)."""
        nc = self.n_columns or 3
        ld = (nc + 3) // 4 * 4
        host = np.zeros((self._rows, ld), np.float32)
        r = 0
        for P in self._chunks:
            host[r:r + P.shape[0], :nc] = P
            r += P.shape[0]
        self.points = torch.from_numpy(host).to(device)
        self._chunks = []
        # per file, dense by superpoint id: first row (int64) and count (int32, -1 for an id the store lacks)
        per_file = {}
        for (fname, sp_id), (row, n) in self._index.items():
            if sp_id >= 0:
                per_file.setdefault(fname, []).append((sp_id, row, n))
        self._dense = {}
        for fname, entries in per_file.items():
            ids, rows, counts = (np.array(c, dtype=np.int64) for c in zip(*entries))
            first = np.zeros(int(ids.max()) + 1, np.int64)
            count = -np.ones(int(ids.max()) + 1, np.int32)
            first[ids], count[ids] = rows, counts
            self._dense[fname] = (torch.from_numpy(first).to(device), torch.from_numpy(count).to(device))
        return self

    def count(self, fname, sp_id):
        return self._index[(fname, int(sp_id))][1]

    def start(self, fname, sp_id):
        return self._index[(fname, int(sp_id))][0]

    def device_index(self, fname):
        """(first row int64 [ids], count int32 [ids]) on the device, indexed by superpoint id (count -1: not in the
        store), or None for a file without superpoints."""
        return self._dense.get(fname)

    def device_columns(self, cols):
        """The source columns `cols` as a device int32 tensor, kept per column list; written element by element
        from the host's integers, so no host buffer is copied and the stream is not synchronised."""
        cols = tuple(cols)
        t = self._columns.get(cols)
        if t is None:
            t = torch.empty(len(cols), dtype=torch.int32, device=self.points.device)
            for f, c in enumerate(cols):
                t[f:f + 1].fill_(c)
            self._columns[cols] = t
        return t


def sample_indices(n, npts, rs):
    """ref: learning/spg.py:209-214 — the draws (and their order) of the reference."""
    if n > npts:
        return rs.choice(n, npts)
    if n < npts:
        return np.concatenate([np.arange(n), rs.choice(n, npts - n)])
    return np.arange(n)


def augment_matrix(args, rnd=random):
    """3x3 of `augment_cloud` (ref: learning/spg.py:240-253), same draws in the same order.
    transforms3d's zfdir2mat / axangle2mat are written out: uniform zoom, rotation about z,
    reflections of x and y."""
    M = np.eye(3)
    if args.pc_augm_scale > 1:
        s = rnd.uniform(1 / args.pc_augm_scale, args.pc_augm_scale)
        M = np.dot(np.eye(3) * s, M)
    if args.pc_augm_rot == 1:
        angle = rnd.uniform(0, 2 * math.pi)
        c, sn = math.cos(angle), math.sin(angle)
        M = np.dot(np.array([[c, -sn, 0.0], [sn, c, 0.0], [0.0, 0.0, 1.0]]), M)
    if args.pc_augm_mirror_prob > 0:
        if rnd.random() < args.pc_augm_mirror_prob / 2:
            M = np.dot(np.diag([-1.0, 1.0, 1.0]), M)
        if rnd.random() < args.pc_augm_mirror_prob / 2:
            M = np.dot(np.diag([1.0, -1.0, 1.0]), M)
    return M


def load_superpoints(store, fname, sp_ids, args, train, test_seed_offset=0, device_rng=False,
                     seed=0):
    """The cloud part of `loader` for the nodes `sp_ids` of one graph (ref: learning/spg.py:146-166).

    Returns (clouds_flag int64 [N] host array, clouds [Nv, F, L] device, clouds_global [Nv] device)
    — the reference's (clouds_flag, np.stack(clouds), np.concatenate(clouds_global)).
    `args`: ptn_minpts, ptn_npts, pc_xyznormalize, pc_attribs and, for train, pc_augm_scale,
    pc_augm_rot, pc_augm_mirror_prob, pc_augm_jitter.
    Host draws follow the reference exactly (numpy global state in training, RandomState(id+offset)
    in evaluation); with device_rng=True no per-point draw happens on the host."""
    if store.points is None:
        raise RuntimeError("SuperpointStore.finalize(device) has not been called")
    L = int(args.ptn_npts)
    cols = attrib_columns(args.pc_attribs, store.n_columns)
    flags, starts, counts, idx, mats, noise = [], [], [], [], [], []
    augment = bool(train)
    jitter = augment and bool(getattr(args, "pc_augm_jitter", 0))
    for s in sp_ids:
        n = store.count(fname, s)
        if n < args.ptn_minpts:
            flags.append(-1)
            continue
        flags.append(0)
        starts.append(store.start(fname, s))
        counts.append(n)
        if not device_rng:
            rs = np.random.random.__self__ if train else np.random.RandomState(seed=int(s) + test_seed_offset)
            idx.append(sample_indices(n, L, rs))
        if augment:
            mats.append(augment_matrix(args))
            if jitter and not device_rng:
                noise.append(np.clip(0.01 * np.random.randn(L, len(cols)), -0.05, 0.05).astype(np.float32))
    dev = store.points.device
    nv = len(starts)
    clouds = torch.empty((nv, len(cols), L), dtype=torch.float32, device=dev)
    diam = torch.empty((nv,), dtype=torch.float32, device=dev)
    if nv:
        ops.cloud_build(
            store.points, torch.tensor(starts, dtype=torch.int64).to(dev),
            torch.tensor(counts, dtype=torch.int32).to(dev),
            None if device_rng else torch.from_numpy(np.stack(idx).astype(np.int32)).to(dev),
            torch.tensor(cols, dtype=torch.int32).to(dev), L, bool(args.pc_xyznormalize),
            torch.from_numpy(np.stack(mats)).to(dev) if mats else None,
            torch.from_numpy(np.stack(noise)).to(dev) if noise else None,
            0.01 if (jitter and device_rng) else 0.0, 0.05, seed, clouds, diam)
    return np.array(flags), clouds, diam


class GraphStore(object):
    """Superpoint graphs of one or more files, resident on the device (the graph half of the reference's
    `loader`, learning/spg.py:106-143).

    `add(node_gt, node_gt_size, edges, edge_feats, name)` takes spg_reader's tuple in its order (after
    scaler01); `finalize(device)` uploads once.  Kept per vertex: the target row [node_gt | node_gt_size] (int64,
    spg_to_igraph's 't') and s = node_gt_size.sum(1) (int64); per edge: source and target (int32, file order) and
    the feature row (float32); per file: the spg_graph_build views of its stably target-sorted edges, whose target
    and source CSRs together are the undirected adjacency the neighbourhood BFS walks.  No batch writes to them.
    `add` validates on the host and raises as numpy would: IndexError for an edge id out of range, ValueError for
    inconsistent lengths, files of 2^31 vertices or more or a name added twice; TypeError for edge features that are
    not float32."""

    def __init__(self):
        self._host, self._files = {}, {}
        self.device = None

    def add(self, node_gt, node_gt_size, edges, edge_feats, name):
        if self.device is not None:
            raise RuntimeError("GraphStore.add after finalize")
        if name in self._host:
            raise ValueError("%s: a graph of this name was added already" % (name,))
        node_gt, node_gt_size = np.asarray(node_gt), np.asarray(node_gt_size)
        n = node_gt.shape[0]
        if n >= 2 ** 31:
            raise ValueError("%s: %d vertices; files of 2^31 vertices or more are not supported" % (name, n))
        if node_gt.ndim != 2 or node_gt_size.ndim != 2 or node_gt_size.shape[0] != n:
            raise ValueError("%s: node_gt %s and node_gt_size %s are not [n, 1] and [n, C]"
                             % (name, node_gt.shape, node_gt_size.shape))
        _inputs.check_ints(edges, "edges")
        edges = np.asarray(edges)
        if edges.ndim != 2 or edges.shape[1] != 2:
            raise ValueError("%s: edges must be [E, 2] (got shape %s)" % (name, edges.shape))
        fshape = _inputs.check_dtype(edge_feats, "edge_feats", "float32")
        if len(fshape) != 2 or fshape[0] != edges.shape[0]:
            raise ValueError("%s: edge_feats has shape %s for %d edges" % (name, tuple(fshape), edges.shape[0]))
        if edges.size and (int(edges.min()) < 0 or int(edges.max()) >= n):
            bad = int(edges.max()) if int(edges.max()) >= n else int(edges.min())
            raise IndexError("%s: index %d is out of bounds for axis 0 with size %d" % (name, bad, n))
        self._host[name] = dict(
            n=n, targets=np.concatenate([node_gt, node_gt_size], axis=1).astype(np.int64),
            s=node_gt_size.sum(1).astype(np.int64), src=edges[:, 0].astype(np.int32),
            tgt=edges[:, 1].astype(np.int32), feats=np.ascontiguousarray(edge_feats))
        return self

    def finalize(self, device):
        """Uploads every added file and builds its adjacency on the device."""
        device = torch.device(device)
        for name, h in self._host.items():
            order = np.argsort(h["tgt"], kind="stable")
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
            f = dict(name=name, n=h["n"], E=h["src"].size, targets=up(h["targets"]), s=up(h["s"]), src=up(h["src"]),
                     tgt=up(h["tgt"]), feats=up(h["feats"]))
            degs = up(np.bincount(h["tgt"], minlength=h["n"]).astype(np.int64))
            idxn = up(h["src"][order].astype(np.int64))
            views = ops.EccGraph.from_device(idxn, degs, n_in=h["n"], check=False).to(idxn.device)
            f["adjacency"] = {k: views[k] for k in ops.EccGraph.GRAPH_FIELDS}
            self._files[name] = f
        self._host = {}
        self.device = device
        return self

    def file(self, name):
        if self.device is None:
            raise RuntimeError("GraphStore.finalize(device) has not been called")
        return self._files[name]


def graph_draws(n, train, args):
    """The sampling draws of `loader` for a graph of n vertices (ref: learning/spg.py:134-143), from Python's
    global `random` in the reference's order: the permutation (perm[i] = new id of vertex i) when
    0 < hardcutoff < n, then the centres (new ids) when 0 < nneigh < n.  Returns (perm or None, centres or None,
    cut): cut > 0 is k_big_enough's k, which keeps everything unless it is below the sub-graph's size."""
    perm = centres = None
    if not train:
        return perm, centres, 0
    hc, nn = int(args.spg_augm_hardcutoff), int(args.spg_augm_nneigh)
    if 0 < hc < n:
        perm = list(range(n))
        random.shuffle(perm)
    if 0 < nn < n:
        centres = random.sample(range(n), k=nn)
    return perm, centres, max(hc, 0)


def load_batch(gstore, cstore, names, train, args, test_seed_offset=0, device_rng=False, seed=0):
    """`loader(entry, train, args, db_path, test_seed_offset)` for every name, then `eccpc_collate`
    (ref: learning/spg.py:130-193).  Returns (targets, GIs, (clouds_meta, clouds_flag, clouds, clouds_global))
    with targets int64 [N, 2 + C], clouds and clouds_global on the device, GIs = [GraphConvInfo] whose idxn,
    degs_gpu and edgefeats are on the device with its kernel views built.

    Graph by graph, as the reference: the sampling draws, the selection on the device, one read-back of the counts
    and kept ids (none when the whole graph is kept; one copy of the whole [2 + n] word array, so one
    synchronisation, where reading the count first would take two), then load_superpoints' cloud draws for graphs with edges.
    Graphs without edges are dropped; the collate's exceptions are the reference's (RuntimeError when no graph
    has an edge, TypeError when the first has none or a graph with edges has no cloud).

    device_rng=True draws every random choice of the batch on the device instead (Philox4x32-10 keyed by `seed`;
    the reference's distributions, not its streams; Python's `random` and numpy's global state are not touched) and
    builds the batch with one synchronisation whatever the number of graphs: every graph's draws, selection and
    cloud table are enqueued first, then one read-back of the counts, kept ids and flags sizes the rest.  Training
    streams are keyed by (seed, position in `names`, superpoint or vertex), evaluation clouds by (seed,
    id + test_seed_offset); see include/spg_b200.h spg_batch_draw for the counter layout.  KeyError for a kept
    superpoint of a graph with edges that the store lacks, as store.count raises on the host path."""
    if device_rng:
        return _load_batch_device(gstore, cstore, names, train, args, test_seed_offset, seed)
    dev = gstore.device
    picks = []
    for name in names:
        f = gstore.file(name)
        n = f["n"]
        perm, centres, cut = graph_draws(n, train, args)
        if perm is None and centres is None and not 0 < cut < n:
            new_index = edge_pos = kept_dev = None
            n_kept, n_edges, ids = n, f["E"], list(range(n))
        else:
            to_dev = lambda a: None if a is None else torch.tensor(a, dtype=torch.int32).to(dev)
            new_index, edge_pos, out = ops.batch_select(
                f["src"], f["tgt"], f["adjacency"], f["s"], to_dev(perm), to_dev(centres),
                int(args.spg_augm_order), int(args.ptn_minpts), cut)
            host = out.cpu().numpy()
            n_kept, n_edges = int(host[0]), int(host[1])
            ids, kept_dev = host[2:2 + n_kept].tolist(), out[2:2 + n_kept]
        clouds = load_superpoints(cstore, name, ids, args, train, test_seed_offset) if n_edges else None
        picks.append((f, new_index, edge_pos, kept_dev, n_kept, n_edges, ids, clouds))
    kept, targets, gi = _collate(dev, picks, [p[7][1].shape[0] if p[5] else 0 for p in picks])
    clouds_meta = ["{}.{:d}".format(p[0]["name"], v) for p in kept for v in p[6]]
    clouds_flag = torch.from_numpy(np.concatenate([p[7][0] for p in kept]))
    clouds = torch.cat([p[7][1] for p in kept], 0)
    clouds_global = torch.cat([p[7][2] for p in kept], 0)
    return targets, [gi], (clouds_meta, clouds_flag, clouds, clouds_global)


def _collate(dev, picks, n_clouds):
    """eccpc_collate's graph part (ref: learning/spg.py:178-193).  picks: per graph (file, new_index, edge_pos,
    kept ids on the device, n_kept, n_edges, kept ids, clouds); new_index None: the whole graph is kept.  n_clouds:
    per graph, its clouds of at least ptn_minpts points.  Raises the collate's exceptions; returns (the picks of the
    graphs with edges, targets, GraphConvInfo)."""
    from .spg_ecc import GraphConvInfo

    kept = [p for p in picks if p[5]]
    if not kept:
        raise RuntimeError("torch.cat(): expected a non-empty list of Tensors")
    if not picks[0][5]:
        raise TypeError("object of type 'NoneType' has no len()")
    if any(c == 0 for p, c in zip(picks, n_clouds) if p[5]):
        raise TypeError("expected np.ndarray (got list)")
    feats_w = {p[0]["feats"].shape[1] for p in kept}
    cols = {p[0]["targets"].shape[1] for p in kept}
    if len(feats_w) > 1 or len(cols) > 1:
        raise ValueError("the graphs of a batch have different edge-feature or target widths")
    N, E = sum(p[4] for p in kept), sum(p[5] for p in kept)
    i64 = dict(dtype=torch.int64, device=dev)
    edge_index, degs = torch.empty((2, E), **i64), torch.empty(N, **i64)
    edgefeats = torch.empty((E, feats_w.pop()), dtype=torch.float32, device=dev)
    targets = torch.empty((N, cols.pop()), **i64)
    vo = eo = 0
    for f, new_index, edge_pos, kept_ids, n_kept, n_edges, _, _ in kept:
        if new_index is None:
            i32 = dict(dtype=torch.int32, device=dev)
            new_index = kept_ids = torch.arange(n_kept, **i32)
            edge_pos = torch.arange(n_edges + 1, **i32)
        ops.batch_edges(f["src"], f["tgt"], new_index, edge_pos, kept_ids, n_kept, n_edges, vo, f["feats"],
                        f["targets"], edge_index[0, eo:eo + n_edges], edge_index[1, eo:eo + n_edges],
                        degs[vo:vo + n_kept], edgefeats[eo:eo + n_edges], targets[vo:vo + n_kept])
        vo, eo = vo + n_kept, eo + n_edges
    return kept, targets, GraphConvInfo.from_device_arrays(edge_index, degs, edgefeats)


def _load_batch_device(gstore, cstore, names, train, args, test_seed_offset, seed):
    """load_batch(device_rng=True): graph draws, selection and cloud table of every graph, one read-back, then the
    cloud draws, the clouds and the collated edges."""
    if cstore.points is None:
        raise RuntimeError("SuperpointStore.finalize(device) has not been called")
    dev = gstore.device
    files = [gstore.file(name) for name in names]
    hc, nn = (int(args.spg_augm_hardcutoff), int(args.spg_augm_nneigh)) if train else (0, 0)
    order, minpts = int(args.spg_augm_order) if train else 0, int(args.ptn_minpts)
    n_all = sum(f["n"] for f in files)
    fo = 2 * len(files) + n_all
    # read back at once: every graph's [2 + n] selection words, then every graph's [n] clouds_flag
    words = torch.empty(fo + n_all, dtype=torch.int32, device=dev)
    valid, count = torch.empty(n_all, dtype=torch.int32, device=dev), torch.empty(n_all, dtype=torch.int32, device=dev)
    first_row, key = torch.empty(n_all, dtype=torch.int64, device=dev), torch.empty(n_all, dtype=torch.int64, device=dev)
    graphs, o, v = [], 0, 0
    for b, f in enumerate(files):
        n = f["n"]
        perm, centres = ops.batch_draw(n, seed, b, 0 < hc < n, nn if 0 < nn < n else 0, dev)
        out = words[o:o + 2 + n]
        new_index, edge_pos, _ = ops.batch_select(f["src"], f["tgt"], f["adjacency"], f["s"], perm, centres, order,
                                                  minpts, max(hc, 0), out=out)
        sl = slice(v, v + n)
        ops.batch_cloud_flags(out, b, cstore.device_index(f["name"]), minpts, words[fo + v:fo + v + n], valid[sl],
                              first_row[sl], count[sl], key[sl])
        graphs.append((f, new_index, edge_pos, out, o, v))
        o, v = o + 2 + n, v + n
    start, n_points, cloud_key = ops.batch_clouds(valid, first_row, count, key)
    host = words.cpu().numpy()
    picks = []
    for f, new_index, edge_pos, out, o, v in graphs:
        n_kept, n_edges = int(host[o]), int(host[o + 1])
        ids, flags = host[o + 2:o + 2 + n_kept], host[fo + v:fo + v + n_kept]
        if n_edges and (flags == -2).any():
            raise KeyError((f["name"], int(ids[np.argmax(flags == -2)])))
        picks.append((f, new_index, edge_pos, out[2:2 + n_kept], n_kept, n_edges, ids, flags))
    n_clouds = [int((p[7] == 0).sum()) for p in picks]
    kept, targets, gi = _collate(dev, picks, n_clouds)
    nv, L = sum(c for p, c in zip(picks, n_clouds) if p[5]), int(args.ptn_npts)
    cols = attrib_columns(args.pc_attribs, cstore.n_columns)
    clouds = torch.empty((nv, len(cols), L), dtype=torch.float32, device=dev)
    clouds_global = torch.empty((nv,), dtype=torch.float32, device=dev)
    if nv:
        aug = (float(args.pc_augm_scale), int(args.pc_augm_rot), float(args.pc_augm_mirror_prob),
               bool(getattr(args, "pc_augm_jitter", 0))) if train else (0.0, 0, 0.0, False)
        idx, mats, noise = ops.batch_cloud_draw(cloud_key, n_points, nv, L, len(cols), seed, train, test_seed_offset,
                                                *aug)
        ops.cloud_build(cstore.points, start, n_points, idx, cstore.device_columns(cols), L,
                        bool(args.pc_xyznormalize), mats, noise, 0.0, 0.05, 0, clouds, clouds_global)
    clouds_meta = [p[0]["name"] + "." + str(v) for p in kept for v in p[6].tolist()]
    clouds_flag = torch.from_numpy(np.concatenate([p[7] for p in kept]).astype(np.int64))
    return targets, [gi], (clouds_meta, clouds_flag, clouds, clouds_global)
