"""The learned partition's training batches built on the device: `graph_loader` for every file of a batch followed by
`graph_collate` (ref: supervized_partition/graph_processing.py:347-472, `augment_cloud_whole` :534-546), for the
learned-embedding branch (`ver_value` containing 'ptn' or equal to 'xyz').

    from superpoint_graph_b200.spg_partition_loader import PartitionStore, load_batch

    store = PartitionStore()
    store.add("Area_1/office_1.h5", *read_structure(path, False))   # read_structure's tuple, in its order
    store.finalize(device)                                            # one upload; the files stay resident
    fname, edg_source, edg_target, is_transition, labels, objects, (clouds, clouds_global, nei), xyz = \\
        load_batch(store, names, train, args)

The reference reads every file again at every step, builds the [N, 6, k] local clouds in numpy and uploads them
(480 B per vertex at k_nn_local = 20).  Here the per-file arrays live in HBM once and the kernels of
csrc/partition_loader.cu write the collated batch; the host only makes the per-file random draws (the reference
vertex and angle of the rotation, the jitter noise unless device_rng=True) and the sub-graph choice.  With the same
numpy seed the batch is the reference's bit for bit, except the rotation, which the reference hands to BLAS.

Outputs are CUDA tensors: edges int64, is_transition uint8, labels / objects int64 (the reference: labels as read,
usually uint32), clouds float32 [N, 3 + 3 use_rgb, k], clouds_global float32 [N, G], xyz float32 [N, 3]; `fname`
and the `nei` placeholder are as the reference gives them.  DESIGN.md §4 lists what is mirrored on purpose.
"""
import math
import os

import numpy as np
import torch

from . import ops

__all__ = ["PartitionStore", "load_batch", "rotation_matrix", "host_draws", "global_columns"]

_INT32_MAX = 2 ** 31 - 1


def _rows(a, n, what, width=None):
    a = np.asarray(a)
    if a.shape[0] != n or (width is not None and (a.ndim != 2 or a.shape[1] != width)):
        raise ValueError("%s has shape %s for %d vertices" % (what, a.shape, n))
    return a


def _int32(a, what):
    a = np.asarray(a)
    if a.size and (int(a.min()) < -_INT32_MAX - 1 or int(a.max()) > _INT32_MAX):
        raise ValueError("%s does not fit in int32" % what)
    return np.ascontiguousarray(a, dtype=np.int32)


def _ids(a, n, what):
    a = np.asarray(a)
    if a.size and (int(a.min()) < 0 or int(a.max()) >= n):
        raise IndexError("%s: index %d is out of bounds for %d vertices"
                         % (what, int(a.max()) if int(a.max()) >= n else int(a.min()), n))
    return np.ascontiguousarray(a, dtype=np.int32)


class PartitionStore(object):
    """The per-file arrays of `read_structure` (graph_processing.py:224-247), resident on the device.

    Kept per vertex: xyz, rgb (as read, 0..255), elevation, xyn in float32 (36 B), the neighbour ids of
    `local_geometry` in int32 (4 B per column), labels in int32 (4 B per column) and objects in int32 (4 B): with
    30 neighbour columns and 14 label columns, 216 B per vertex.  Per edge: source and target in int32 and
    is_transition in uint8 (9 B).  No batch ever writes to these arrays.  `add` validates on the host once and
    raises as numpy would: IndexError for an edge or neighbour id out of range, ValueError for inconsistent
    lengths, files of 2^31 vertices or more, or values that do not fit in int32."""

    def __init__(self):
        self._host, self._files = {}, {}
        self.floats = self.ints = self.bytes = None
        self.device = None

    def add(self, name, xyz, rgb, edg_source, edg_target, is_transition, local_geometry, labels, objects, elevation,
            xyn):
        if self.floats is not None:
            raise RuntimeError("PartitionStore.add after finalize")
        xyz = np.asarray(xyz)
        n = xyz.shape[0]
        if n >= 2 ** 31:
            raise ValueError("%s: %d vertices; files of 2^31 vertices or more are not supported" % (name, n))
        _rows(xyz, n, "xyz", 3)
        rgb = _rows(rgb, n, "rgb", 3)
        elevation = _rows(np.asarray(elevation).reshape(-1), n, "elevation")
        xyn = _rows(xyn, n, "xyn", 2)
        labels = np.asarray(labels)
        if labels.ndim != 2:
            raise ValueError("labels must be [n_ver, n_columns] (got shape %s)" % (labels.shape,))
        _rows(labels, n, "labels")
        objects = _rows(np.asarray(objects).reshape(-1), n, "objects")
        local_geometry = np.asarray(local_geometry)
        if local_geometry.ndim != 2:
            raise ValueError("local_geometry must be the [n_ver, k] neighbour ids (ver_value 'ptn' or 'xyz')")
        _rows(local_geometry, n, "local_geometry")
        src, tgt = np.asarray(edg_source).reshape(-1), np.asarray(edg_target).reshape(-1)
        is_tr = np.asarray(is_transition).reshape(-1)
        if src.shape != tgt.shape or is_tr.shape != src.shape:
            raise ValueError("%s: %d sources, %d targets, %d is_transition" % (name, src.size, tgt.size, is_tr.size))
        self._host[name] = dict(
            n=n, E=src.size, K=local_geometry.shape[1], C=labels.shape[1],
            floats=np.concatenate([np.asarray(xyz, np.float32).reshape(-1), np.asarray(rgb, np.float32).reshape(-1),
                                   np.asarray(elevation, np.float32), np.asarray(xyn, np.float32).reshape(-1)]),
            ints=np.concatenate([_ids(src, n, "edg_source"), _ids(tgt, n, "edg_target"),
                                 _ids(local_geometry, n, "local_geometry").reshape(-1),
                                 _int32(labels, "labels").reshape(-1), _int32(objects, "objects")]),
            tr=np.ascontiguousarray(is_tr, dtype=np.uint8), src=src, tgt=tgt)
        return self

    def finalize(self, device):
        """Uploads every added file: one float32, one int32 and one uint8 array."""
        device = torch.device(device)
        fo = io = bo = 0
        for name, h in self._host.items():
            self._files[name] = dict(n=h["n"], E=h["E"], K=h["K"], C=h["C"], fo=fo, io=io, bo=bo,
                                     src_host=h["src"], tgt_host=h["tgt"])
            fo, io, bo = fo + h["floats"].size, io + h["ints"].size, bo + h["tr"].size
        cat = lambda key, dt: (np.concatenate([h[key] for h in self._host.values()]) if self._host
                               else np.zeros(0, dt))
        self.floats = torch.from_numpy(cat("floats", np.float32)).to(device)
        self.ints = torch.from_numpy(cat("ints", np.int32)).to(device)
        self.bytes = torch.from_numpy(cat("tr", np.uint8)).to(device)
        self.device = device
        self._host = {}
        for f in self._files.values():
            self._views(f)
        return self

    def _views(self, f):
        n, E, K, C = f["n"], f["E"], f["K"], f["C"]
        fl, it = self.floats.narrow(0, f["fo"], 9 * n), self.ints.narrow(0, f["io"], 2 * E + n * (K + C + 1))
        f["xyz"], f["rgb"] = fl[:3 * n].view(n, 3), fl[3 * n:6 * n].view(n, 3)
        f["elevation"], f["xyn"] = fl[6 * n:7 * n], fl[7 * n:].view(n, 2)
        f["src"], f["tgt"] = it[:E], it[E:2 * E]
        o = 2 * E
        f["geometry"] = it[o:o + n * K].view(n, K)
        f["labels"] = it[o + n * K:o + n * (K + C)].view(n, C)
        f["objects"] = it[o + n * (K + C):]
        f["is_transition"] = self.bytes.narrow(0, f["bo"], E)

    def file(self, name):
        if self.floats is None:
            raise RuntimeError("PartitionStore.finalize(device) has not been called")
        return self._files[name]

    def resident_bytes(self):
        return sum(t.numel() * t.element_size() for t in (self.floats, self.ints, self.bytes) if t is not None)


def rotation_matrix(angle):
    """transforms3d.axangles.axangle2mat([0, 0, 1], angle).astype('f4') (graph_processing.py:539), Rodrigues'
    formula term by term with the axis (0, 0, 1)."""
    x, y, z = 0.0, 0.0, 1.0
    c, s = math.cos(angle), math.sin(angle)
    C = 1.0 - c
    return np.array([[x * x * C + c, x * y * C - z * s, x * z * C + y * s],
                     [y * x * C + z * s, y * y * C + c, y * z * C - x * s],
                     [z * x * C - y * s, z * y * C + x * s, z * z * C + c]]).astype("f4")


def host_draws(n, args, use_rgb, device_rng=False):
    """The draws of augment_cloud_whole (graph_processing.py:534-546) for one file of n vertices, from numpy's
    global state in the reference's order: randint, uniform, the xyz normals, the rgb normals.  Returns
    (ref_index or None, M float32 [3, 3] or None, noise_xyz float32 [n, 3] or None, noise_rgb or None);
    device_rng leaves the normals to the device."""
    ri = M = nx = nr = None
    if args.pc_augm_rot:
        ri = np.random.randint(n)
        M = rotation_matrix(np.random.uniform(0, 2 * math.pi))
    if args.pc_augm_jitter and not device_rng:
        sigma, clip = 0.002, 0.005
        nx = np.clip(sigma * np.random.standard_normal((n, 3)), -1 * clip, clip).astype(np.float32)
        if use_rgb:
            nr = np.clip(sigma * np.random.standard_normal((n, 3)), -1 * clip, clip).astype(np.float32)
    return ri, M, nx, nr


def global_columns(global_feat):
    """(flags, width) of clouds_global by the reference's substring tests (graph_processing.py:403-411)."""
    flags, width = 0, 1
    for key, flag, w in (("e", ops.LPL_GLOBAL_E, 1), ("rgb", ops.LPL_GLOBAL_RGB, 3), ("XY", ops.LPL_GLOBAL_XYN, 2),
                         ("xy", ops.LPL_GLOBAL_XY, 2)):
        if key in global_feat:
            flags, width = flags | flag, width + w
    return flags, width


def _learned(args):
    if args.ver_value in ("geof", "geofrgb"):
        raise ValueError("ver_value %r: the device loader serves the learned-embedding branch only (ver_value "
                         "containing 'ptn', or 'xyz'); use the reference's graph_loader" % args.ver_value)
    if not ("ptn" in args.ver_value or args.ver_value == "xyz"):
        raise ValueError("ver_value %r is not a learned-embedding value" % args.ver_value)


def _subgraph_mask(f, args, b, selected):
    if selected is not None and selected[b] is not None:
        m = np.asarray(selected[b])
        if m.shape != (f["n"],):
            raise ValueError("selected[%d] has shape %s for %d vertices" % (b, m.shape, f["n"]))
        return m.astype(bool)
    try:
        from partition.ply_c import libply_c
    except ImportError:
        try:
            import libply_c
        except ImportError:
            raise RuntimeError("sub-sampling a file of %d vertices to max_ver_train = %d needs the reference's "
                               "`libply_c.random_subgraph` (partition/ply_c); build it, or pass selected= (one boolean "
                               "vertex mask per file)" % (f["n"], int(args.max_ver_train)))
    _, ver = libply_c.random_subgraph(f["n"], f["src_host"].astype("uint32"), f["tgt_host"].astype("uint32"),
                                      int(args.max_ver_train))
    return np.asarray(ver).astype(bool)


def load_batch(store, names, train, args, selected=None, device_rng=False, seed=0):
    """graph_loader(name, train, args) for every name, then graph_collate (ref: graph_processing.py:347-472).

    args: ver_value, k_nn_local, use_rgb, global_feat, and for train pc_augm_rot, pc_augm_jitter, max_ver_train.
    selected: optional list of one boolean vertex mask per file, used where the reference sub-samples (train and
    0 < max_ver_train < n_ver) in place of libply_c.random_subgraph.  device_rng: the jitter normals come from
    Philox on the device, keyed by `seed` and the file's position in the batch.  One device-to-host copy per
    batch when a file is sub-sampled (the kept edge counts, which size the edge outputs); none otherwise."""
    _learned(args)
    files = [store.file(nm) for nm in names]
    short = tuple(nm.split(os.sep)[-2] + "/" + nm.split(os.sep)[-1] for nm in names)
    B = len(files)
    dev = store.device
    use_rgb = bool(args.use_rgb)
    Fch = 3 + 3 * use_rgb
    gflags, G = global_columns(args.global_feat)
    ks = {min(int(args.k_nn_local), f["K"]) for f in files}
    Cs = {f["C"] for f in files}
    if len(ks) > 1 or len(Cs) > 1:
        raise ValueError("the files of a batch have different neighbour or label widths")
    k, C = ks.pop() if ks else int(args.k_nn_local), Cs.pop() if Cs else 0
    rot = bool(train) and bool(args.pc_augm_rot)
    jitter = bool(train) and bool(args.pc_augm_jitter)
    # host draws and sub-graph masks, file by file in batch order (the reference's order)
    draws, masks = [], []
    for b, f in enumerate(files):
        draws.append(host_draws(f["n"], args, use_rgb, device_rng) if train else (None, None, None, None))
        sub = bool(train) and 0 < args.max_ver_train < f["n"]
        masks.append(_subgraph_mask(f, args, b, selected) if sub else None)
    n_sel = [int(m.sum()) if m is not None else f["n"] for m, f in zip(masks, files)]
    i64 = dict(dtype=torch.int64, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    # small per-batch parameters: the rotation of every file (one upload), the kept vertex counts
    rot_dev = None
    if rot:
        rot_dev = torch.from_numpy(np.stack([d[1].reshape(-1) for d in draws]) if B else np.zeros((0, 9), "f4")).to(dev)
    need_aug = rot or jitter
    counts = torch.tensor(n_sel, **i64)
    if any(m is not None for m in masks):
        mask_dev = torch.from_numpy(np.concatenate([m.astype(np.uint8) for m in masks if m is not None])).to(dev)
    if jitter and not device_rng:
        noise_xyz = torch.from_numpy(np.concatenate([d[2] for d in draws])).to(dev)
        noise_rgb = torch.from_numpy(np.concatenate([d[3] for d in draws])).to(dev) if use_rgb else None
    n_tot = sum(f["n"] for f in files)
    if need_aug:
        aug_xyz = torch.empty((n_tot, 3), dtype=torch.float32, device=dev)
        aug_rgb = torch.empty((n_tot, 3), dtype=torch.float32, device=dev)
    object_max = torch.empty(max(B, 1), **i32)
    sel, new_index, edge_pos = [None] * B, [None] * B, [None] * B
    vo, mo = 0, 0
    for b, f in enumerate(files):
        n = f["n"]
        if need_aug:
            nx = noise_xyz[vo:vo + n] if (jitter and not device_rng) else None
            nr = noise_rgb[vo:vo + n] if (jitter and not device_rng and use_rgb) else None
            ops.lp_augment(f["xyz"], f["rgb"], rot_dev[b] if rot else None, draws[b][0] if rot else 0, nx, nr,
                           jitter and device_rng, jitter and use_rgb, 0.002, 0.005, seed, b, aug_xyz[vo:vo + n],
                           aug_rgb[vo:vo + n])
        if masks[b] is not None:
            new_index[b], edge_pos[b] = torch.empty(n + 1, **i32), torch.empty(f["E"] + 1, **i32)
            sel[b] = torch.empty(max(n_sel[b], 1), **i32)
            ops.lp_subgraph_select(mask_dev[mo:mo + n], f["objects"], f["src"], f["tgt"], new_index[b], sel[b],
                                   edge_pos[b], object_max[b])
            mo += n
        else:
            ops.lp_subgraph_select(None, f["objects"], f["src"], f["tgt"], None, None, None, object_max[b])
        vo += n
    # the one synchronisation: kept edge counts of the sub-sampled files
    n_edg = [f["E"] for f in files]
    sub = [b for b in range(B) if masks[b] is not None]
    if sub:
        kept = torch.cat([edge_pos[b][files[b]["E"]:] for b in sub]).cpu().tolist()
        for b, c in zip(sub, kept):
            n_edg[b] = int(c)
    obj_off = torch.empty(max(B, 1), **i64)
    ops.lp_object_offsets(object_max[:B], counts, obj_off[:B])
    N, E = sum(n_sel), sum(n_edg)
    edg_source, edg_target = torch.empty(E, **i64), torch.empty(E, **i64)
    is_transition = torch.empty(E, dtype=torch.uint8, device=dev)
    labels, objects = torch.empty((N, C), **i64), torch.empty(N, **i64)
    clouds = torch.empty((N, Fch, k), dtype=torch.float32, device=dev)
    clouds_global = torch.empty((N, G), dtype=torch.float32, device=dev)
    xyz = torch.empty((N, 3), dtype=torch.float32, device=dev)
    vo, ro, eo = 0, 0, 0
    for b, f in enumerate(files):
        n, ns, ne = f["n"], n_sel[b], n_edg[b]
        if ne:
            ops.lp_subgraph_edges(f["src"], f["tgt"], f["is_transition"], new_index[b], edge_pos[b], ro,
                                  edg_source[eo:eo + ne], edg_target[eo:eo + ne], is_transition[eo:eo + ne])
        xs, rs = (aug_xyz[vo:vo + n], aug_rgb[vo:vo + n]) if need_aug else (f["xyz"], f["rgb"])
        ops.lp_local_clouds(xs, rs, not need_aug, f["geometry"], k, sel[b], ns, f["elevation"], f["xyn"],
                            f["labels"], f["objects"], obj_off[b:b + 1], use_rgb, gflags, clouds[ro:ro + ns],
                            clouds_global[ro:ro + ns], xyz[ro:ro + ns], labels[ro:ro + ns], objects[ro:ro + ns])
        vo, ro, eo = vo + n, ro + ns, eo + ne
    nei = _collate_nei(n_sel)
    return short, edg_source, edg_target, is_transition, labels, objects, (clouds, clouds_global, nei), xyz


def _collate_nei(n_sel):
    """graph_collate's `nei` (:459,468-470): np.vstack of the per-file np.array([0]) placeholders (:428), with the
    collate's offsets applied to the rows its vertex ranges happen to cover."""
    nei = np.vstack([np.array([0]) for _ in n_sel]) if n_sel else np.zeros((0, 1), dtype=np.int64)
    cs = np.array(n_sel).cumsum()
    for i in range(1, len(n_sel)):
        non_valid = (nei[cs[i - 1]:cs[i], ] == -1).nonzero()
        nei[cs[i - 1]:cs[i], ] += int(cs[i - 1])
        nei[cs[i - 1] + non_valid[0], non_valid[1]] = -1
    return nei
