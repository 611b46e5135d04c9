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

from . import ops

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
        return self

    def count(self, fname, sp_id):
        return self._index[(fname, int(sp_id))][1]

    def start(self, fname, sp_id):
        return self._index[(fname, int(sp_id))][0]


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
