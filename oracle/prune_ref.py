"""numpy restatement of the reference's voxel pruning (partition/ply_c/ply_c.cpp:149-380 `prune`) and of its
chunked use in partition/provider.py:250-303 (`read_semantic3d_format`).

Every step rounds as the C++ does: the bins are float32 numpy arithmetic, the voxels are ordered by their first point
(np.unique's return_index), and the positions are sequential fp32 sums in point order (np.add.at adds in index
order), so the outputs are the reference's bit for bit.  Returns numpy arrays with the reference's dtypes: xyz
float32 [m, 3], rgb uint8 [m, 3], labels uint32 [m, n_labels + 1], objects uint32 [m, n_objects + 1].
"""
import numpy as np

__all__ = ["prune", "prune_chunked", "bins"]


def bins(xyz, voxel_size):
    """uint32 [n, 3]: floor((x - x_min) / voxel) in float32 (ply_c.cpp:306-331); ValueError for a bin >= 2^32."""
    xyz = np.asarray(xyz, dtype=np.float32)
    v = np.float32(voxel_size)
    b = np.floor((xyz - xyz.min(0)) / v)
    if not (b < np.float32(2.0 ** 32)).all():
        raise ValueError("a voxel bin of 2^32 or more")
    return b.astype(np.uint32)


def prune(xyz, voxel_size, rgb, labels, objects, n_labels, n_objects):
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    rgb = np.asarray(rgb)
    n = xyz.shape[0]
    if n == 0 or not np.isfinite(xyz).all():
        raise ValueError("an empty or non-finite cloud")
    b = bins(xyz, voxel_size).astype(np.int64)
    span = b.max(0) + 1
    if float(span[0]) * float(span[1]) * float(span[2]) < 2.0 ** 62:  # one integer key per voxel: a faster unique
        key = (b[:, 0] * span[1] + b[:, 1]) * span[2] + b[:, 2]
        _, first, inverse = np.unique(key, return_index=True, return_inverse=True)
    else:
        _, first, inverse = np.unique(b, axis=0, return_index=True, return_inverse=True)
    inverse = inverse.reshape(-1)
    rank = np.empty(len(first), np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(first))  # insertion order: by first point
    row = rank[inverse]
    m = len(first)
    acc = np.zeros((m, 3), np.float32)
    np.add.at(acc, row, xyz)
    count = np.bincount(row, minlength=m).astype(np.uint32)
    fcount = count.astype(np.float32)[:, None]
    col = np.zeros((m, 3), np.uint32)
    np.add.at(col, row, rgb.astype(np.uint32))
    out_xyz = acc / fcount
    out_rgb = (col.astype(np.float32) / fcount).astype(np.uint8)
    out_labels = np.zeros((m, n_labels + 1), np.uint32)
    out_objects = np.zeros((m, n_objects + 1), np.uint32)
    if n_labels > 0:
        lab = np.asarray(labels).reshape(-1).astype(np.int64)
        if (lab < 0).any() or (lab > n_labels).any():
            raise IndexError("a label outside [0, n_labels]")
        np.add.at(out_labels, (row, lab), 1)
        if n_objects > 0:
            obj = np.asarray(objects).reshape(-1).astype(np.int64)
            if (obj < 0).any() or (obj > n_objects).any():
                raise IndexError("an object outside [0, n_objects]")
            np.add.at(out_objects, (row, obj), 1)
    return out_xyz, out_rgb, out_labels, out_objects


def prune_chunked(xyz, voxel_size, rgb, labels, objects, n_labels, n_objects, chunk_rows):
    """Every chunk of chunk_rows points pruned on its own, the four outputs stacked in chunk order."""
    n = len(xyz)
    parts = []
    for s in range(0, n, chunk_rows):
        sl = slice(s, min(n, s + chunk_rows))
        parts.append(prune(xyz[sl], voxel_size, rgb[sl], labels[sl] if n_labels > 0 else labels,
                           objects[sl] if n_labels > 0 and n_objects > 0 else objects, n_labels, n_objects))
    return tuple(np.vstack([p[k] for p in parts]) for k in range(4))
