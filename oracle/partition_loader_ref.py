"""Numpy restatement of the learned partition's batch loader (ref: supervized_partition/graph_processing.py:347-436
`graph_loader` for the learned-embedding branch, :439-472 `graph_collate`, :534-546 `augment_cloud_whole`).

The random draws and the sub-graph masks are inputs instead of numpy's global state and libply_c: per file,
`draws = (ref_index or None, M float32 [3, 3] or None, noise_xyz float32 [n, 3] or None, noise_rgb or None)`
(noise already clipped and cast, as the reference adds it) and `mask` (boolean [n]) or None.  Everything else is
the reference's numpy code, step for step.  Test infrastructure only.
"""
import os

import numpy as np


def augment(xyz, rgb, draws):
    """augment_cloud_whole with explicit draws; xyz is not modified (the reference's file is re-read every step)."""
    ri, M, nx, nr = draws
    xyz = np.array(xyz, dtype=np.float32)
    if M is not None:
        ref_point = xyz[ri, :3]
        ref_point[2] = 0  # a view: vertex ri's own z becomes 0 (graph_processing.py:537-538)
        xyz = np.matmul(xyz[:, :3] - ref_point, M) + ref_point
    if nx is not None:
        xyz = xyz + nx
        if nr is not None:
            rgb = np.clip(rgb + nr, -1, 1)
    return xyz, rgb


def graph_loader(name, arrays, train, args, draws=None, mask=None, augmented=None):
    """One file: the tuple graph_loader returns (numpy clouds / clouds_global / objects instead of tensors).
    augmented=(xyz, rgb) stands for rgb / 255 and the augmentation (the rest is built from it)."""
    xyz, rgb, edg_source, edg_target, is_transition, local_geometry, labels, objects, elevation, xyn = arrays
    short_name = name.split(os.sep)[-2] + "/" + name.split(os.sep)[-1]
    rgb = rgb / 255
    n_ver = np.shape(xyz)[0]
    selected_ver = np.full((n_ver,), True, dtype="?")
    if augmented is not None:
        xyz, rgb = augmented
    elif train:
        xyz, rgb = augment(xyz, rgb, draws)
    if train and (0 < args.max_ver_train < n_ver):
        selected_ver = np.asarray(mask).astype("?")
        selected_edg = (selected_ver[edg_source] * selected_ver[edg_target]).astype("?")
        new_ver_index = -np.ones((n_ver,), dtype=int)
        new_ver_index[selected_ver.nonzero()] = range(selected_ver.sum())
        edg_source = new_ver_index[edg_source[selected_edg]]
        edg_target = new_ver_index[edg_target[selected_edg]]
        is_transition = is_transition[selected_edg]
        labels = labels[selected_ver, ]
        objects = objects[selected_ver, ]
        elevation = elevation[selected_ver]
        xyn = xyn[selected_ver, ]
    nei = local_geometry[selected_ver, :args.k_nn_local].astype("int64")
    clouds = xyz[nei, ]
    diameters = np.sqrt(clouds.var(1).sum(1))
    clouds = (clouds - xyz[selected_ver, np.newaxis, :]) / (diameters[:, np.newaxis, np.newaxis] + 1e-10)
    if args.use_rgb:
        clouds = np.concatenate([clouds, rgb[nei, ]], axis=2)
    clouds = clouds.transpose([0, 2, 1])
    clouds_global = diameters[:, None]
    if "e" in args.global_feat:
        clouds_global = np.hstack((clouds_global, elevation[:, None]))
    if "rgb" in args.global_feat:
        clouds_global = np.hstack((clouds_global, rgb[selected_ver, ]))
    if "XY" in args.global_feat:
        clouds_global = np.hstack((clouds_global, xyn))
    if "xy" in args.global_feat:
        clouds_global = np.hstack((clouds_global, xyz[selected_ver, :2]))
    nei = np.array([0])
    xyz = xyz[selected_ver, ]
    return (short_name, edg_source, edg_target, is_transition, labels, objects.astype("int64"),
            np.ascontiguousarray(clouds), clouds_global, nei, xyz)


def graph_collate(batch):
    """graph_collate on numpy arrays (torch.cat -> np.concatenate); objects offset by the running sum of each
    file's max (not max + 1)."""
    short_name, edg_source, edg_target, is_transition, labels, objects, clouds, clouds_global, nei, xyz = \
        list(zip(*batch))
    n_batch = len(short_name)
    batch_ver_size_cumsum = np.array([c.shape[0] for c in labels]).cumsum()
    batch_n_edg_cumsum = np.array([c.shape[0] for c in edg_source]).cumsum()
    batch_n_objects_cumsum = np.array([c.max() for c in objects]).cumsum()
    clouds = np.concatenate(clouds, 0)
    clouds_global = np.concatenate(clouds_global, 0)
    xyz = np.vstack(xyz)
    is_transition = np.concatenate(is_transition, 0)
    labels = np.vstack(labels)
    edg_source = np.hstack(edg_source)
    edg_target = np.hstack(edg_target)
    nei = np.vstack(nei)
    objects = np.concatenate(objects, 0)
    for i_batch in range(1, n_batch):
        edg_source[batch_n_edg_cumsum[i_batch - 1]:batch_n_edg_cumsum[i_batch]] += int(batch_ver_size_cumsum[i_batch - 1])
        edg_target[batch_n_edg_cumsum[i_batch - 1]:batch_n_edg_cumsum[i_batch]] += int(batch_ver_size_cumsum[i_batch - 1])
        objects[batch_ver_size_cumsum[i_batch - 1]:batch_ver_size_cumsum[i_batch], ] += int(batch_n_objects_cumsum[i_batch - 1])
        non_valid = (nei[batch_ver_size_cumsum[i_batch - 1]:batch_ver_size_cumsum[i_batch], ] == -1).nonzero()
        nei[batch_ver_size_cumsum[i_batch - 1]:batch_ver_size_cumsum[i_batch], ] += int(batch_ver_size_cumsum[i_batch - 1])
        nei[batch_ver_size_cumsum[i_batch - 1] + non_valid[0], non_valid[1]] = -1
    return short_name, edg_source, edg_target, is_transition, labels, objects, (clouds, clouds_global, nei), xyz


def load_batch(files, names, train, args, draws=None, masks=None):
    """graph_loader for every name (files: name -> read_structure tuple), then graph_collate."""
    return graph_collate([graph_loader(nm, files[nm], train, args, draws[b] if draws else None,
                                       masks[b] if masks else None) for b, nm in enumerate(names)])
