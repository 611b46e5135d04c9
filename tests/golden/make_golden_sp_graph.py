"""Writes tests/golden/sp_graph.npz: the reference's own superpoint graphs of three seeded clouds.

    SPG_REFERENCE=<superpoint_graph checkout> python tests/golden/make_golden_sp_graph.py

Imports the reference's unmodified partition/graphs.py and runs `compute_sp_graph(xyz, d_max, in_component,
components, labels, n_labels)` (partition/partition.py:184) on every cloud, labels mode and d_max:

  room    floor, walls, a table top and a cylinder (a surface cloud)
  lidar   a ground plane and a wall whose density falls off with the range from the sensor
  offset  a room-like cloud moved by 10^4 m

Cut pursuit cannot be built here, so the partitions are stand-ins: voxel cells of the cloud, numbered in cell order
as uint32 (libcp returns in_component as uint32, cutpursuit.cpp:22), plus crafted components appended to the cloud:
one point repeated (one unique row), two distinct points with a duplicate, a cell with duplicated points, a collinear
segment and a lone point next to it (superedges of a single vertex pair).

Labels: none (`[]`), 1-D integer labels in 0..n_labels + 1 (the value n_labels + 1 falls outside every bin of the
reference's histogram) and a 2-D histogram [n, n_labels + 1].  d_max: 0 and a value that cuts some pairs.

Current scipy has no `Delaunay.vertices` (removed in 1.11; it is `.simplices`), so the alias is patched in before
the call.  The simplices the reference used are captured and stored (uint16: every cloud has fewer than 2^16
points), so the tests do not depend on the local scipy's triangulation.  The numpy and scipy versions are recorded in
`meta`.  The labels-independent outputs are stored once per (cloud, d_max) and sp_labels once per (cloud, labels).
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "sp_graph.npz")
SEED = 20261017
N_LABELS = 5
D_MAX = {"room": 0.3, "lidar": 1.0, "offset": 0.3}
VOXEL = {"room": 0.6, "lidar": 3.0, "offset": 0.6}
LABEL_MODES = ("none", "1d", "hist")
SP_KEYS = ("sp_centroids", "sp_length", "sp_surface", "sp_volume", "sp_point_count")
SE_KEYS = ("source", "target", "se_delta_mean", "se_delta_std", "se_delta_norm", "se_delta_centroid",
           "se_length_ratio", "se_surface_ratio", "se_volume_ratio", "se_point_count_ratio")


def room(rng, n, offset=0.0):
    parts = []
    m = n // 5
    parts.append(np.c_[rng.uniform(0, 4, m), rng.uniform(0, 3, m), np.zeros(m)])          # floor
    parts.append(np.c_[rng.uniform(0, 4, m), np.zeros(m), rng.uniform(0, 2.5, m)])        # wall y = 0
    parts.append(np.c_[np.zeros(m), rng.uniform(0, 3, m), rng.uniform(0, 2.5, m)])        # wall x = 0
    parts.append(np.c_[rng.uniform(1.5, 2.7, m), rng.uniform(1, 1.8, m), np.full(m, 0.75)])  # table top
    r = n - 4 * m
    a = rng.uniform(0, 2 * np.pi, r)
    parts.append(np.c_[3.3 + 0.2 * np.cos(a), 2.4 + 0.2 * np.sin(a), rng.uniform(0, 1.2, r)])  # cylinder
    return np.concatenate(parts) + offset


def lidar(rng, n):
    m = (3 * n) // 4
    rg = np.exp(rng.uniform(np.log(0.5), np.log(30.0), m))  # density ~ 1 / range^2 on the ground
    a = rng.uniform(0, 2 * np.pi, m)
    ground = np.c_[rg * np.cos(a), rg * np.sin(a), rng.normal(0, 0.01, m)]
    w = n - m
    d = np.exp(rng.uniform(np.log(2.0), np.log(20.0), w))
    wall = np.c_[d, np.full(w, 5.0), rng.uniform(0, 3, w) * 2.0 / np.sqrt(d)]
    return np.concatenate([ground, wall])


def partition(rng, base, cell, centre):
    """Voxel-cell components of `base`, then the crafted components around `centre` (all float32)."""
    xyz = base.astype(np.float32)
    vox = np.floor((xyz.astype(np.float64) - xyz.min(0)) / cell).astype(np.int64)
    _, comp = np.unique(vox, axis=0, return_inverse=True)
    comp = comp.reshape(-1)
    dup = rng.choice(np.nonzero(comp == comp[0])[0], 3)  # duplicated points inside a voxel component
    xyz = np.concatenate([xyz, xyz[dup]])
    comp = np.concatenate([comp, comp[dup]])
    c = np.asarray(centre, np.float64)
    crafted = [
        np.tile(c + [0.05, 0.05, 0.5], (4, 1)),                                           # one repeated point
        np.array([c + [0.3, 0.1, 0.45], c + [0.32, 0.14, 0.52], c + [0.3, 0.1, 0.45]]),   # two distinct + a dup
        c + [0.6, 0.2, 0.3] + np.linspace(0, 1, 12)[:, None] * [0.4, -0.2, 0.1],          # collinear
        (c + [1.05, 0.05, 0.37])[None],                                                   # a lone point
    ]
    n_com = int(comp.max()) + 1
    for i, pts in enumerate(crafted):
        xyz = np.concatenate([xyz, pts.astype(np.float32)])
        comp = np.concatenate([comp, np.full(len(pts), n_com + i)])
    return xyz, comp.astype(np.uint32)


def clouds():
    rng = np.random.default_rng(SEED)
    out = []
    for name, base, centre in (("room", room(rng, 1500), (1.0, 1.0, 0.0)),
                               ("lidar", lidar(rng, 2000), (3.0, 3.0, 0.0)),
                               ("offset", room(rng, 1000, offset=np.array([1e4, -1e4, 1e4])),
                                (1e4 + 1.0, -1e4 + 1.0, 1e4))):
        xyz, comp = partition(rng, base, VOXEL[name], centre)
        n = xyz.shape[0]
        lab1 = rng.integers(0, N_LABELS + 2, n).astype(np.uint8)
        hist = rng.integers(0, 4, (n, N_LABELS + 1)).astype(np.uint32)
        out.append((name, xyz, comp, {"none": [], "1d": lab1, "hist": hist}))
    return out


def main():
    ref = os.environ.get("SPG_REFERENCE")
    if not ref:
        sys.exit("set SPG_REFERENCE to a superpoint_graph checkout")
    sys.path.insert(0, os.path.join(ref, "partition"))
    import scipy
    import scipy.spatial

    scipy.spatial.Delaunay.vertices = property(lambda s: s.simplices)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import graphs  # the reference's unmodified partition/graphs.py

    captured = []

    def delaunay(points):
        tri = scipy.spatial.Delaunay(points)
        captured.append(tri.simplices.copy())
        return tri

    graphs.Delaunay = delaunay
    out, meta = {}, dict(scipy=scipy.__version__, numpy=np.__version__, seed=SEED, n_labels=N_LABELS,
                         d_max=D_MAX, label_modes=LABEL_MODES, clouds=[])
    for name, xyz, comp, labels in clouds():
        assert xyz.shape[0] < 2 ** 16
        n_com = int(comp.max()) + 1
        components = [np.nonzero(comp == c)[0] for c in range(n_com)]
        out[name + ".xyz"] = xyz
        out[name + ".in_component"] = comp
        out[name + ".labels.1d"] = labels["1d"]
        out[name + ".labels.hist"] = labels["hist"]
        meta["clouds"].append(dict(name=name, n=int(xyz.shape[0]), n_com=n_com))
        simplices = None
        for d_max in (0.0, D_MAX[name]):
            for mode in LABEL_MODES:
                captured.clear()
                g = graphs.compute_sp_graph(xyz, d_max, comp, components, labels[mode], N_LABELS)
                s = captured[0]
                if simplices is None:
                    simplices = s
                    out[name + ".simplices"] = s.astype(np.uint16)
                assert np.array_equal(s, simplices)
                tag = "%s.%g" % (name, d_max)
                for k in SP_KEYS + SE_KEYS:
                    if mode == LABEL_MODES[0]:
                        out[tag + "." + k] = g[k]
                    else:
                        assert np.array_equal(out[tag + "." + k], g[k], equal_nan=True), (tag, k)
                key = "%s.sp_labels.%s" % (name, mode)
                if mode != "none":
                    assert key not in out or np.array_equal(out[key], g["sp_labels"])
                    out[key] = g["sp_labels"]
                else:
                    assert isinstance(g["sp_labels"], list) and not g["sp_labels"]
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
