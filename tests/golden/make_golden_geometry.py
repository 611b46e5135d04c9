"""Writes tests/golden/geometry.npz: the reference's own k-NN graphs of six synthetic clouds.

    SPG_REFERENCE=<superpoint_graph checkout> python tests/golden/make_golden_geometry.py

Imports the reference's unmodified partition/graphs.py (scikit-learn's kd-tree, numpy.matlib) and runs
`compute_graph_nn(xyz, k1)` and `compute_graph_nn_2(xyz, k1, k2)` at (k1, k2) = (10, 45) (partition/partition.py:
146-152) and (5, 20) (supervized_partition/graph_processing.py:146,176) on seeded clouds:

  room     floor, walls, a table top and a cylinder (a surface cloud)
  lidar    a ground plane and a wall whose density falls off with the range from the sensor
  lattice  a regular 7 x 7 x 6 lattice of spacing 0.25 (exact distance ties)
  line     points on one line
  blob     60 coincident points (more than k + 2) among scattered ones
  offset   a room-like cloud moved by 10^4 m

`compute_geof` (partition/ply_c/ply_c.cpp:384-462) has no golden: libply_c needs Boost.Python and Eigen to build.
Its truth is the float64 restatement in oracle/geometry_ref.py.  The scikit-learn, scipy and numpy versions are
recorded in `meta`; the ids are stored as uint16 (every cloud has fewer than 2^16 points) to keep the file small.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "geometry.npz")
PAIRS = ((10, 45), (5, 20))


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
    return (np.concatenate(parts) + offset).astype(np.float32)


def lidar(rng, n):
    m = (3 * n) // 4
    rg = np.exp(rng.uniform(np.log(0.5), np.log(30.0), m))  # density ~ 1 / range^2 on the ground
    a = rng.uniform(0, 2 * np.pi, m)
    ground = np.c_[rg * np.cos(a), rg * np.sin(a), rng.normal(0, 0.01, m)]
    w = n - m
    d = np.exp(rng.uniform(np.log(2.0), np.log(20.0), w))
    wall = np.c_[d, np.full(w, 5.0), rng.uniform(0, 3, w) * 2.0 / np.sqrt(d)]
    return np.concatenate([ground, wall]).astype(np.float32)


def lattice():
    g = np.stack(np.meshgrid(np.arange(7), np.arange(7), np.arange(6), indexing="ij"), -1).reshape(-1, 3)
    return (0.25 * g).astype(np.float32)


def line(rng, n):
    t = rng.uniform(-5, 5, n)
    return np.c_[1 + t, 2 - 0.5 * t, 0.3 * t].astype(np.float32)


def blob(rng, n):
    b = np.tile(np.array([[1.0, 2.0, 3.0]]), (60, 1))
    return np.concatenate([b, rng.normal([1, 2, 3], 0.5, (n - 60, 3))]).astype(np.float32)


def clouds():
    rng = np.random.default_rng(20261017)
    return [("room", room(rng, 400)), ("lidar", lidar(rng, 400)), ("lattice", lattice()), ("line", line(rng, 150)),
            ("blob", blob(rng, 200)), ("offset", room(rng, 300, offset=np.array([1e4, -1e4, 1e4])))]


def main():
    ref = os.environ.get("SPG_REFERENCE")
    if not ref:
        sys.exit("set SPG_REFERENCE to a superpoint_graph checkout")
    sys.path.insert(0, os.path.join(ref, "partition"))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import graphs  # the reference's unmodified partition/graphs.py
    import scipy
    import sklearn

    out, meta = {}, dict(sklearn=sklearn.__version__, scipy=scipy.__version__, numpy=np.__version__,
                         seed=20261017, pairs=PAIRS, clouds=[])
    for name, xyz in clouds():
        assert xyz.shape[0] < 2 ** 16
        out[name + ".xyz"] = xyz
        meta["clouds"].append(dict(name=name, n=int(xyz.shape[0])))
        for k1, k2 in PAIRS:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                g1 = graphs.compute_graph_nn(xyz, k1)
                g2, target2 = graphs.compute_graph_nn_2(xyz, k1, k2)
            tag = "%s.%d_%d" % (name, k1, k2)
            assert np.array_equal(g1["source"], g2["source"]) and g1["source"].dtype == np.uint32
            out[tag + ".source"] = g2["source"].astype(np.uint16)
            out[tag + ".target"] = g2["target"].astype(np.uint16)
            out[tag + ".distances"] = g2["distances"]
            out[tag + ".target2"] = target2.astype(np.uint16)
            out[tag + ".nn.target"] = g1["target"].astype(np.uint16)
            out[tag + ".nn.distances"] = g1["distances"]
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
