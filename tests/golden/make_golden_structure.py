"""Writes tests/golden/structure.npz: the reference's own learned-partition structure of three seeded clouds.

    SPG_REFERENCE=<superpoint_graph checkout> python tests/golden/make_golden_structure.py

The graph comes from the reference's unmodified partition/graphs.py `compute_graph_nn_2` (sklearn's kd-tree k-NN;
current scipy has no `Delaunay.vertices`, so the alias is patched in, and the simplices it used are captured and
stored).  The rest is the SOURCE TEXT of supervized_partition/graph_processing.py:144-190, read from the checkout and
executed unmodified, after :126 for s3dis's pruned objects and with :136-138's values for sema3d without labels, in
a namespace holding:
  * `libply_c.connected_comp`: oracle/partition_ref.py's stand-in on scipy's connected_components (cutoff 0,
    components numbered by their smallest vertex, as boost numbers them); the mask it gets is (is_transition ==
    0).astype('uint8'), so the signed-char reading does not arise;
  * `RANSACRegressor`: sklearn's;
  * args.compute_geof = 0 (libply_c.compute_geof is not built here; the device's geof is spg_geometry's).

Clouds (float32, <= 2 500 points):
  room   floor, walls, a table top and a cylinder
  scan   a ground plane and a wall whose density falls off with the range from the sensor (long Delaunay edges)
  dup    a small room with a tenth of its points duplicated exactly
Cases cover s3dis, vkitti and sema3d without labels, use_voronoi on and off, plane_model on and off.  The RANSAC
plane (coef_, intercept_) of every plane case is stored with it.  Versions are recorded in `meta`.
"""
import json
import os
import sys
import textwrap
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT = os.path.join(HERE, "structure.npz")
SEED = 20261018
K_ADJ, K_LOCAL = 5, 10
N_LABELS, N_OBJECTS = 6, 9
# (case, cloud, dataset, use_voronoi, plane_model)
CASES = (("room_s3dis", "room", "s3dis", 0.0, 0),
         ("room_s3dis_vor", "room", "s3dis", 0.05, 1),
         ("scan_vkitti_vor", "scan", "vkitti", 1.0, 1),
         ("scan_vkitti", "scan", "vkitti", 0.0, 0),
         ("dup_sema3d_vor", "dup", "sema3d", 0.05, 0),
         ("dup_vkitti_vor", "dup", "vkitti", 0.05, 1))
# target_local_geometry is the cloud's stored `neighbors` (as uint32)
KEYS = ("source", "target", "distances", "is_transition", "labels", "objects", "elevation", "xyn")


def room(rng, n):
    m = n // 5
    parts = [np.c_[rng.uniform(0, 4, m), rng.uniform(0, 3, m), rng.normal(0, 0.003, m)],      # floor
             np.c_[rng.uniform(0, 4, m), np.zeros(m), rng.uniform(0, 2.5, m)],                # wall y = 0
             np.c_[np.zeros(m), rng.uniform(0, 3, m), rng.uniform(0, 2.5, m)],                # wall x = 0
             np.c_[rng.uniform(1.5, 2.7, m), rng.uniform(1, 1.8, m), np.full(m, 0.75)]]       # table top
    r = n - 4 * m
    a = rng.uniform(0, 2 * np.pi, r)
    parts.append(np.c_[3.3 + 0.2 * np.cos(a), 2.4 + 0.2 * np.sin(a), rng.uniform(0, 1.2, r)])  # cylinder
    return np.concatenate(parts).astype(np.float32)


def scan(rng, n):
    m = (3 * n) // 4
    rg = np.exp(rng.uniform(np.log(0.5), np.log(30.0), m))  # density ~ 1 / range^2 on the ground
    a = rng.uniform(0, 2 * np.pi, m)
    ground = np.c_[rg * np.cos(a), rg * np.sin(a), 0.02 * rg * np.cos(a) + rng.normal(0, 0.01, m)]
    w = n - m
    d = np.exp(rng.uniform(np.log(2.0), np.log(20.0), w))
    wall = np.c_[d, np.full(w, 5.0), rng.uniform(0, 3, w) * 2.0 / np.sqrt(d)]
    return np.concatenate([ground, wall]).astype(np.float32)


def dup(rng, n):
    base = room(rng, n - n // 10) * np.float32(0.5)
    return np.concatenate([base, base[rng.choice(len(base), n // 10, replace=False)]])


def clouds():
    rng = np.random.default_rng(SEED)
    out = {}
    for name, xyz in (("room", room(rng, 2000)), ("scan", scan(rng, 2500)), ("dup", dup(rng, 1200))):
        n = xyz.shape[0]
        # label and object histograms as prune returns them; labels follow height bands, objects space cells
        labels = rng.integers(0, 2, (n, N_LABELS + 1)).astype(np.uint32)
        labels[np.arange(n), 1 + (np.floor(xyz[:, 2] * 2).astype(np.int64) % N_LABELS)] += 3
        objects = rng.integers(0, 2, (n, N_OBJECTS + 1)).astype(np.uint32)
        cell = (np.floor(xyz[:, 0]).astype(np.int64) * 7 + np.floor(xyz[:, 1]).astype(np.int64)) % N_OBJECTS
        objects[np.arange(n), 1 + cell] += 4
        rgb = rng.integers(0, 256, (n, 3)).astype(np.uint8)
        out[name] = (xyz, rgb, labels, objects)
    return out


def block_source(ref):
    lines = open(os.path.join(ref, "supervized_partition", "graph_processing.py")).read().split("\n")
    return textwrap.dedent("\n".join(lines[143:190])), lines[125].strip()  # :144-190 and :126


def main():
    ref = os.environ.get("SPG_REFERENCE")
    if not ref:
        sys.exit("set SPG_REFERENCE to a superpoint_graph checkout")
    sys.path.insert(0, os.path.join(ref, "partition"))
    import scipy
    import scipy.spatial
    import sklearn
    from sklearn.linear_model import RANSACRegressor

    from oracle.partition_ref import connected_comp

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
    block, line126 = block_source(ref)
    assert block.startswith("n_ver = xyz.shape[0]") and "write_structure" not in block, block[:80]
    assert line126 == "objects = objects[:,1:].argmax(axis=1)+1", line126
    out, meta = {}, dict(numpy=np.__version__, scipy=scipy.__version__, sklearn=sklearn.__version__, seed=SEED,
                         k_nn_adj=K_ADJ, k_nn_local=K_LOCAL, cases=[])
    data = clouds()
    for name, (xyz, rgb, labels, objects) in data.items():
        out[name + ".xyz"], out[name + ".rgb"] = xyz, rgb
        out[name + ".labels"], out[name + ".objects"] = labels, objects
    for case, cloud, dataset, voronoi, plane in CASES:
        xyz, rgb, labels, objects = data[cloud]
        args = types.SimpleNamespace(k_nn_adj=K_ADJ, k_nn_local=K_LOCAL, use_voronoi=voronoi, compute_geof=0,
                                     plane_model=plane)
        ns = {"np": np, "args": args, "xyz": xyz, "labels": labels.copy(), "objects": objects.copy(),
              "dataset": dataset, "compute_graph_nn_2": graphs.compute_graph_nn_2, "RANSACRegressor": RANSACRegressor,
              "libply_c": types.SimpleNamespace(connected_comp=connected_comp), "print": lambda *a: None}
        ns["args"].dataset = dataset
        if dataset == "s3dis":
            exec(line126, ns)
        if dataset == "sema3d":  # :136-138, a cloud without a label file
            ns.update(has_labels=False, labels=np.array([0]), objects=np.array([0]), is_transition=np.array(False))
        captured.clear()
        exec(block, ns)
        if voronoi > 0:
            key = cloud + ".simplices"
            assert len(captured) == 1
            if key in out:
                assert np.array_equal(out[key], captured[0])
            out[key] = captured[0].astype(np.uint16)
        nb = ns["local_neighbors"].reshape(len(xyz), K_LOCAL)
        if cloud + ".neighbors" in out:
            assert np.array_equal(out[cloud + ".neighbors"], nb)
        out[cloud + ".neighbors"] = nb.astype(np.uint16)
        g = ns["graph_nn"]
        res = dict(source=g["source"], target=g["target"], distances=g["distances"], is_transition=ns["is_transition"],
                   labels=ns["labels"], objects=ns["objects"], elevation=ns["elevation"], xyn=ns["xyn"])
        for k in KEYS:
            out["%s.%s" % (case, k)] = np.asarray(res[k])
        if plane:
            est = ns["reg"].estimator_
            out[case + ".plane"] = np.r_[np.asarray(est.coef_, np.float64).reshape(-1),
                                         np.float64(est.intercept_)]
        meta["cases"].append(dict(case=case, cloud=cloud, dataset=dataset, use_voronoi=voronoi, plane_model=plane))
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
