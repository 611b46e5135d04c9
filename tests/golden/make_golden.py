"""Generates tests/golden/*.npz by running the UNMODIFIED reference (a superpoint_graph checkout) on CPU.

    SPG_REFERENCE=<path of the reference checkout> python tests/golden/make_golden.py

Every file is at most 1 MB.  When igraph is not installed, the reference's learning package imports with a stub module in
its place (only GraphConvInfo.set_batch touches igraph objects, and it is driven below with a
minimal duck-typed graph).  Everything stored is produced by reference code: the oracle
(oracle/*.py) and the CUDA path are both tested against these files.
"""
import json
import os
import sys
import types

import numpy as np
import torch

REF = os.environ["SPG_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))

sys.modules.setdefault("igraph", types.ModuleType("igraph"))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(REF, "learning"))
from learning import ecc, graphnet, modules, pointnet  # noqa: E402


def npy(t):
    return t.detach().cpu().numpy().copy()  # copy: state-dict views alias live buffers


def sd_np(module, prefix=""):
    return {prefix + k: npy(v) for k, v in module.state_dict().items()}


def save(name, **arrays):
    np.savez_compressed(os.path.join(OUT, name), **arrays)
    print("wrote", name, sum(a.nbytes for a in arrays.values() if hasattr(a, "nbytes")) // 1024, "KiB")


# ----------------------------------------------------------------------------- ECC function
def ecc_unit_fixture():
    """The reference's own unit-test scenario (learning/ecc/test_GraphConvModule.py:29-36,61-75)
    driven through .apply (the legacy call style of the file no longer runs)."""
    torch.manual_seed(11)
    np.random.seed(11)
    n, e, cin, cout = 20, 50, 10, 15
    degs = torch.LongTensor([5, 0, 15, 20, 10])
    idxn = torch.from_numpy(np.random.randint(n, size=e))
    x = torch.randn(n, cin, dtype=torch.float64)
    w = torch.randn(e, cin, cout, dtype=torch.float64)
    out30 = ecc.GraphConvFunction.apply(x, w, cin, cout, idxn, None, degs, degs, 30)
    out1 = ecc.GraphConvFunction.apply(x, w, cin, cout, idxn, None, degs, degs, 1)
    assert (out30 - out1).norm() < 1e-6
    # with edge-feature compaction
    w30 = torch.randn(30, cin, cout, dtype=torch.float64)
    idxe = torch.from_numpy(np.random.randint(30, size=e))
    oute = ecc.GraphConvFunction.apply(x, w30, cin, cout, idxn, idxe, degs, degs, 30)
    # vector filters incl. backward (runs unmodified on torch 2.x)
    xv = torch.randn(n, cin, dtype=torch.float64, requires_grad=True)
    wv = torch.randn(e, cin, dtype=torch.float64, requires_grad=True)
    outv = ecc.GraphConvFunction.apply(xv, wv, cin, cin, idxn, None, degs, degs, 30)
    gv = torch.randn(5, cin, dtype=torch.float64)
    outv.backward(gv)
    save("ecc_unit.npz", x=npy(x), w=npy(w), idxn=npy(idxn), degs=npy(degs), out=npy(out30),
         w30=npy(w30), idxe=npy(idxe), out_idxe=npy(oute), xv=npy(xv), wv=npy(wv), outv=npy(outv),
         gv=npy(gv), gxv=npy(xv.grad), gwv=npy(wv.grad))


def ecc_spg_shaped():
    torch.manual_seed(5)
    rng = np.random.default_rng(5)
    N, H = 100, 32
    degs_np = rng.integers(0, 4, size=N)  # (the [E, 32, 32] matrix filters keep the file under 1 MB)
    degs_np[[3, 17, 90]] = 0
    degs_np[40] = 37  # one heavy node
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn = torch.from_numpy(rng.integers(0, N, size=E).astype(np.int64))
    x = torch.randn(N, H, requires_grad=True)
    wv = torch.randn(E, H, requires_grad=True)
    out = ecc.GraphConvFunction.apply(x, wv, H, H, idxn, None, degs, degs, 1e20)
    g = torch.randn(N, H)
    out.backward(g)
    wm = torch.randn(E, H, H) * 0.2
    outm = ecc.GraphConvFunction.apply(x.detach(), wm, H, H, idxn, None, degs, degs, 1e20)
    save("ecc_spg.npz", x=npy(x), wv=npy(wv), idxn=npy(idxn), degs=npy(degs), out=npy(out),
         g=npy(g), gx=npy(x.grad), gw=npy(wv.grad), wm=npy(wm), outm=npy(outm))


# ------------------------------------------------------------------------------ GRUCellEx
def gru_cell():
    torch.manual_seed(7)
    for tag, ln, ig in (("", True, True), ("_plain", False, False)):
        cell = modules.GRUCellEx(32, 32, bias=True, layernorm=ln, ingate=ig)
        with torch.no_grad():
            cell.bias_ih.normal_(0, 0.3)
            cell.bias_hh.normal_(0, 0.3)
        x = torch.randn(50, 32, requires_grad=True)
        h = torch.randn(50, 32, requires_grad=True)
        hy = cell(x, h)
        g = torch.randn(50, 32)
        hy.backward(g)
        arrs = dict(x=npy(x), h=npy(h), hy=npy(hy), g=npy(g), gx=npy(x.grad), gh=npy(h.grad))
        arrs.update({"sd." + k: v for k, v in sd_np(cell).items()})
        arrs.update({"grad." + k: npy(p.grad) for k, p in cell.named_parameters()})
        save("gru%s.npz" % tag, **arrs)


# ------------------------------------------------------------------------------- PointNet
def pointnet_small():
    """Small widths, full training-mode forward/backward + eval forward after the update of the
    running statistics."""
    cfg = dict(nf_conv=[16, 16, 32], nf_fc=[32, 16, 8], nf_conv_stn=[8, 16], nf_fc_stn=[16, 8],
               nfeat=6, nfeat_stn=6)
    net = pointnet.PointNet(cfg["nf_conv"], cfg["nf_fc"], cfg["nf_conv_stn"], cfg["nf_fc_stn"],
                            cfg["nfeat"], cfg["nfeat_stn"], prelast_do=0)
    torch.manual_seed(3)
    with torch.no_grad():  # make the STN non-trivial (its projection is zero-initialised)
        net.stn.proj.weight.normal_(0, 0.2)
        net.stn.proj.bias.normal_(0, 0.2)
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
        net.convs[1].weight[::3] *= -1  # negative BN scales exercise the max-pool ordering
    sd0 = sd_np(net)
    B, L = 9, 24
    x = torch.randn(B, cfg["nfeat"], L) * 0.5
    xg = torch.rand(B) * 3
    net.train()
    out = net(x, xg)
    g = torch.randn_like(out)
    out.backward(g)
    grads = {"grad." + k: npy(p.grad) for k, p in net.named_parameters()}
    sd1 = sd_np(net)  # running stats after one training forward
    net.eval()
    out_eval = net(x, xg)
    T = net.stn(x[:, :cfg["nfeat_stn"], :])
    arrs = dict(x=npy(x), xg=npy(xg), out_train=npy(out), g=npy(g), out_eval=npy(out_eval),
                T_eval=npy(T), cfg=json.dumps(cfg))
    arrs.update({"sd0." + k: v for k, v in sd0.items()})
    arrs.update({"sd1." + k: v for k, v in sd1.items()})
    arrs.update(grads)
    save("pointnet_small.npz", **arrs)


# --------------------------------------------------------------------------- GraphNetwork
class _ES(object):
    def __init__(self, attrs):
        self._a = attrs

    def attributes(self):
        return list(self._a.keys())

    def __getitem__(self, idx):
        return _ES({k: [v[i] for i in idx] for k, v in self._a.items()})

    def get_attribute_values(self, a):
        return self._a[a]


class _Graph(object):
    """The subset of igraph.Graph that GraphConvInfo.set_batch uses."""

    def __init__(self, nv, edges, feats):
        self._nv, self._edges = nv, [tuple(int(v) for v in e) for e in edges]
        self.es = _ES({"f": [list(map(float, f)) for f in feats]})
        self.vs = list(range(nv))

    def get_edgelist(self):
        return self._edges

    def indegree(self, vs, loops=True):
        d = [0] * self._nv
        for _, t in self._edges:
            d[t] += 1
        return d

    def vcount(self):
        return self._nv


def _edge_feat_func(edgeattrs):
    return torch.from_numpy(np.asarray(edgeattrs["f"], dtype=np.float32)), None


def graph_conv_info():
    rng = np.random.default_rng(9)
    graphs, raw = [], {}
    for gi, (nv, ne) in enumerate(((7, 30), (12, 55))):
        edges = rng.integers(0, nv, size=(ne, 2))
        feats = rng.standard_normal((ne, 13)).astype(np.float32)
        graphs.append(_Graph(nv, edges, feats))
        raw["edges%d" % gi], raw["feats%d" % gi], raw["nv%d" % gi] = edges, feats, np.array(nv)
    info = ecc.GraphConvInfo(graphs, _edge_feat_func)
    idxn, idxe, degs, _, ef = info.get_buffers()
    assert idxe is None
    save("graph_conv_info.npz", idxn=npy(idxn), degs=npy(degs), edgefeats=npy(ef),
         edge_indexes=npy(info.get_pyg_buffers()), **raw)
    return info


def graph_networks():
    rng = np.random.default_rng(21)
    N = 60
    degs_np = rng.integers(0, 9, size=N)
    degs_np[[0, 31]] = 0
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn = torch.from_numpy(rng.integers(0, N, size=E).astype(np.int64))
    ef = torch.from_numpy(rng.standard_normal((E, 13)).astype(np.float32))
    labels = torch.from_numpy(rng.integers(0, 13, size=N).astype(np.int64))
    labels[[5, 6]] = -100
    cw = torch.from_numpy(rng.uniform(0.5, 2.0, size=13).astype(np.float32))

    class GI(object):  # what RNNGraphConvModule reads from a GraphConvInfo
        def get_buffers(self):
            return idxn, None, degs, None, ef

        def get_pyg_buffers(self):
            return None

    base = dict(idxn=npy(idxn), degs=npy(degs), edgefeats=npy(ef), labels=npy(labels), cw=npy(cw))
    for tag, config, bwd in (("vv", "gru_3_1_1_1_0,f_13", True), ("cat", "gru_2,f_8", True),
                             ("mat", "gru_2_0,f_13", False)):
        torch.manual_seed(13)
        net = graphnet.GraphNetwork(config, 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0,
                                    cuda=False)
        net.set_info([GI()], False)
        sd0 = sd_np(net)
        emb = torch.randn(N, 32, requires_grad=True)
        net.train()
        out = net(emb)
        arrs = dict(base)
        arrs.update(emb=npy(emb), out_train=npy(out), config=config)
        arrs.update({"sd0." + k: v for k, v in sd0.items()})
        if bwd:
            ncls = out.shape[1]
            loss = torch.nn.functional.cross_entropy(out, labels.clamp(max=ncls - 1) if ncls < 13 else labels,
                                                     weight=cw[:ncls])
            loss.backward()
            arrs.update(loss=npy(loss), gemb=npy(emb.grad))
            arrs.update({"grad." + k: npy(p.grad) for k, p in net.named_parameters()})
        net.eval()
        arrs.update(out_eval=npy(net(emb.detach())))
        save("graphnet_%s.npz" % tag, **arrs)


def shards():
    cases = []
    for degs, lim in (([5, 0, 15, 20, 10], 1), ([5, 0, 15, 20, 10], 30), ([5, 0, 15, 20, 10], 50),
                      ([5, 0, 15, 20, 10], 1e10), ([1, 2, 3, 4, 5, 6, 7], 7), ([0, 0, 3], 2)):
        cases.append({"degs": degs, "limit": lim,
                      "shards": [list(s) for s in ecc.get_edge_shards(np.array(degs), lim)]})
    with open(os.path.join(OUT, "edge_shards.json"), "w") as f:
        json.dump(cases, f, indent=1)
    print("wrote edge_shards.json")


def train_steps():
    """Two full reference training steps (main.py:199-213) on a tiny model: pins loss values and a
    checksum of the updated parameters."""
    from types import SimpleNamespace
    rng = np.random.default_rng(33)
    N, L, F = 40, 16, 6
    degs_np = rng.integers(0, 7, size=N)
    degs_np[[2]] = 0
    E = int(degs_np.sum())
    degs = torch.from_numpy(degs_np.astype(np.int64))
    idxn = torch.from_numpy(rng.integers(0, N, size=E).astype(np.int64))
    ef = torch.from_numpy(rng.standard_normal((E, 13)).astype(np.float32))
    flag = torch.zeros(N, dtype=torch.long)
    flag[[4, 9, 30]] = -1
    nv = int((flag == 0).sum())
    clouds = torch.from_numpy(rng.standard_normal((nv, F, L)).astype(np.float32) * 0.4)
    cglob = torch.from_numpy(rng.uniform(0.1, 3.0, size=nv).astype(np.float32))
    labels = torch.from_numpy(rng.integers(0, 13, size=N).astype(np.int64))
    labels[[7]] = -100

    class GI(object):
        def get_buffers(self):
            return idxn, None, degs, None, ef

        def get_pyg_buffers(self):
            return None

    model = torch.nn.Module()
    torch.manual_seed(1)
    model.ecc = graphnet.GraphNetwork("gru_3_1_1_1_0,f_13", 8, [13, 16, 32, 16], True, 0, 2, 1e20,
                                      use_pyg=0, cuda=False)
    model.ptn = pointnet.PointNet([16, 16, 32], [32, 16, 8], [8, 16], [16, 8], F, F, prelast_do=0)
    sd_ecc0, sd_ptn0 = sd_np(model.ecc), sd_np(model.ptn)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    emb = pointnet.CloudEmbedder(SimpleNamespace(cuda=False, ptn_mem_monger=0))
    model.ecc.set_info([GI()], False)
    model.train()
    losses, outs = [], []
    for _ in range(2):
        opt.zero_grad()
        e = emb.run(model, None, flag, clouds, cglob)
        out = model.ecc(e)
        loss = torch.nn.functional.cross_entropy(out, labels)
        loss.backward()
        for p in model.parameters():
            p.grad.data.clamp_(-1, 1)
        opt.step()
        losses.append(float(loss))
        outs.append(npy(out))
    arrs = dict(idxn=npy(idxn), degs=npy(degs), edgefeats=npy(ef), flag=npy(flag), clouds=npy(clouds),
                cglob=npy(cglob), labels=npy(labels), losses=np.array(losses), out0=outs[0],
                out1=outs[1])
    arrs.update({"ecc0." + k: v for k, v in sd_ecc0.items()})
    arrs.update({"ptn0." + k: v for k, v in sd_ptn0.items()})
    arrs.update({"ecc2." + k: v for k, v in sd_np(model.ecc).items()})
    arrs.update({"ptn2." + k: v for k, v in sd_np(model.ptn).items()})
    save("train_steps.npz", **arrs)



# ----------------------------------------------------------------------------- batch loader
class _FakeH5File(dict):
    """Stand-in for h5py.File over an in-memory {dataset name: ndarray}: `load_superpoint` only
    does `hf['<id>']`, `.shape[0]` and `[:]` (learning/spg.py:200-205)."""
    store = {}

    def __init__(self, fname, mode="r"):
        super(_FakeH5File, self).__init__(_FakeH5File.store[fname])


def _import_reference_spg():
    for name in ("transforms3d", "h5py"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["h5py"].File = _FakeH5File
    from learning import spg  # noqa: E402
    return spg


def loader_clouds():
    """The reference's own `load_superpoint` (evaluation mode: per-superpoint RandomState, no
    augmentation) on synthetic parsed superpoints of 1..700 points, two attribute selections."""
    from types import SimpleNamespace
    spg = _import_reference_spg()
    rng = np.random.default_rng(31)
    counts = [1, 39, 40, 41, 127, 128, 129, 300, 700, 64]
    parsed = {}
    for sid, n in enumerate(counts):
        P = rng.standard_normal((n, 15)).astype(np.float32)
        P[:, :3] = P[:, :3] * rng.uniform(0.2, 4.0) + rng.uniform(-20, 20, size=3)
        P[:, 11:14] = rng.uniform(0, 1, size=(n, 3))
        parsed["%d" % sid] = P
    _FakeH5File.store = {"mem.h5": parsed}
    out = {"counts": np.array(counts)}
    for sid, P in parsed.items():
        out["P%s" % sid] = P
    cases = (("s3dis", "xyzrgbelpsvXYZ", 1, 128, 40, 0), ("sema", "xyzrgbelpsv", 1, 128, 40, 3),
             ("nonorm", "xyzelpsv", 0, 64, 1, 0))
    for tag, attribs, norm, npts, minpts, offset in cases:
        args = SimpleNamespace(ptn_minpts=minpts, ptn_npts=npts, pc_xyznormalize=norm, pc_attribs=attribs)
        flags, clouds, diams = [], [], []
        for sid in range(len(counts)):
            cloud, diam = spg.load_superpoint(args, "mem.h5", sid, False, offset)
            flags.append(0 if cloud is not None else -1)
            if cloud is not None:
                clouds.append(cloud.T)
                diams.append(diam)
        out["%s_flag" % tag] = np.array(flags)
        out["%s_clouds" % tag] = np.stack(clouds)
        out["%s_global" % tag] = np.concatenate(diams)
        out["%s_cfg" % tag] = np.array([norm, npts, minpts, offset])
        out["%s_attribs" % tag] = np.array(attribs)
    save("loader_clouds.npz", **out)


def metrics_confusion():
    """learning/metrics.py ConfusionMatrix driven as eval()/eval_final() do (main.py:257-262,297-305)."""
    from learning import metrics
    rng = np.random.default_rng(17)
    C, out = 13, {}
    cm = metrics.ConfusionMatrix(C)
    for b, n in enumerate((50, 1, 333)):
        o = rng.standard_normal((n, C)).astype(np.float32)
        o[::7, 3] = o[::7, 5] = 9.0  # ties: argmax keeps the first
        tvec = rng.integers(0, 400, size=(n, C)).astype(np.int64)
        tvec[rng.random((n, C)) < 0.6] = 0
        t = tvec.argmax(1)
        t[rng.random(n) < 0.2] = -100
        idx = t != -100
        cm.count_predicted_batch(tvec[idx, ...], np.argmax(o[idx, :], 1))
        out["o%d" % b], out["t%d" % b], out["tvec%d" % b] = o, t, tvec
        out["pred%d" % b] = np.argmax(o, 1)
    out["cm"] = cm.confusion_matrix.copy()
    out["oa"] = np.array(cm.get_overall_accuracy())
    out["miou"] = np.array(cm.get_average_intersection_union())
    out["iou"] = np.array(cm.get_intersection_union_per_class())
    out["macc"] = np.array(cm.get_mean_class_accuracy())
    # multi-sample averaging of eval_final (main.py:292-295)
    samples = [rng.standard_normal((40, C)).astype(np.float32) for _ in range(10)]
    out["ms_samples"] = np.stack(samples, 0)
    out["ms_mean"] = np.mean(np.stack(samples, 0), 0)
    save("metrics_confusion.npz", **out)


def upsampling():
    """partition/provider.py `interpolate_labels` / `reduced_labels2full`: the module as a whole does not
    import under Python 3.12 (mixed tab/space indentation at provider.py:417, plyfile / libply_c absent), so
    the SOURCE TEXT of the two functions is read from the reference checkout at generation time and executed
    unmodified in a namespace holding what they use (numpy, scikit-learn's NearestNeighbors)."""
    from sklearn.neighbors import NearestNeighbors
    lines = open(os.path.join(REF, "partition", "provider.py")).read().split("\n")

    def grab(name):
        start = next(i for i, l in enumerate(lines) if l.startswith("def %s(" % name))
        end = next(i for i in range(start + 1, len(lines)) if lines[i].startswith("#---") or lines[i].startswith("def "))
        return "\n".join(lines[start:end])

    ns = {"np": np, "NearestNeighbors": NearestNeighbors}
    exec(grab("reduced_labels2full"), ns)
    exec(grab("interpolate_labels"), ns)
    provider = types.SimpleNamespace(**{k: ns[k] for k in ("reduced_labels2full", "interpolate_labels")})
    rng = np.random.default_rng(23)
    n, m = 700, 5000
    xyz = rng.uniform(0, 10, size=(n, 3)).astype(np.float32)
    xyz_up = np.concatenate([xyz + rng.normal(0, 0.05, size=xyz.shape).astype(np.float32),
                             rng.uniform(-1, 11, size=(m - n, 3)).astype(np.float32)], 0)
    logits = rng.standard_normal((n, 13)).astype(np.float32)
    lab_up = provider.interpolate_labels(xyz_up, xyz, logits, 0)
    hard = rng.integers(0, 13, size=n)
    lab_up_hard = provider.interpolate_labels(xyz_up, xyz, hard, 0)
    # superpoint labels -> points
    comp_of = rng.integers(0, 40, size=n)
    components = [np.nonzero(comp_of == c)[0] for c in range(40)]
    labels_red = rng.integers(0, 13, size=40).astype(np.uint8)
    full = provider.reduced_labels2full(labels_red, components, n)
    save("upsampling.npz", xyz=xyz, xyz_up=xyz_up, logits=logits, lab_up=np.asarray(lab_up, dtype=np.int64),
         hard=hard.astype(np.int64), lab_up_hard=np.asarray(lab_up_hard, dtype=np.int64), comp_of=comp_of.astype(np.int64),
         labels_red=labels_red, full=full)


if __name__ == "__main__":
    torch.set_num_threads(4)
    if sys.argv[1:] == ["loader"]:  # only the section-8(f) fixtures
        loader_clouds()
        metrics_confusion()
        upsampling()
        sys.exit(0)
    ecc_unit_fixture()
    ecc_spg_shaped()
    gru_cell()
    pointnet_small()
    graph_conv_info()
    graph_networks()
    shards()
    train_steps()
    loader_clouds()
    metrics_confusion()
    upsampling()
