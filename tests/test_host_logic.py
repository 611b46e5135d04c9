"""CPU: host-side logic of the product (no kernels are launched): the C-ABI library and its header,
graph bookkeeping (bit-exact integer outputs), the model_config parser / state-dict contract,
the drop-in module aliases, the synthetic generator."""
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name), allow_pickle=False)
    return {k: z[k] for k in z.files}


# --------------------------------------------------------------------------------- C-ABI
def test_library_exports_every_declared_symbol():
    from superpoint_graph_b200 import _lib
    protos = _lib.parse_header()
    assert len(protos) >= 30
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for name in protos:
        assert hasattr(dll, name), "missing export %s" % name
    L = _lib.lib()
    assert L.spg_version() >= 100
    assert b"not supported" in L.spg_error_string(-2)
    assert L.spg_prof_num_kernels() > 20
    names = {L.spg_prof_kernel_name(i).decode() for i in range(L.spg_prof_num_kernels())}
    assert {"ecc_vv_fwd", "ecc_mat_fwd", "gru_cell_fwd", "gemm_f32", "clamp_adam"} <= names


def test_header_cites_reference_for_every_compute_entry_point():
    text = open(os.path.join(ROOT, "include", "spg_b200.h")).read()
    assert text.count("ref:") >= 12
    assert 'extern "C"' in text and "torch" not in text.lower().replace("pytorch", "")


def test_cuda_sources_target_sm90a_only():
    from superpoint_graph_b200 import build
    assert "arch=compute_90a,code=sm_90a" in " ".join(build.NVCC_FLAGS)
    for src in build.sources():
        body = open(src).read()
        assert "triton" not in body.lower()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "superpoint_graph_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                body = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", body, re.M), f


def test_ops_reject_cpu_tensors_without_fallback():
    from superpoint_graph_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.gemm(torch.randn(4, 4), 4, True, torch.randn(4, 4), 4, True, 4, 4, 4)
    from superpoint_graph_b200.spg_modules import GRUCellEx
    with pytest.raises(RuntimeError):
        GRUCellEx(32, 32)(torch.randn(3, 32), torch.randn(3, 32))


# ------------------------------------------------------------------- graph bookkeeping
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
    def __init__(self, nv, edges, feats):
        self._nv, self._edges = nv, [tuple(int(v) for v in e) for e in edges]
        self.es = _ES({"f": [list(map(float, f)) for f in feats]})
        self.vs = list(range(nv))

    def get_edgelist(self):
        return self._edges

    def indegree(self, vs, loops=True):
        d = [0] * self._nv
        for _, tt in self._edges:
            d[tt] += 1
        return d

    def vcount(self):
        return self._nv


def test_graph_conv_info_bit_exact(golden_dir):
    from superpoint_graph_b200.spg_ecc import GraphConvInfo
    g = load(golden_dir, "graph_conv_info.npz")
    graphs = [_Graph(int(g["nv%d" % i]), g["edges%d" % i], g["feats%d" % i]) for i in range(2)]
    info = GraphConvInfo(graphs, lambda ea: (torch.from_numpy(np.asarray(ea["f"], dtype=np.float32)), None))
    idxn, idxe, degs, degs_gpu, ef = info.get_buffers()
    assert idxe is None and degs_gpu is None
    assert idxn.dtype == torch.int64 and np.array_equal(idxn.numpy(), g["idxn"])
    assert np.array_equal(degs.numpy(), g["degs"])
    assert np.array_equal(info.get_pyg_buffers().numpy(), g["edge_indexes"])
    assert np.array_equal(ef.numpy(), g["edgefeats"])


def test_csr_views_are_consistent(golden_dir):
    from superpoint_graph_b200.ops import build_csr_host
    g = load(golden_dir, "graph_conv_info.npz")
    idxn, degs = g["idxn"], g["degs"]
    n = degs.shape[0]
    h = build_csr_host(idxn, degs, n)
    assert h["tgt_rowptr"][0] == 0 and h["tgt_rowptr"][-1] == idxn.shape[0]
    assert np.array_equal(np.diff(h["tgt_rowptr"]), degs)
    assert np.array_equal(h["edge_tgt"], g["edge_indexes"][1])
    # source CSR: a stable permutation grouping edges by source
    perm = h["src_perm"]
    assert sorted(perm.tolist()) == list(range(idxn.shape[0]))
    assert np.all(np.diff(idxn[perm]) >= 0)
    for j in range(n):
        seg = perm[h["src_rowptr"][j]:h["src_rowptr"][j + 1]]
        assert np.all(idxn[seg] == j) and np.all(np.diff(seg) > 0)
    # empty graph / zero-degree tails
    e = build_csr_host(np.zeros(0, dtype=np.int64), np.zeros(3, dtype=np.int64), 3)
    assert e["tgt_rowptr"].tolist() == [0, 0, 0, 0] and e["src_rowptr"].tolist() == [0, 0, 0, 0]


def test_edge_shards(golden_dir):
    from superpoint_graph_b200.spg_ecc import get_edge_shards
    for case in json.load(open(os.path.join(golden_dir, "edge_shards.json"))):
        got = get_edge_shards(np.array(case["degs"]), case["limit"])
        assert [list(s) for s in got] == case["shards"], case


# ------------------------------------------------------------ model construction contract
def test_state_dict_keys_shapes_and_init_match_reference(golden_dir):
    """Keys/shapes are the checkpoint contract; initial values are reproduced too because module
    construction order and RNG consumption follow the reference (PointNet reseeds to 0)."""
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    from superpoint_graph_b200.spg_pointnet import PointNet
    for tag, config in (("vv", "gru_3_1_1_1_0,f_13"), ("cat", "gru_2,f_8"), ("mat", "gru_2_0,f_13")):
        g = load(golden_dir, "graphnet_%s.npz" % tag)
        torch.manual_seed(13)
        net = GraphNetwork(config, 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0, cuda=False)
        want = {k[4:]: v for k, v in g.items() if k.startswith("sd0.")}
        got = net.state_dict()
        assert list(got.keys()) == list(want.keys())
        for k, v in want.items():
            assert tuple(got[k].shape) == tuple(v.shape), k
            np.testing.assert_allclose(got[k].numpy(), v, rtol=0, atol=1e-6, err_msg=k)  # QR rounding varies with threads
    g = load(golden_dir, "train_steps.npz")
    ptn = PointNet([16, 16, 32], [32, 16, 8], [8, 16], [16, 8], 6, 6, prelast_do=0)
    want = {k[5:]: v for k, v in g.items() if k.startswith("ptn0.")}
    got = ptn.state_dict()
    assert list(got.keys()) == list(want.keys())
    for k, v in want.items():
        np.testing.assert_allclose(got[k].numpy(), v, rtol=0, atol=1e-6, err_msg=k)  # QR rounding varies with threads


def test_model_config_trap_vv_token():
    """`gru_10_0` means matrix filters (third token is vv=0), bare `gru_10` vector filters."""
    from superpoint_graph_b200.spg_graphnet import GraphNetwork
    n = lambda c: sum(p.numel() for p in GraphNetwork(c, 32, [13, 32, 128, 64], True, 0, 2, 1e20, use_pyg=0, cuda=False).parameters())
    assert n("gru_10_0,f_13") == 90573
    assert n("gru_10_1_1_1_0,f_13") == 22925
    assert n("gru_10,f_8") == 25320
    with pytest.raises(NotImplementedError):
        GraphNetwork("xyz_1", 32, [13, 32], use_pyg=0)
    with pytest.raises(NotImplementedError):
        GraphNetwork("gru_10", 32, [13, 32, 128, 64], use_pyg=1)


def test_dropin_aliases():
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from superpoint_graph_b200 import dropin; dropin.install()\n"
        "from learning import pointnet, graphnet, modules, ecc\n"
        "import ecc as ecc2\n"
        "assert ecc2 is ecc and hasattr(ecc, 'GraphConvInfo') and hasattr(ecc, 'GraphConvFunction')\n"
        "assert pointnet.PointNet.__module__.startswith('superpoint_graph_b200')\n"
        "import inspect\n"
        "sig = inspect.signature(pointnet.PointNet.__init__)\n"
        "assert list(sig.parameters)[1:8] == ['nf_conv','nf_fc','nf_conv_stn','nf_fc_stn','nfeat','nfeat_stn','nfeat_global']\n"
        "sig = inspect.signature(modules.RNNGraphConvModule.__init__)\n"
        "assert list(sig.parameters)[1:] == ['cell','filter_net','nfeat','vv','gc_info','nrepeats','cat_all','edge_mem_limit','use_pyg','cuda']\n"
        "print('ok')\n" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr


# ---------------------------------------------------------------------------- synthetic
def test_synthetic_batch_shapes():
    from superpoint_graph_b200.synthetic import batch_counts, make_batch
    b = make_batch(n_nodes=500, seed=1)
    N, nv, pts, E = batch_counts(b)
    assert N == 500 and b["clouds"].shape == (nv, 14, 128) and pts == nv * 128
    assert int(b["degs"].sum()) == E and (b["degs"] == 0).any()
    assert 7 * N < E < 14 * N
    assert int((b["clouds_flag"] == 0).sum()) == nv
    tgt = np.repeat(np.arange(N), b["degs"].numpy())
    assert np.all(np.diff(tgt) >= 0)
    b2 = make_batch(n_nodes=500, seed=1)
    assert all(torch.equal(b[k], b2[k]) for k in b)
    xyz = b["clouds"][:, :3, :]
    assert float(xyz.abs().max()) <= 1.0 + 1e-5 and abs(float(xyz.mean())) < 1e-3


def test_host_batch_validates_the_collated_graph_arrays():
    """HostBatch checks (idxn, degs) once on the host (the device builder then runs unchecked)."""
    from superpoint_graph_b200.synthetic import make_batch
    from superpoint_graph_b200.trainer import HostBatch
    b = make_batch(n_nodes=40, seed=3, nfeat=14, n_classes=13, minpts=40)
    hb = HostBatch(b)
    assert hb.idxn.dtype == torch.int64 and hb.degs.dtype == torch.int64
    assert int(hb.degs.sum()) == hb.idxn.numel()
    assert hb.h2d_bytes() == sum(getattr(hb, f).numel() * getattr(hb, f).element_size() for f in HostBatch.FIELDS)
    bad = dict(b)
    bad["idxn"] = b["idxn"].clone()
    bad["idxn"][0] = 40
    with pytest.raises(ValueError, match="idxn out of range"):
        HostBatch(bad)
    bad = dict(b)
    bad["degs"] = b["degs"].clone()
    bad["degs"][0] += 1
    with pytest.raises(ValueError, match="does not match the number of edges"):
        HostBatch(bad)


def test_launch_policy_switch_is_a_host_side_setter(monkeypatch):
    """spg_set_pdl needs no device; an explicit SPG_PDL in the environment makes ops.set_pdl a no-op."""
    from superpoint_graph_b200 import _lib, ops
    _lib.call("spg_set_pdl", 0)
    _lib.call("spg_set_pdl", 1)
    calls = []
    monkeypatch.setattr(_lib, "call", lambda name, *a: calls.append((name, a)))
    monkeypatch.delenv("SPG_PDL", raising=False)
    ops.set_pdl(0)
    monkeypatch.setenv("SPG_PDL", "1")
    ops.set_pdl(0)
    assert calls == [("spg_set_pdl", (0,))]
