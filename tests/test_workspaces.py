"""The workspace contract shared by every entry point that sizes its scratch with a `spg_*_workspace` query:
the reported size is exact (a run in exactly that many bytes matches a run in a generous workspace, bit for bit,
and writes nothing past it), a misaligned workspace is SPG_E_ALIGN, one byte short is SPG_E_BADARG, and both are
rejected before anything is launched.

Each case runs one stage's chain of calls at a small size; with probe=True, `call` first tries every call that
takes a workspace with a misaligned and with a short one."""
import ctypes

import pytest
import torch

SPG_E_BADARG, SPG_E_ALIGN = -1, -3
TAIL = 4096
SENTINEL, GENEROUS_FILL = 0xA5, 0x5A


class _Ws(object):
    """A workspace of the bytes `query` reports: exact with a sentinel tail behind it, or twice as large."""

    def __init__(self, lib, query, sizes, exact):
        nbytes = ctypes.c_int64(-1)
        assert getattr(lib, query)(*sizes, ctypes.byref(nbytes)) == 0, query
        self.reported = nbytes.value
        assert self.reported > 0 and self.reported % 256 == 0, (query, self.reported)
        self.bytes = self.reported if exact else 2 * self.reported + TAIL  # what the calls are told
        self.buf = torch.full((self.bytes + TAIL,), SENTINEL if exact else GENEROUS_FILL, dtype=torch.uint8,
                              device="cuda")
        assert self.buf.data_ptr() % 256 == 0


def _run(chain, exact, probe):
    from superpoint_graph_b200 import _lib, ops

    lib = _lib.lib()
    spaces = []

    def alloc(query, *sizes):
        spaces.append(_Ws(lib, query, sizes, exact))
        return spaces[-1]

    def args_with(args, ws_args):
        out = []
        for a in args:
            if isinstance(a, _Ws):
                out += ws_args(a)
            else:
                out.append(a.data_ptr() if isinstance(a, torch.Tensor) else a)
        return out + [_lib.current_stream()]

    def call(name, *args):
        fn = getattr(lib, name)
        if probe:
            before = ops.total_launches()
            assert fn(*args_with(args, lambda w: [w.buf.data_ptr() + 16, w.bytes])) == SPG_E_ALIGN, name
            assert fn(*args_with(args, lambda w: [w.buf.data_ptr(), w.bytes - 1])) == SPG_E_BADARG, name
            assert ops.total_launches() == before, name
        rc = fn(*args_with(args, lambda w: [w.buf.data_ptr(), w.bytes]))
        assert rc == 0, (name, rc)

    outs = chain(alloc, call)
    torch.cuda.synchronize()
    return outs, spaces


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _zeros(shape, dtype):
    return torch.zeros(shape, dtype=dtype, device="cuda")


def _graph(alloc, call):
    n, E = 6, 9
    degs = torch.tensor([2, 0, 3, 1, 2, 1], dtype=torch.int64).cuda()
    idxn = torch.randint(0, n, (E,), generator=_gen(0)).cuda()
    out = [_zeros(E, torch.int32), _zeros(n + 1, torch.int32), _zeros(E, torch.int32), _zeros(n + 1, torch.int32),
           _zeros(E, torch.int32), _zeros(1, torch.int32)]
    ws = alloc("spg_graph_build_workspace", n, n, E)
    call("spg_graph_build", idxn, degs, n, n, E, *out, ws)
    return out


def _knn(alloc, call):
    n, k, k1 = 64, 4, 2
    xyz = torch.rand(n, 3, generator=_gen(1)).cuda()  # in [0, 1): cells of 0.25 from the origin
    grid = (0.0, 0.0, 0.0, 0.25, 4, 4, 4)
    ws = alloc("spg_knn_workspace", n)
    n_cells = _zeros(1, torch.int32)
    call("spg_knn_grid", xyz, n, *grid, ws, n_cells)
    out = [n_cells, _zeros(n * k1, torch.int64), _zeros(n * k1, torch.int64), _zeros(n * k1, torch.float32),
           _zeros(n * k, torch.int64)]
    call("spg_knn_query", n, k, k1, *grid, ws, *out[1:])
    return out


def _sp_graph(alloc, call):
    n, n_com, T = 40, 5, 12
    g = _gen(2)
    xyz = torch.rand(n, 3, generator=g).cuda()
    comp = (torch.arange(n) % n_com).cuda()
    simplices = torch.stack([torch.randperm(n, generator=g)[:4] for _ in range(T)]).cuda()
    sp = [_zeros((n_com, 3), torch.float32), _zeros(n_com, torch.float32), _zeros(n_com, torch.float32),
          _zeros(n_com, torch.float32), _zeros(n_com, torch.int64)]
    status = _zeros(1, torch.int32)
    call("spg_sp_points", xyz, comp, n, n_com, None, 0, 0, 0, alloc("spg_sp_points_workspace", n), *sp, None,
         status)
    offsets = _zeros(T + 1, torch.int32)
    call("spg_sp_edges_count", comp, n, simplices, 1, T, offsets, alloc("spg_sp_edges_workspace", T, 0), status)
    n_cand = int(offsets[T])
    ws = alloc("spg_sp_edges_workspace", T, n_cand)
    n_sedg = _zeros(1, torch.int64)
    call("spg_sp_edges_build", xyz, comp, n, simplices, 1, T, offsets, n_cand, 0.0, ws, n_sedg)
    m = int(n_sedg)
    assert m > 0
    edges = [_zeros(m, torch.int64), _zeros(m, torch.int64), _zeros((m, 3), torch.float32),
             _zeros((m, 3), torch.float32), _zeros(m, torch.float32), _zeros((m, 3), torch.float32)] + [
        _zeros(m, torch.float32) for _ in range(4)]
    call("spg_sp_edges_features", xyz, T, n_cand, ws, m, *sp, *edges)
    return sp + [status, offsets, n_sedg] + edges


def _prune(alloc, call):
    n, rows, voxel, n_labels, n_objects = 100, 40, 0.3, 3, 4
    g = _gen(3)
    xyz = torch.rand(n, 3, generator=g).cuda()
    rgb = torch.randint(0, 256, (n, 3), generator=g).to(torch.uint8).cuda()
    labels = torch.randint(0, n_labels + 1, (n,), generator=g).cuda()
    objects = torch.randint(0, n_objects + 1, (n,), generator=g).cuda()
    ws = alloc("spg_prune_workspace", n, rows)
    words = _zeros(4, torch.int64)
    call("spg_prune_bounds", xyz, n, rows, voxel, labels, n_labels, objects, n_objects, ws, words)
    n_voxels = _zeros(1, torch.int64)
    call("spg_prune_voxels", xyz, n, rows, voxel, *[int(b) for b in words[1:].cpu()], ws, n_voxels)
    m = int(n_voxels)
    out = [_zeros((m, 3), torch.float32), _zeros((m, 3), torch.uint8), _zeros((m, n_labels + 1), torch.int64),
           _zeros((m, n_objects + 1), torch.int64)]
    call("spg_prune_reduce", xyz, rgb, labels, n_labels, objects, n_objects, n, rows, ws, m, *out)
    return [words, n_voxels] + out


def _subgraph(alloc, call):
    n, E = 30, 50
    g = _gen(4)
    mask = (torch.rand(n, generator=g) < 0.6).to(torch.uint8).cuda()
    objects = torch.randint(0, 7, (n,), generator=g).to(torch.int32).cuda()
    src = torch.randint(0, n, (E,), generator=g).to(torch.int32).cuda()
    tgt = torch.randint(0, n, (E,), generator=g).to(torch.int32).cuda()
    out = [_zeros(n + 1, torch.int32), _zeros(n, torch.int32), _zeros(E + 1, torch.int32), _zeros(1, torch.int32)]
    call("spg_lp_subgraph_select", mask, objects, n, src, tgt, E, *out, alloc("spg_lp_subgraph_workspace", n, E))
    return out


def _learned_partition(alloc, call):
    V, E, C = 30, 60, 6
    g = _gen(5)
    src = torch.randint(0, V, (E,), generator=g).cuda()
    tgt = torch.randint(0, V, (E,), generator=g).cuda()
    is_tr = torch.randint(0, 2, (E,), generator=g).to(torch.uint8).cuda()
    pic = torch.randint(0, C, (V,), generator=g).cuda()
    objects = torch.randint(0, 4, (V,), generator=g).cuda()
    # each call is given the bytes reported for the counts it sizes by (no components for the first two)
    inc = [_zeros(V + 1, torch.int32), _zeros(2 * E, torch.int32)]
    call("spg_lp_incidence", src, tgt, V, E, *inc, alloc("spg_lp_workspace", V, E, 0))
    xpart = [_zeros(E, torch.float32), _zeros(V, torch.int32), _zeros(V, torch.int32), _zeros(1, torch.int32)]
    call("spg_lp_xpart", src, tgt, is_tr, pic, V, E, 50.0, *xpart, alloc("spg_lp_workspace", V, E, 0))
    seal = [_zeros(E, torch.float32), _zeros(C, torch.int32)]
    call("spg_lp_seal", src, tgt, is_tr, pic, objects, V, E, C, 50.0, *seal, alloc("spg_lp_workspace", V, E, C))
    return inc + xpart + seal


CASES = {"graph_build": _graph, "knn": _knn, "sp_graph": _sp_graph, "prune": _prune, "lp_subgraph": _subgraph,
         "learned_partition": _learned_partition}


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_reported_bytes_suffice_and_nothing_is_written_past_them(case):
    got, spaces = _run(CASES[case], exact=True, probe=False)
    want, _ = _run(CASES[case], exact=False, probe=False)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and torch.equal(_bytes(a), _bytes(b)), (case, i)
    for ws in spaces:
        assert bool((ws.buf[ws.reported:] == SENTINEL).all()), case


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_misaligned_or_short_workspace_is_rejected_before_any_launch(case):
    _run(CASES[case], exact=True, probe=True)
