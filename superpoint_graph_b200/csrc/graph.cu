// Device-side builder of the CSR views every ECC kernel reads, from the reference's collated
// (idxn, degs) pair (learning/ecc/GraphConvInfo.py:48-69 produces them on the host; the reference
// then uploads idxn/degs and re-derives offsets inside its kernels, ecc/cuda_kernels.py:55-139).
//
//   idxn32      int32 copy of idxn (source node of every edge, edges sorted by target)
//   tgt_rowptr  exclusive scan of the in-degrees                          [n_out + 1]
//   edge_tgt    target node of every edge                                 [n_edges]
//   src_perm    STABLE permutation that sorts the edges by source node    [n_edges]
//   src_rowptr  first position of every source node in that order         [n_in + 1]
//
// The scan and the stable sort are CUB device primitives (least-significant-digit radix sort is stable,
// so src_perm is bit-identical to numpy's argsort(kind="stable") that the host builder uses); the three
// kernels around them are this file's.  Integer work, HBM/latency bound, a few microseconds at batch size.
#include <cub/cub.cuh>

#include "workspace.cuh"

namespace spg {

constexpr int GB_THREADS = 256;

__global__ void __launch_bounds__(GB_THREADS)
graph_prepare_kernel(const int64_t* __restrict__ idxn, const int64_t* __restrict__ degs, int64_t n_out,
                     int64_t n_in, int64_t n_edges, int* __restrict__ idxn32, int* __restrict__ iota,
                     int* __restrict__ degs32, int* __restrict__ tgt_rowptr, int* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) tgt_rowptr[0] = 0;
    if (i < n_edges) {
        const int64_t s = idxn[i];
        if (s < 0 || s >= n_in) atomicOr(status, 1);
        idxn32[i] = (int)s;
        iota[i] = (int)i;
    }
    if (i < n_out) {
        const int64_t d = degs[i];
        if (d < 0 || d > n_edges) atomicOr(status, 2);
        degs32[i] = (int)d;
    }
}

// thread per edge: its target is the row whose [rowptr[v], rowptr[v+1]) holds it
__global__ void __launch_bounds__(GB_THREADS)
graph_edge_tgt_kernel(const int* __restrict__ tgt_rowptr, int64_t n_out, int64_t n_edges,
                      int* __restrict__ edge_tgt, int* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e == 0 && tgt_rowptr[n_out] != (int)n_edges) atomicOr(status, 4);  // sum(degs) != n_edges
    if (e >= n_edges) return;
    int64_t lo = 0, hi = n_out;  // last v with rowptr[v] <= e
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(tgt_rowptr + mid) <= (int)e) lo = mid; else hi = mid;
    }
    edge_tgt[e] = (int)lo;
}

// thread per source node (and one past the end): lower bound in the source-sorted key array
__global__ void __launch_bounds__(GB_THREADS)
graph_src_rowptr_kernel(const int* __restrict__ keys_sorted, int64_t n_in, int64_t n_edges,
                        int* __restrict__ src_rowptr) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v > n_in) return;
    int64_t lo = 0, hi = n_edges;  // first position with key >= v
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys_sorted + mid) < (int)v) lo = mid + 1; else hi = mid;
    }
    src_rowptr[v] = (int)lo;
}

static int key_bits(int64_t n_in) {
    int b = 1;
    while (b < 31 && (1ll << b) < n_in) ++b;
    return b;
}

struct GraphWs {
    int *degs32, *iota, *keys;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n_out, int64_t n_in, int64_t n_edges, void* base, GraphWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::InclusiveSum, (const int*)nullptr, (int*)nullptr, (int)n_out);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                  (int*)nullptr, (int)n_edges, 0, key_bits(n_in));
    Planner p(base);
    w->degs32 = p.take<int>(n_out);
    w->iota = p.take<int>(n_edges);
    w->keys = p.take<int>(n_edges);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_graph_build_workspace(int64_t n_out, int64_t n_in, int64_t n_edges, int64_t* bytes) {
    if (!bytes || n_out < 0 || n_in < 0 || n_edges < 0) return SPG_E_BADARG;
    if (too_big(n_out) || too_big(n_in) || too_big(n_edges)) return SPG_E_UNSUPPORTED;
    GraphWs w;
    const int rc = layout(n_out, n_in, n_edges, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_graph_build(const int64_t* idxn, const int64_t* degs, int64_t n_out, int64_t n_in, int64_t n_edges,
                    int32_t* idxn32, int32_t* tgt_rowptr, int32_t* edge_tgt, int32_t* src_rowptr,
                    int32_t* src_perm, int32_t* status, void* workspace, int64_t workspace_bytes,
                    spg_stream_t stream) {
    if (n_out < 0 || n_in < 0 || n_edges < 0) return SPG_E_BADARG;
    if (too_big(n_out) || too_big(n_in) || too_big(n_edges)) return SPG_E_UNSUPPORTED;
    if (!tgt_rowptr || !src_rowptr || !status) return SPG_E_BADARG;
    if ((n_edges > 0 && (!idxn || !idxn32 || !edge_tgt || !src_perm)) || (n_out > 0 && !degs)) return SPG_E_BADARG;
    GraphWs w;
    int rc = layout(n_out, n_in, n_edges, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;

    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int), s);
    if (e != cudaSuccess) return (int)e;
    const int64_t n_max = (n_edges > n_out ? n_edges : n_out) > 0 ? (n_edges > n_out ? n_edges : n_out) : 1;
    SPG_LAUNCH(K_GRAPH_BUILD, s, graph_prepare_kernel, (unsigned)ceil_div64(n_max, GB_THREADS), GB_THREADS, 0,
               idxn, degs, n_out, n_in, n_edges, idxn32, w.iota, w.degs32, tgt_rowptr, status);
    if (n_out > 0)
        SPG_CUB(w.cub, cub::DeviceScan::InclusiveSum, (const int*)w.degs32, tgt_rowptr + 1, (int)n_out, s);
    SPG_LAUNCH(K_GRAPH_BUILD, s, graph_edge_tgt_kernel, (unsigned)ceil_div64(n_edges > 0 ? n_edges : 1, GB_THREADS),
               GB_THREADS, 0, (const int*)tgt_rowptr, n_out, n_edges, edge_tgt, status);
    if (n_edges > 0)
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const int*)idxn32, w.keys, (const int*)w.iota, src_perm,
                (int)n_edges, 0, key_bits(n_in), s);
    SPG_LAUNCH(K_GRAPH_BUILD, s, graph_src_rowptr_kernel, (unsigned)ceil_div64(n_in + 1, GB_THREADS), GB_THREADS, 0,
               (const int*)w.keys, n_in, n_edges, src_rowptr);
    return launch_status();
}

}  // extern "C"
