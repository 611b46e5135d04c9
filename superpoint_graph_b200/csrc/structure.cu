// The learned partition's graph structure (ref: supervized_partition/graph_processing.py:144-193), the step between
// a pruned cloud and read_structure / PartitionStore:
//
//   st_vor      the Voronoi adjacency of compute_graph_nn_2(voronoi > 0) (ref: partition/graphs.py:42-64): the 6 T
//               directed candidates of the simplices in column-block order, d2 = (dx dx + dy dy) + dz dz rounded op
//               by op in float32, those with d2 < voronoi kept in candidate order (a count pass and an emit pass
//               over fixed chunks, a block scan inside each), then the union with the k-NN edges deduplicated by
//               one radix sort of the keys (t << 31) | s and a unique pass: edges sorted by (target, source)
//   st_cc       libply_c's connected_comp (ref: partition/ply_c/connected_components.cpp:17-110, cutoff 0) on the
//               union-find of cc.cuh; members by a stable radix sort of the component ids
//   st_labels   first-maximum argmax of label / object histograms, per-edge transitions
//   st_select   the ids of flagged items in order (CUB select), row gathers
//   st_points   elevation (z - min z, or z minus a plane in fp64) and xyn in float32, geof's column 3 doubled
//
// No float atomics; integer atomics only count, so every output is bit-reproducible.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "cc.cuh"
#include "workspace.cuh"

namespace spg {

constexpr int ST_THREADS = 256;
constexpr int VOR_ITEMS = 16;                           // candidates per thread
constexpr int64_t VOR_CHUNK = ST_THREADS * VOR_ITEMS;   // candidates per block of the count and emit passes

static unsigned st_grid(int64_t n) { return (unsigned)ceil_div64(n > 0 ? n : 1, ST_THREADS); }

static int st_bits(uint64_t n) {  // smallest b with 2^b >= n (at least 1)
    int b = 1;
    while (b < 64 && (1ull << b) < n) ++b;
    return b;
}

static int64_t vor_blocks(int64_t n_tets) { return ceil_div64(6 * n_tets, VOR_CHUNK); }

// ------------------------------------------------------------------------------------------ Voronoi adjacency
__constant__ int kPairA[6] = {0, 0, 0, 1, 1, 2};
__constant__ int kPairB[6] = {1, 2, 3, 2, 3, 3};

// candidate c = p T + r: (simplices[r][A[p]], simplices[r][B[p]]); keep it when both ids are in range and
// d2 < vor in float32 (graphs.py:48-49); out-of-range ids set status bit 2
template <class I>
__device__ __forceinline__ bool vor_candidate(const float* __restrict__ xyz, int64_t n, const I* __restrict__ simp,
                                              int64_t n_tets, int64_t c, float vor, int64_t* s_out, int64_t* t_out,
                                              float* d2_out, uint32_t* status) {
    const int p = (int)(c / n_tets);
    const int64_t r = c - (int64_t)p * n_tets;
    const int64_t s = (int64_t)simp[4 * r + kPairA[p]], t = (int64_t)simp[4 * r + kPairB[p]];
    if (s < 0 || s >= n || t < 0 || t >= n) {
        atomicOr(status, 2u);
        return false;
    }
    const float dx = __fsub_rn(__ldg(xyz + 3 * s), __ldg(xyz + 3 * t));
    const float dy = __fsub_rn(__ldg(xyz + 3 * s + 1), __ldg(xyz + 3 * t + 1));
    const float dz = __fsub_rn(__ldg(xyz + 3 * s + 2), __ldg(xyz + 3 * t + 2));
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    *s_out = s;
    *t_out = t;
    *d2_out = d2;
    return d2 < vor;
}

template <class I>
__global__ void __launch_bounds__(ST_THREADS)
st_vor_count_kernel(const float* __restrict__ xyz, int64_t n, const I* __restrict__ simp, int64_t n_tets, float vor,
                    int64_t* __restrict__ block_counts, int64_t n_blocks, uint32_t* __restrict__ status) {
    SPG_PDL_ENTRY();
    using Reduce = cub::BlockReduce<int, ST_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    const int64_t n_cand = 6 * n_tets;
    const int64_t c0 = (int64_t)blockIdx.x * VOR_CHUNK + (int64_t)threadIdx.x * VOR_ITEMS;
    int kept = 0;
    for (int i = 0; i < VOR_ITEMS && c0 + i < n_cand; ++i) {
        int64_t s, t;
        float d2;
        kept += vor_candidate(xyz, n, simp, n_tets, c0 + i, vor, &s, &t, &d2, status);
    }
    const int total = Reduce(tmp).Sum(kept);
    if (threadIdx.x == 0) {
        block_counts[blockIdx.x] = total;
        atomicAdd((unsigned long long*)(block_counts + n_blocks), (unsigned long long)total);
    }
}

template <class I>
__global__ void __launch_bounds__(ST_THREADS)
st_vor_emit_kernel(const float* __restrict__ xyz, int64_t n, const I* __restrict__ simp, int64_t n_tets, float vor,
                   const int64_t* __restrict__ block_off, uint32_t* __restrict__ status,
                   unsigned long long* __restrict__ keys, float* __restrict__ distances) {
    SPG_PDL_ENTRY();
    using Scan = cub::BlockScan<int, ST_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t n_cand = 6 * n_tets;
    const int64_t c0 = (int64_t)blockIdx.x * VOR_CHUNK + (int64_t)threadIdx.x * VOR_ITEMS;
    uint32_t mask = 0;
    int kept = 0;
    for (int i = 0; i < VOR_ITEMS && c0 + i < n_cand; ++i) {
        int64_t s, t;
        float d2;
        if (vor_candidate(xyz, n, simp, n_tets, c0 + i, vor, &s, &t, &d2, status)) {
            mask |= 1u << i;
            ++kept;
        }
    }
    int pos;
    Scan(tmp).ExclusiveSum(kept, pos);
    int64_t o = block_off[blockIdx.x] + pos;
    for (int i = 0; mask >> i; ++i) {
        if (!((mask >> i) & 1u)) continue;
        int64_t s, t;
        float d2;
        vor_candidate(xyz, n, simp, n_tets, c0 + i, vor, &s, &t, &d2, status);
        keys[o] = ((unsigned long long)t << 31) | (unsigned long long)s;
        distances[o] = d2;
        ++o;
    }
}

// the k-NN edges (i, knn_target[i k + j]) after the kept candidates (graphs.py:53-56)
__global__ void __launch_bounds__(ST_THREADS)
st_vor_knn_keys_kernel(const int64_t* __restrict__ knn_target, int64_t n_knn, int64_t k, int64_t n,
                       unsigned long long* __restrict__ keys, uint32_t* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_knn) return;
    int64_t t = knn_target[e];
    if (t < 0 || t >= n) {
        atomicOr(status, 2u);
        t = 0;
    }
    keys[e] = ((unsigned long long)t << 31) | (unsigned long long)(e / k);
}

__global__ void __launch_bounds__(ST_THREADS)
st_vor_split_kernel(const unsigned long long* __restrict__ keys, int64_t m, const int64_t* __restrict__ n_edges,
                    int64_t* __restrict__ source, int64_t* __restrict__ target) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m || e >= *n_edges) return;
    const unsigned long long k = keys[e];
    source[e] = (int64_t)(k & 0x7fffffffull);
    target[e] = (int64_t)(k >> 31);
}

struct VorWs {
    int64_t* block_off;
    unsigned long long *keys, *keys_sorted;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n, int64_t n_tets, int64_t n_knn, int64_t n_kept, void* base, VorWs* w) {
    const int64_t nb = vor_blocks(n_tets), m = n_kept + n_knn;
    size_t cub_bytes = 1;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int64_t*)nullptr, (int64_t*)nullptr, nb);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortKeys, (const unsigned long long*)nullptr,
                  (unsigned long long*)nullptr, m, 0, 31 + st_bits((uint64_t)n));
    SPG_CUB_BYTES(cub_bytes, cub::DeviceSelect::Unique, (const unsigned long long*)nullptr,
                  (unsigned long long*)nullptr, (int64_t*)nullptr, m);
    Planner p(base);
    w->block_off = p.take<int64_t>(nb);
    w->keys = p.take<unsigned long long>(m);
    w->keys_sorted = p.take<unsigned long long>(m);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

static bool vor_args_ok(int64_t n, int64_t n_tets) {
    return n > 0 && n < (1ll << 31) - 1 && n_tets >= 0 && n_tets <= (1ll << 29);
}

// ------------------------------------------------------------------------------------------ connected components
// parent = identity, comp_size = 0 (n_ver + 1 entries: the last one closes the offsets scan), members' sort values
__global__ void __launch_bounds__(ST_THREADS)
st_cc_init_kernel(int64_t n_ver, int* __restrict__ parent, int* __restrict__ comp_size, int64_t* __restrict__ iota) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_ver) return;
    comp_size[i] = 0;
    if (i == n_ver) return;
    parent[i] = (int)i;
    iota[i] = i;
}

// union of the endpoints of every edge whose mask byte, read as a signed char, is > 0 (connected_components.cpp:25)
__global__ void __launch_bounds__(ST_THREADS)
st_cc_hook_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt, const uint8_t* __restrict__ active,
                  int64_t n_ver, int64_t n_edges, int* __restrict__ parent, uint32_t* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int64_t s = src[e], t = tgt[e];
    if (s < 0 || s >= n_ver || t < 0 || t >= n_ver) {
        atomicOr(status, 2u);
        return;
    }
    if ((signed char)active[e] > 0) cc_union(parent, (int)s, (int)t);
}

struct CcWs {
    int *parent, *is_root, *root_rank, *comp_size;
    int64_t *iota, *keys_sorted;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n_ver, void* base, CcWs* w) {
    size_t cub_bytes = 1;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int*)nullptr, (int*)nullptr, n_ver);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int*)nullptr, (int64_t*)nullptr, n_ver + 1);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const int64_t*)nullptr, (int64_t*)nullptr,
                  (const int64_t*)nullptr, (int64_t*)nullptr, n_ver, 0, st_bits((uint64_t)n_ver));
    Planner p(base);
    w->parent = p.take<int>(n_ver);
    w->is_root = p.take<int>(n_ver);
    w->root_rank = p.take<int>(n_ver);
    w->comp_size = p.take<int>(n_ver + 1);
    w->iota = p.take<int64_t>(n_ver);
    w->keys_sorted = p.take<int64_t>(n_ver);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

// ------------------------------------------------------------------------------------------ labels, transitions
// out[i] = add + the first column of maximum count among a[i, col0:] (np.argmax); zero_empty: 0 where that row
// sums to 0 (graph_processing.py:152-154); weight (may be NULL): 0 there, else 1 (:161-162)
__global__ void __launch_bounds__(ST_THREADS)
st_argmax_kernel(const int64_t* __restrict__ a, int64_t n, int64_t cols, int64_t col0, int64_t add, int zero_empty,
                 int64_t* __restrict__ out, float* __restrict__ weight) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t* row = a + i * cols;
    int64_t best = row[col0], arg = 0;
    unsigned long long sum = (unsigned long long)best;
    for (int64_t j = col0 + 1; j < cols; ++j) {
        const int64_t v = row[j];
        sum += (unsigned long long)v;
        if (v > best) {
            best = v;
            arg = j - col0;
        }
    }
    const bool empty = sum == 0;
    out[i] = zero_empty && empty ? 0 : arg + add;
    if (weight) weight[i] = empty ? 0.f : 1.f;
}

// mode 0: lab[s] != lab[t] (:149, :165, :169); 1: hs != (ht * (hs != 0) * (ht != 0)) (:155-156, numpy's
// precedence: the products bind before !=); 2: lab[s] == lab[t] (the active edges of :171-173)
__global__ void __launch_bounds__(ST_THREADS)
st_transitions_kernel(const int64_t* __restrict__ lab, int64_t n, const int64_t* __restrict__ src,
                      const int64_t* __restrict__ tgt, int64_t n_edges, int mode, uint8_t* __restrict__ out,
                      uint32_t* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int64_t s = src[e], t = tgt[e];
    if (s < 0 || s >= n || t < 0 || t >= n) {
        atomicOr(status, 2u);
        out[e] = 0;
        return;
    }
    const int64_t hs = lab[s], ht = lab[t];
    out[e] = mode == 1 ? (uint8_t)(hs != ht * (int64_t)(hs != 0) * (int64_t)(ht != 0))
                       : (uint8_t)((hs != ht) == (mode == 0));
}

// ------------------------------------------------------------------------------------------ selection, gathers
__global__ void __launch_bounds__(ST_THREADS)
st_select_flags_kernel(const uint8_t* __restrict__ flags, int64_t n, int want, uint8_t* __restrict__ sel) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) sel[i] = (flags[i] != 0) == (want != 0);
}

__global__ void __launch_bounds__(ST_THREADS)
st_gather_rows_kernel(const uint8_t* __restrict__ src, int64_t n_rows, int64_t row_bytes,
                      const int64_t* __restrict__ index, int64_t m, uint8_t* __restrict__ out,
                      uint32_t* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m * row_bytes) return;
    const int64_t r = j / row_bytes, b = j - r * row_bytes, i = index[r];
    if (i < 0 || i >= n_rows) {
        atomicOr(status, 2u);
        out[j] = 0;
        return;
    }
    out[j] = src[i * row_bytes + b];
}

struct SelWs {
    uint8_t* sel;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n, void* base, SelWs* w) {
    size_t cub_bytes = 1;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceSelect::Flagged, thrust::counting_iterator<int64_t>(0),
                  (const uint8_t*)nullptr, (int64_t*)nullptr, (int64_t*)nullptr, n);
    Planner p(base);
    w->sel = p.take<uint8_t>(n);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

// ------------------------------------------------------------------------------------------ per-point fields
// bounds: spg_knn_bounds' words (order-preserving keys of the per-axis minimum 0-2 and maximum 3-5)
__global__ void __launch_bounds__(ST_THREADS)
st_points_kernel(const float* __restrict__ xyz, int64_t n, const uint32_t* __restrict__ bounds, int plane, double c0,
                 double c1, double b, float* __restrict__ elevation, float* __restrict__ xyn,
                 uint8_t* __restrict__ low, float* __restrict__ geof) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const float mx = float_unkey(bounds[0]), my = float_unkey(bounds[1]), mz = float_unkey(bounds[2]);
    const float Mx = float_unkey(bounds[3]), My = float_unkey(bounds[4]);
    const float dz = __fsub_rn(z, mz);
    if (low) low[i] = dz < 0.5f;  // graph_processing.py:182
    if (elevation) {
        elevation[i] = plane ? (float)__dsub_rn((double)z, __dadd_rn(__dadd_rn(__dmul_rn((double)x, c0),
                                                                                 __dmul_rn((double)y, c1)), b))
                             : dz;  // :184, :186
    }
    if (xyn) {  // :189-190: (xy - mi) / (ma - mi + float32(1e-8))
        const float eps = 1e-8f;
        xyn[2 * i] = __fdiv_rn(__fsub_rn(x, mx), __fadd_rn(__fsub_rn(Mx, mx), eps));
        xyn[2 * i + 1] = __fdiv_rn(__fsub_rn(y, my), __fadd_rn(__fsub_rn(My, my), eps));
    }
    if (geof) geof[4 * i + 3] = __fmul_rn(2.f, geof[4 * i + 3]);  // :177
}

}  // namespace spg

using namespace spg;

// ------------------------------------------------------------------------------------------ C-ABI
int64_t spg_st_vor_blocks(int64_t n_tets) { return n_tets > 0 ? vor_blocks(n_tets) : 0; }

int spg_st_vor_workspace(int64_t n, int64_t n_tets, int64_t n_knn, int64_t n_kept, int64_t* bytes) {
    if (!bytes || !vor_args_ok(n, n_tets) || n_knn < 0 || n_kept < 0 || n_kept > 6 * n_tets) return SPG_E_BADARG;
    VorWs w;
    const int rc = layout(n, n_tets, n_knn, n_kept, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_st_vor_count(const float* xyz, int64_t n, const void* simplices, int ids64, int64_t n_tets, float voronoi,
                     int64_t* block_counts, uint32_t* status, spg_stream_t stream) {
    if (!vor_args_ok(n, n_tets) || !xyz || !block_counts || !status || (n_tets > 0 && !simplices))
        return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t nb = vor_blocks(n_tets);
    cudaError_t e = cudaMemsetAsync(block_counts + nb, 0, sizeof(int64_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (nb == 0) return SPG_OK;
    if (ids64)
        SPG_LAUNCH(K_ST_VOR, s, st_vor_count_kernel<int64_t>, nb, ST_THREADS, 0, xyz, n,
                   (const int64_t*)simplices, n_tets, voronoi, block_counts, nb, status);
    else
        SPG_LAUNCH(K_ST_VOR, s, st_vor_count_kernel<int32_t>, nb, ST_THREADS, 0, xyz, n,
                   (const int32_t*)simplices, n_tets, voronoi, block_counts, nb, status);
    return launch_status();
}

int spg_st_vor_build(const float* xyz, int64_t n, const void* simplices, int ids64, int64_t n_tets, float voronoi,
                     const int64_t* block_counts, const int64_t* knn_target, int64_t k_nn1, int64_t n_kept,
                     void* workspace, int64_t workspace_bytes, float* distances, int64_t* source, int64_t* target,
                     int64_t* n_edges, uint32_t* status, spg_stream_t stream) {
    if (!vor_args_ok(n, n_tets) || k_nn1 < 1 || n_kept < 0 || n_kept > 6 * n_tets) return SPG_E_BADARG;
    if (!xyz || !knn_target || !source || !target || !n_edges || !status) return SPG_E_BADARG;
    if (n_tets > 0 && (!simplices || !block_counts)) return SPG_E_BADARG;
    if (n_kept > 0 && !distances) return SPG_E_BADARG;
    const int64_t n_knn = n * k_nn1, m = n_kept + n_knn, nb = vor_blocks(n_tets);
    VorWs w;
    int rc = layout(n, n_tets, n_knn, n_kept, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (n_kept > 0) {
        SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, block_counts, w.block_off, nb, s);
        if (ids64)
            SPG_LAUNCH(K_ST_VOR, s, st_vor_emit_kernel<int64_t>, nb, ST_THREADS, 0, xyz, n,
                       (const int64_t*)simplices, n_tets, voronoi, (const int64_t*)w.block_off, status, w.keys,
                       distances);
        else
            SPG_LAUNCH(K_ST_VOR, s, st_vor_emit_kernel<int32_t>, nb, ST_THREADS, 0, xyz, n,
                       (const int32_t*)simplices, n_tets, voronoi, (const int64_t*)w.block_off, status, w.keys,
                       distances);
    }
    SPG_LAUNCH(K_ST_VOR, s, st_vor_knn_keys_kernel, st_grid(n_knn), ST_THREADS, 0, knn_target, n_knn, k_nn1, n,
               w.keys + n_kept, status);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortKeys, (const unsigned long long*)w.keys, w.keys_sorted, m, 0,
            31 + st_bits((uint64_t)n), s);
    SPG_CUB(w.cub, cub::DeviceSelect::Unique, (const unsigned long long*)w.keys_sorted, w.keys, n_edges, m, s);
    SPG_LAUNCH(K_ST_VOR, s, st_vor_split_kernel, st_grid(m), ST_THREADS, 0, (const unsigned long long*)w.keys, m,
               (const int64_t*)n_edges, source, target);
    return launch_status();
}

int spg_st_cc_workspace(int64_t n_ver, int64_t* bytes) {
    if (!bytes || n_ver < 1 || too_big(n_ver)) return SPG_E_BADARG;
    CcWs w;
    const int rc = layout(n_ver, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_st_cc(const int64_t* src, const int64_t* tgt, const uint8_t* active, int64_t n_ver, int64_t n_edges,
              void* workspace, int64_t workspace_bytes, int64_t* in_component, int64_t* offsets, int64_t* members,
              int64_t* n_comp, uint32_t* status, spg_stream_t stream) {
    if (n_ver < 1 || too_big(n_ver) || n_edges < 0) return SPG_E_BADARG;
    if (!in_component || !offsets || !members || !n_comp || !status) return SPG_E_BADARG;
    if (n_edges > 0 && (!src || !tgt || !active)) return SPG_E_BADARG;
    CcWs w;
    int rc = layout(n_ver, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_ST_CC, s, st_cc_init_kernel, st_grid(n_ver + 1), ST_THREADS, 0, n_ver, w.parent, w.comp_size,
               w.iota);
    if (n_edges > 0)
        SPG_LAUNCH(K_ST_CC, s, st_cc_hook_kernel, st_grid(n_edges), ST_THREADS, 0, src, tgt, active, n_ver, n_edges,
                   w.parent, status);
    SPG_LAUNCH(K_ST_CC, s, cc_flatten_kernel, st_grid(n_ver), CC_THREADS, 0, w.parent, n_ver, w.is_root);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int*)w.is_root, w.root_rank, n_ver, s);
    SPG_LAUNCH(K_ST_CC, s, cc_label_kernel<int64_t>, st_grid(n_ver), CC_THREADS, 0, (const int*)w.parent,
               (const int*)w.root_rank, (const int*)w.is_root, n_ver, in_component, w.comp_size, n_comp);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int*)w.comp_size, offsets, n_ver + 1, s);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const int64_t*)in_component, w.keys_sorted,
            (const int64_t*)w.iota, members, n_ver, 0, st_bits((uint64_t)n_ver), s);
    return launch_status();
}

int spg_st_argmax(const int64_t* a, int64_t n, int64_t cols, int64_t col0, int64_t add, int zero_empty,
                  int64_t* out, float* weight, spg_stream_t stream) {
    if (n < 0 || cols < 1 || col0 < 0 || col0 >= cols) return SPG_E_BADARG;
    if (n == 0) return SPG_OK;
    if (!a || !out) return SPG_E_BADARG;
    SPG_LAUNCH(K_ST_LABELS, (cudaStream_t)stream, st_argmax_kernel, st_grid(n), ST_THREADS, 0, a, n, cols, col0, add,
               zero_empty, out, weight);
    return launch_status();
}

int spg_st_transitions(const int64_t* lab, int64_t n, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                       int mode, uint8_t* is_transition, uint32_t* status, spg_stream_t stream) {
    if (n < 0 || n_edges < 0 || mode < 0 || mode > 2 || !status) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n_edges == 0) return SPG_OK;
    if (!lab || !src || !tgt || !is_transition) return SPG_E_BADARG;
    SPG_LAUNCH(K_ST_LABELS, s, st_transitions_kernel, st_grid(n_edges), ST_THREADS, 0, lab, n, src, tgt, n_edges,
               mode, is_transition, status);
    return launch_status();
}

int spg_st_select_workspace(int64_t n, int64_t* bytes) {
    if (!bytes || n < 1) return SPG_E_BADARG;
    SelWs w;
    const int rc = layout(n, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_st_select(const uint8_t* flags, int64_t n, int want, void* workspace, int64_t workspace_bytes, int64_t* index,
                  int64_t* count, spg_stream_t stream) {
    if (n < 1 || !flags || !index || !count) return SPG_E_BADARG;
    SelWs w;
    int rc = layout(n, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SPG_LAUNCH(K_ST_SELECT, s, st_select_flags_kernel, st_grid(n), ST_THREADS, 0, flags, n, want, w.sel);
    SPG_CUB(w.cub, cub::DeviceSelect::Flagged, thrust::counting_iterator<int64_t>(0), (const uint8_t*)w.sel, index,
            count, n, s);
    return launch_status();
}

int spg_st_gather_rows(const void* src, int64_t n_rows, int64_t row_bytes, const int64_t* index, int64_t m, void* out,
                       uint32_t* status, spg_stream_t stream) {
    if (n_rows < 0 || row_bytes < 1 || m < 0 || !status) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (m == 0) return SPG_OK;
    if (!src || !index || !out) return SPG_E_BADARG;
    SPG_LAUNCH(K_ST_SELECT, s, st_gather_rows_kernel, st_grid(m * row_bytes), ST_THREADS, 0, (const uint8_t*)src,
               n_rows, row_bytes, index, m, (uint8_t*)out, status);
    return launch_status();
}

int spg_st_points(const float* xyz, int64_t n, const uint32_t* bounds, int plane, double c0, double c1, double b,
                  float* elevation, float* xyn, uint8_t* low, float* geof, spg_stream_t stream) {
    if (n < 0 || (n > 0 && (!xyz || !bounds))) return SPG_E_BADARG;
    if (n == 0) return SPG_OK;
    SPG_LAUNCH(K_ST_POINTS, (cudaStream_t)stream, st_points_kernel, st_grid(n), ST_THREADS, 0, xyz, n, bounds, plane,
               c0, c1, b, elevation, xyn, low, geof);
    return launch_status();
}
