// Voxel pruning of a point cloud (ref: partition/ply_c/ply_c.cpp:149-380 `prune`), the step before the first phase
// of both partition pipelines (partition/partition.py:124, supervized_partition/graph_processing.py:124,142), and its
// chunked form (partition/provider.py:250-303 `read_semantic3d_format`: every chunk of chunk_rows points pruned on
// its own, the results stacked in chunk order):
//
//   prune_bounds  per chunk the minimum and maximum of every axis (order-preserving keys, integer atomics), then the
//                 largest bin of every axis; status 1: a non-finite coordinate, 2: a bin >= 2^32, 4: a label outside
//                 [0, n_labels], 8: an object outside [0, n_objects] (each checked only where the reference reads it)
//   prune_keys    (chunk, bx, by, bz) packed into the fewest bits that hold the observed maxima; one stable CUB radix
//                 sort of (key, point) over those bits, or two (the low 64 bits, then the rest) when they exceed 64
//   prune_rows    the first point of every run (the smallest index: the sort is stable) flagged in point order; an
//                 exclusive scan of those flags numbers the voxels in order of first touch, which is the reference's
//                 insertion order and, chunks being contiguous, the stacking order; the runs' starts and rows
//   prune_reduce  the points gathered into sorted order; one thread per voxel runs the reference's serial fp32 sum in
//                 point order, / float(count), and the uint32 colour sums; the label and object histograms with
//                 warp-aggregated integer atomics
//
// No float atomics anywhere: two runs give identical bits.
#include <cub/cub.cuh>

#include "workspace.cuh"

namespace spg {

constexpr int PR_THREADS = 256;

// the reference's bin: (uint32) floor((x - x_min) / voxel), every step in fp32 (ply_c.cpp:329-331)
__device__ __forceinline__ float pr_binf(float x, float lo, float voxel) {
    return floorf(__fdiv_rn(__fsub_rn(x, lo), voxel));
}

// bounds words (uint32, workspace): [C][6] = ~(min key) of x y z, max key of x y z of chunk c
struct PruneGeom {
    const float* xyz;
    int64_t n;
    int64_t chunk_rows;  // rows per chunk (n for one chunk)
    float voxel;
    const unsigned* bounds;
    int bits_y, bits_z, bits_x;  // field widths: key = (((chunk << bx) | x) << by | y) << bz | z
    int bits_total;
};

__device__ __forceinline__ void pr_key(const PruneGeom& g, int64_t i, uint64_t& lo, uint64_t& hi) {
    const int64_t c = i / g.chunk_rows;
    const unsigned* b = g.bounds + 6 * c;
    const unsigned bx = (unsigned)pr_binf(__ldg(g.xyz + 3 * i), float_unkey(~__ldg(b)), g.voxel);
    const unsigned by = (unsigned)pr_binf(__ldg(g.xyz + 3 * i + 1), float_unkey(~__ldg(b + 1)), g.voxel);
    const unsigned bz = (unsigned)pr_binf(__ldg(g.xyz + 3 * i + 2), float_unkey(~__ldg(b + 2)), g.voxel);
    unsigned __int128 k = (unsigned __int128)c;
    k = (k << g.bits_x) | bx;
    k = (k << g.bits_y) | by;
    k = (k << g.bits_z) | bz;
    lo = (uint64_t)k;
    hi = (uint64_t)(k >> 64);
}

// ------------------------------------------------------------------------------------------------ bounds
// grid (blocks per chunk, chunks); status and bounds preset to 0 (the minima are kept complemented)
__global__ void __launch_bounds__(PR_THREADS) prune_bounds_kernel(const float* __restrict__ xyz, int64_t n,
                                                                  int64_t chunk_rows, const int64_t* __restrict__ labels,
                                                                  const int64_t* __restrict__ objects, int n_labels,
                                                                  int n_objects, unsigned* __restrict__ bounds,
                                                                  unsigned* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t c = blockIdx.y;
    const int64_t i0 = c * chunk_rows;
    const int64_t i1 = min(n, i0 + chunk_rows);
    unsigned lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u}, bad = 0u;
    for (int64_t i = i0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < i1;
         i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float v = __ldg(xyz + 3 * i + k);
            if (!isfinite(v)) {
                bad |= 1u;
                continue;
            }
            // -0 keys below +0; the reference's `<` does not order them, so either may be the minimum: both give the same bins
            const unsigned key = float_key(v);
            lo[k] = min(lo[k], key);
            hi[k] = max(hi[k], key);
        }
        if (labels) {
            const int64_t l = __ldg(labels + i);
            if (l < 0 || l > n_labels) bad |= 4u;
            if (objects) {
                const int64_t o = __ldg(objects + i);
                if (o < 0 || o > n_objects) bad |= 8u;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
        bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (lo[k] != ~0u) atomicMax(bounds + 6 * c + k, ~lo[k]);
            if (hi[k] != 0u) atomicMax(bounds + 6 * c + 3 + k, hi[k]);
        }
        if (bad) atomicOr(status, bad);
    }
}

// words (int64): [0] status, [1..3] the largest bin of every axis over all chunks; one block
__global__ void __launch_bounds__(PR_THREADS) prune_bins_kernel(const unsigned* __restrict__ bounds,
                                                                int64_t n_chunks, float voxel,
                                                                const unsigned* __restrict__ status,
                                                                unsigned long long* __restrict__ words) {
    SPG_PDL_ENTRY();
    __shared__ unsigned long long s_max[3];
    __shared__ unsigned s_bad;
    if (threadIdx.x < 3) s_max[threadIdx.x] = 0ull;
    if (threadIdx.x == 0) s_bad = 0u;
    __syncthreads();
    for (int64_t c = threadIdx.x; c < n_chunks; c += blockDim.x) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const unsigned klo = ~__ldg(bounds + 6 * c + k), khi = __ldg(bounds + 6 * c + 3 + k);
            if (klo == ~0u) continue;  // no finite coordinate (reported by status 1)
            // the bins are monotone in x, so the chunk's largest bin is the bin of its maximum
            const float b = pr_binf(float_unkey(khi), float_unkey(klo), voxel);
            if (!(b < 4294967296.f)) {
                atomicOr(&s_bad, 2u);
                continue;
            }
            atomicMax(&s_max[k], (unsigned long long)(unsigned)b);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        words[0] = (unsigned long long)(__ldg(status) | s_bad);
        words[1] = s_max[0];
        words[2] = s_max[1];
        words[3] = s_max[2];
    }
}

// ------------------------------------------------------------------------------------------------ keys
// pass 0: the low 64 bits of every point's key and its index; pass 1: the high bits of the points in the order of
// the first sort
template <int kPass>
__global__ void __launch_bounds__(PR_THREADS) prune_keys_kernel(const PruneGeom g, const int32_t* __restrict__ order,
                                                                uint64_t* __restrict__ keys,
                                                                int32_t* __restrict__ idx) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.n) return;
    const int64_t i = kPass == 0 ? p : (int64_t)__ldg(order + p);
    uint64_t lo, hi;
    pr_key(g, i, lo, hi);
    keys[p] = kPass == 0 ? lo : hi;
    if (kPass == 0) idx[p] = (int32_t)i;
}

// ------------------------------------------------------------------------------------------------ rows
// head[p] = 1 where sorted position p starts a run; first[i] = the same flag at the point's own index
__global__ void __launch_bounds__(PR_THREADS) prune_heads_kernel(const PruneGeom g, const int32_t* __restrict__ order,
                                                                 int32_t* __restrict__ head,
                                                                 int32_t* __restrict__ first) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.n) return;
    const int64_t i = __ldg(order + p);
    int h = 1;
    if (p > 0) {
        uint64_t lo, hi, plo, phi;
        pr_key(g, i, lo, hi);
        pr_key(g, __ldg(order + p - 1), plo, phi);
        h = (lo != plo || hi != phi) ? 1 : 0;
    }
    head[p] = h;
    first[i] = h;
}

// for every run r (inclusive scan of head - 1): run_start[r] = its first sorted position, run_row[r] = its output
// row (the exclusive scan of `first` at its first point); run_start[m] = n, n_voxels[0] = m
__global__ void __launch_bounds__(PR_THREADS) prune_runs_kernel(const int32_t* __restrict__ order,
                                                                const int32_t* __restrict__ head,
                                                                const int32_t* __restrict__ run_of,
                                                                const int32_t* __restrict__ row_of, int64_t n,
                                                                int32_t* __restrict__ run_start,
                                                                int32_t* __restrict__ run_row,
                                                                int64_t* __restrict__ n_voxels) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    if (__ldg(head + p)) {
        const int r = __ldg(run_of + p) - 1;
        run_start[r] = (int32_t)p;
        run_row[r] = __ldg(row_of + __ldg(order + p));
    }
    if (p == n - 1) {
        const int m = __ldg(run_of + p);
        run_start[m] = (int32_t)n;
        n_voxels[0] = m;
    }
}

// ------------------------------------------------------------------------------------------------ reduce
__global__ void __launch_bounds__(PR_THREADS) prune_gather_kernel(const float* __restrict__ xyz,
                                                                  const uint8_t* __restrict__ rgb,
                                                                  const int32_t* __restrict__ order, int64_t n,
                                                                  float* __restrict__ xyz_s,
                                                                  uint32_t* __restrict__ rgb_s) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t i = __ldg(order + p);
    xyz_s[3 * p] = __ldg(xyz + 3 * i);
    xyz_s[3 * p + 1] = __ldg(xyz + 3 * i + 1);
    xyz_s[3 * p + 2] = __ldg(xyz + 3 * i + 2);
    rgb_s[p] = (uint32_t)__ldg(rgb + 3 * i) | ((uint32_t)__ldg(rgb + 3 * i + 1) << 8) |
               ((uint32_t)__ldg(rgb + 3 * i + 2) << 16);
}

// one thread per voxel: ply_c.cpp:254-259 (acc += x in point order from 0.f, uint32 colour sums) and :364-375
// (pos / (float)count, (uint8)((float)col / count))
__global__ void __launch_bounds__(PR_THREADS) prune_reduce_kernel(const float* __restrict__ xyz_s,
                                                                  const uint32_t* __restrict__ rgb_s,
                                                                  const int32_t* __restrict__ run_start,
                                                                  const int32_t* __restrict__ run_row, int64_t m,
                                                                  float* __restrict__ xyz_out,
                                                                  uint8_t* __restrict__ rgb_out) {
    SPG_PDL_ENTRY();
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= m) return;
    const int64_t s0 = __ldg(run_start + r), s1 = __ldg(run_start + r + 1);
    float ax = 0.f, ay = 0.f, az = 0.f;
    uint32_t cr = 0u, cg = 0u, cb = 0u;
    int64_t p = s0;
    constexpr int U = 8;  // loads issued ahead of the dependent adds; the adds stay in point order
    for (; p + U <= s1; p += U) {
        float x[U], y[U], z[U];
        uint32_t c[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            x[u] = __ldg(xyz_s + 3 * (p + u));
            y[u] = __ldg(xyz_s + 3 * (p + u) + 1);
            z[u] = __ldg(xyz_s + 3 * (p + u) + 2);
            c[u] = __ldg(rgb_s + p + u);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            ax = __fadd_rn(ax, x[u]);
            ay = __fadd_rn(ay, y[u]);
            az = __fadd_rn(az, z[u]);
            cr += c[u] & 0xffu;
            cg += (c[u] >> 8) & 0xffu;
            cb += c[u] >> 16;
        }
    }
    for (; p < s1; ++p) {
        ax = __fadd_rn(ax, __ldg(xyz_s + 3 * p));
        ay = __fadd_rn(ay, __ldg(xyz_s + 3 * p + 1));
        az = __fadd_rn(az, __ldg(xyz_s + 3 * p + 2));
        const uint32_t c = __ldg(rgb_s + p);
        cr += c & 0xffu;
        cg += (c >> 8) & 0xffu;
        cb += c >> 16;
    }
    const float cnt = __uint2float_rn((unsigned)(s1 - s0));
    const int64_t row = __ldg(run_row + r);
    xyz_out[3 * row] = __fdiv_rn(ax, cnt);
    xyz_out[3 * row + 1] = __fdiv_rn(ay, cnt);
    xyz_out[3 * row + 2] = __fdiv_rn(az, cnt);
    rgb_out[3 * row] = (uint8_t)__float2uint_rz(__fdiv_rn(__uint2float_rn(cr), cnt));
    rgb_out[3 * row + 1] = (uint8_t)__float2uint_rz(__fdiv_rn(__uint2float_rn(cg), cnt));
    rgb_out[3 * row + 2] = (uint8_t)__float2uint_rz(__fdiv_rn(__uint2float_rn(cb), cnt));
}

// the histograms over sorted positions: lanes that hit the same (row, value) add once, through their leader
__device__ __forceinline__ void pr_hist_add(int64_t* out, int64_t cols, int64_t row, int64_t v, bool on) {
    const unsigned long long slot = on ? (unsigned long long)(row * cols + v) : ~0ull;
    const unsigned act = __activemask();
    const unsigned peers = __match_any_sync(act, slot);
    if (on && (threadIdx.x & 31) == __ffs(peers) - 1)
        atomicAdd(reinterpret_cast<unsigned long long*>(out) + slot, (unsigned long long)__popc(peers));
}

__global__ void __launch_bounds__(PR_THREADS) prune_hist_kernel(const int32_t* __restrict__ order,
                                                                const int32_t* __restrict__ run_of,
                                                                const int32_t* __restrict__ run_row, int64_t n,
                                                                const int64_t* __restrict__ labels, int n_labels,
                                                                const int64_t* __restrict__ objects, int n_objects,
                                                                int64_t* __restrict__ labels_out,
                                                                int64_t* __restrict__ objects_out) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p - (threadIdx.x & 31) >= n) return;  // whole warps only: the lanes past n take part without adding
    const bool in = p < n;
    int64_t row = 0, l = 0, o = 0;
    if (in) {
        const int64_t i = __ldg(order + p);
        row = __ldg(run_row + __ldg(run_of + p) - 1);
        l = __ldg(labels + i);
        if (objects) o = __ldg(objects + i);
    }
    pr_hist_add(labels_out, (int64_t)n_labels + 1, row, l, in && l >= 0 && l <= n_labels);
    if (objects) pr_hist_add(objects_out, (int64_t)n_objects + 1, row, o, in && o >= 0 && o <= n_objects);
}

// ------------------------------------------------------------------------------------------------ plan
struct PruneWs {
    unsigned *bounds, *status;
    uint64_t *keys_in, *keys;
    int32_t *idx_in, *idx, *head, *first, *run_of, *row_of, *run_start, *run_row;
    float* xyz_s;
    uint32_t* rgb_s;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n, int64_t n_chunks, void* base, PruneWs* w) {
    const int m = (int)(n > 0 ? n : 1);
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int32_t*)nullptr, (int32_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::InclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, m);
    const size_t N = (size_t)m, C = (size_t)(n_chunks > 0 ? n_chunks : 1);
    Planner p(base);
    w->bounds = p.take<unsigned>(C * 6);
    w->status = p.take<unsigned>(1);
    w->keys_in = p.take<uint64_t>(N);
    w->keys = p.take<uint64_t>(N);
    w->idx_in = p.take<int32_t>(N);
    w->idx = p.take<int32_t>(N);
    w->head = p.take<int32_t>(N);
    w->first = p.take<int32_t>(N);
    w->run_of = p.take<int32_t>(N);
    w->row_of = p.take<int32_t>(N);
    w->run_start = p.take<int32_t>(N + 1);
    w->run_row = p.take<int32_t>(N);
    w->xyz_s = p.take<float>(3 * N);
    w->rgb_s = p.take<uint32_t>(N);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

static int pr_bits(int64_t v) {
    int b = 0;
    while (b < 63 && (v >> b) != 0) ++b;
    return b;
}

static int64_t pr_chunks(int64_t n, int64_t chunk_rows) { return (n + chunk_rows - 1) / chunk_rows; }

// the chunk rows and the workspace of one call
static int pr_setup(int64_t n, int64_t chunk_rows, void* workspace, int64_t workspace_bytes, PruneWs* w,
                    int64_t* rows) {
    if (n <= 0 || chunk_rows < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    *rows = chunk_rows == 0 || chunk_rows > n ? n : chunk_rows;
    const int rc = layout(n, pr_chunks(n, *rows), workspace, w);
    return rc == SPG_OK ? ws_check(workspace, workspace_bytes, w->bytes) : rc;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_prune_workspace(int64_t n, int64_t chunk_rows, int64_t* bytes) {
    if (!bytes || n <= 0 || chunk_rows < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    const int64_t rows = chunk_rows == 0 || chunk_rows > n ? n : chunk_rows;
    PruneWs w;
    const int rc = layout(n, pr_chunks(n, rows), nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_prune_bounds(const float* xyz, int64_t n, int64_t chunk_rows, float voxel_size, const int64_t* labels,
                     int n_labels, const int64_t* objects, int n_objects, void* workspace, int64_t workspace_bytes,
                     int64_t* words, spg_stream_t stream) {
    if (!xyz || !words || !(voxel_size > 0.f) || n_labels < 0 || n_objects < 0 || (n_labels > 0 && !labels) ||
        (n_labels > 0 && n_objects > 0 && !objects))
        return SPG_E_BADARG;
    PruneWs w;
    int64_t rows;
    const int rc = pr_setup(n, chunk_rows, workspace, workspace_bytes, &w, &rows);
    if (rc != SPG_OK) return rc;
    const int64_t C = pr_chunks(n, rows);
    if (C > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(w.bounds, 0, (size_t)C * 6 * 4, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.status, 0, 4, s);
    if (e != cudaSuccess) return (int)e;
    const int64_t per = ceil_div64(rows, PR_THREADS);
    const int64_t cap = (4 * kNumSMs + C - 1) / C;
    const dim3 grid((unsigned)(per < cap ? per : cap), (unsigned)C);
    const bool with_labels = n_labels > 0;
    SPG_LAUNCH(K_PRUNE_BOUNDS, s, prune_bounds_kernel, grid, PR_THREADS, 0, xyz, n, rows,
               with_labels ? labels : (const int64_t*)nullptr,
               with_labels && n_objects > 0 ? objects : (const int64_t*)nullptr, n_labels, n_objects, w.bounds,
               w.status);
    SPG_LAUNCH(K_PRUNE_BOUNDS, s, prune_bins_kernel, 1, PR_THREADS, 0, (const unsigned*)w.bounds, C, voxel_size,
               (const unsigned*)w.status, (unsigned long long*)words);
    return launch_status();
}

int spg_prune_voxels(const float* xyz, int64_t n, int64_t chunk_rows, float voxel_size, int64_t max_bin_x,
                     int64_t max_bin_y, int64_t max_bin_z, void* workspace, int64_t workspace_bytes,
                     int64_t* n_voxels, spg_stream_t stream) {
    if (!xyz || !n_voxels || !(voxel_size > 0.f) || max_bin_x < 0 || max_bin_y < 0 || max_bin_z < 0 ||
        max_bin_x > 0xffffffffll || max_bin_y > 0xffffffffll || max_bin_z > 0xffffffffll)
        return SPG_E_BADARG;
    PruneWs w;
    int64_t rows;
    int rc = pr_setup(n, chunk_rows, workspace, workspace_bytes, &w, &rows);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    PruneGeom g;
    g.xyz = xyz;
    g.n = n;
    g.chunk_rows = rows;
    g.voxel = voxel_size;
    g.bounds = w.bounds;
    g.bits_x = pr_bits(max_bin_x);
    g.bits_y = pr_bits(max_bin_y);
    g.bits_z = pr_bits(max_bin_z);
    g.bits_total = pr_bits(pr_chunks(n, rows) - 1) + g.bits_x + g.bits_y + g.bits_z;
    const unsigned blocks = (unsigned)ceil_div64(n, PR_THREADS);
    const int N = (int)n;
    SPG_LAUNCH(K_PRUNE_KEYS, s, prune_keys_kernel<0>, blocks, PR_THREADS, 0, g, (const int32_t*)nullptr, w.keys_in,
               w.idx_in);
    const int lo_bits = g.bits_total < 64 ? (g.bits_total > 0 ? g.bits_total : 1) : 64;
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.keys_in, w.keys, (const int32_t*)w.idx_in,
            w.idx, N, 0, lo_bits, s);
    const int32_t* order = w.idx;
    if (g.bits_total > 64) {  // LSD: the high bits last, stable, carrying the order of the first sort
        SPG_LAUNCH(K_PRUNE_KEYS, s, prune_keys_kernel<1>, blocks, PR_THREADS, 0, g, (const int32_t*)w.idx, w.keys_in,
                   (int32_t*)nullptr);
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.keys_in, w.keys, (const int32_t*)w.idx,
                w.idx_in, N, 0, g.bits_total - 64, s);
        order = w.idx_in;
    }
    SPG_LAUNCH(K_PRUNE_ROWS, s, prune_heads_kernel, blocks, PR_THREADS, 0, g, order, w.head, w.first);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.first, w.row_of, N, s);
    SPG_CUB(w.cub, cub::DeviceScan::InclusiveSum, (const int32_t*)w.head, w.run_of, N, s);
    // the final order goes to `idx` whichever sort produced it, for the reduce
    if (order != w.idx) {
        const cudaError_t e = cudaMemcpyAsync(w.idx, order, (size_t)n * 4, cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return (int)e;
    }
    SPG_LAUNCH(K_PRUNE_ROWS, s, prune_runs_kernel, blocks, PR_THREADS, 0, (const int32_t*)w.idx,
               (const int32_t*)w.head, (const int32_t*)w.run_of, (const int32_t*)w.row_of, n, w.run_start, w.run_row,
               n_voxels);
    return launch_status();
}

int spg_prune_reduce(const float* xyz, const uint8_t* rgb, const int64_t* labels, int n_labels,
                     const int64_t* objects, int n_objects, int64_t n, int64_t chunk_rows, const void* workspace,
                     int64_t workspace_bytes, int64_t n_voxels, float* xyz_out, uint8_t* rgb_out,
                     int64_t* labels_out, int64_t* objects_out, spg_stream_t stream) {
    if (!xyz || !rgb || !xyz_out || !rgb_out || !labels_out || !objects_out || n_labels < 0 || n_objects < 0 ||
        n_voxels <= 0 || n_voxels > n || (n_labels > 0 && !labels) || (n_labels > 0 && n_objects > 0 && !objects))
        return SPG_E_BADARG;
    PruneWs w;
    int64_t rows;
    const int rc = pr_setup(n, chunk_rows, const_cast<void*>(workspace), workspace_bytes, &w, &rows);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(labels_out, 0, (size_t)n_voxels * (n_labels + 1) * 8, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(objects_out, 0, (size_t)n_voxels * (n_objects + 1) * 8, s);
    if (e != cudaSuccess) return (int)e;
    const unsigned blocks = (unsigned)ceil_div64(n, PR_THREADS);
    SPG_LAUNCH(K_PRUNE_REDUCE, s, prune_gather_kernel, blocks, PR_THREADS, 0, xyz, rgb, w.idx, n, w.xyz_s, w.rgb_s);
    SPG_LAUNCH(K_PRUNE_REDUCE, s, prune_reduce_kernel, (unsigned)ceil_div64(n_voxels, PR_THREADS), PR_THREADS, 0,
               (const float*)w.xyz_s, (const uint32_t*)w.rgb_s, w.run_start, w.run_row, n_voxels, xyz_out, rgb_out);
    // ply_c.cpp:343-354: the labels counted when n_labels > 0, the objects only with them
    if (n_labels > 0)
        SPG_LAUNCH(K_PRUNE_REDUCE, s, prune_hist_kernel, blocks, PR_THREADS, 0, w.idx, w.run_of, w.run_row, n, labels,
                   n_labels, n_objects > 0 ? objects : (const int64_t*)nullptr, n_objects, labels_out, objects_out);
    return launch_status();
}

}  // extern "C"
