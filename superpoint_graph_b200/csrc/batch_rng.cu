// Device draws of the superpoint graph's batch, for spg_loader.load_batch(device_rng=True): the shuffle and the
// centre sample of `loader` (ref: learning/spg.py:117,135-137), the resample of `load_superpoint` (:209-214) and
// `augment_cloud`'s matrix and jitter (:240-257).  The distributions are the reference's; the streams are
// Philox4x32-10 (philox.cuh) instead of Python's and numpy's MT19937, so no host generator is read or advanced.
//
// Counter layout.  Key = (seed lo, seed hi).  A stream is (a, b, purpose); its 64-bit draw k is
//   Philox(c0 = k >> 1, c1 = a, c2 = b, c3 = purpose), words (2(k & 1), 2(k & 1) + 1) as (low, high)
// and the purposes are 1 permutation, 2 centres, 3 resample, 4 augmentation, 5 jitter, each its own counter word:
//   permutation / centres   (a, b) = (0, graph position in the batch); draw v: the sort key of vertex v (new id v)
//   resample, training      (a, b) = (superpoint id, graph position); draw j: output point j
//   augmentation            same (a, b); draws 0 scale, 1 angle, 2 mirror x, 3 mirror y
//   jitter                  same (a, b); element k = (point j, attribute f), k = j F + f, takes draws 2k and 2k + 1
//   resample, evaluation    (a, b) = (low, high word of id + test_seed_offset), purpose 3 | 0x100
// u53(x) = (x >> 11) 2^-53 is uniform in [0, 1); an index below n is the high word of the 128-bit x n.
//
//   sb_draw        the permutation and centre keys of one graph (CUB then radix-sorts (key, vertex) pairs stably)
//   sb_perm        perm[v] = rank of v's key (igraph's permute_vertices argument), centres = the nneigh smallest
//   sb_flags       each kept vertex's first row and point count from the store's dense index, its clouds_flag, and
//                  the stable compaction of the valid clouds of the whole batch
//   sb_cloud_draw  resample indices [Nv, L], matrices [Nv, 9] (float64, augment_matrix's order), jitter [Nv, L, F]
#include <cub/cub.cuh>

#include "philox.cuh"
#include "workspace.cuh"

namespace spg {

constexpr int BR_THREADS = 256;
constexpr int kCloudDrawThreads = 128;
enum : uint32_t { kPurposePerm = 1, kPurposeCentres = 2, kPurposeResample = 3, kPurposeAugment = 4,
                  kPurposeJitter = 5, kPurposeEval = 0x100 };

__device__ __forceinline__ uint64_t draw64(uint64_t seed, uint32_t a, uint32_t b, uint32_t purpose, uint64_t k) {
    const Philox4 w = philox4x32_10((uint32_t)(k >> 1), a, b, purpose, (uint32_t)seed, (uint32_t)(seed >> 32));
    return (k & 1) ? ((uint64_t)w.v[3] << 32 | w.v[2]) : ((uint64_t)w.v[1] << 32 | w.v[0]);
}

__device__ __forceinline__ double u53(uint64_t x) { return (double)(x >> 11) * 0x1.0p-53; }

__global__ void __launch_bounds__(BR_THREADS)
sb_draw_kernel(uint64_t seed, uint32_t graph_pos, int64_t n, int permute, int centres,
               unsigned long long* __restrict__ perm_keys, unsigned long long* __restrict__ centre_keys,
               int* __restrict__ iota) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    iota[v] = (int)v;
    if (permute) perm_keys[v] = draw64(seed, 0u, graph_pos, kPurposePerm, (uint64_t)v);
    if (centres) centre_keys[v] = draw64(seed, 0u, graph_pos, kPurposeCentres, (uint64_t)v);
}

__global__ void __launch_bounds__(BR_THREADS)
sb_perm_kernel(const int* __restrict__ perm_order, int64_t n, const int* __restrict__ centre_order,
               int64_t n_centres, int* __restrict__ perm, int* __restrict__ centres) {
    SPG_PDL_ENTRY();
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (perm_order && r < n) perm[perm_order[r]] = (int)r;
    if (r < n_centres) centres[r] = centre_order[r];
}

// position i of one graph's slice: kept vertex i (i < selected[0]) or padding
__global__ void __launch_bounds__(BR_THREADS)
sb_cloud_flags_kernel(const int* __restrict__ selected, int64_t n, uint32_t graph_pos,
                      const int64_t* __restrict__ sp_first_row, const int* __restrict__ sp_count, int64_t n_ids,
                      int64_t minpts, int* __restrict__ flags, int* __restrict__ valid, int64_t* __restrict__ first_row,
                      int* __restrict__ count, int64_t* __restrict__ key) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int flag = -1, cnt = 0;
    int64_t row = 0, id = 0;
    if (i < selected[0]) {
        id = selected[2 + i];
        cnt = id < n_ids ? sp_count[id] : -1;
        if (cnt < 0) {
            flag = -2;  // not in the store
        } else {
            row = sp_first_row[id];
            flag = cnt < minpts ? -1 : 0;
        }
    }
    flags[i] = flag;
    valid[i] = selected[1] > 0 && flag == 0;  // only graphs with edges make clouds
    first_row[i] = row;
    count[i] = cnt;
    key[i] = (int64_t)((uint64_t)graph_pos << 32 | (uint64_t)id);
}

__global__ void __launch_bounds__(BR_THREADS)
sb_cloud_compact_kernel(const int* __restrict__ valid, const int* __restrict__ pos, int64_t n,
                        const int64_t* __restrict__ first_row, const int* __restrict__ count,
                        const int64_t* __restrict__ key, int64_t* __restrict__ start_out, int* __restrict__ count_out,
                        int64_t* __restrict__ key_out) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !valid[i]) return;
    const int p = pos[i];
    start_out[p] = first_row[i];
    count_out[p] = count[i];
    key_out[p] = key[i];
}

struct CloudDrawArgs {
    const int64_t* key;  // [Nv] (graph position << 32) | superpoint id
    const int* count;    // [Nv] points of the superpoint
    int L, F, train;
    uint64_t seed;
    int64_t test_seed_offset;
    double scale, mirror_half;
    int rotate;
    int* sample_idx;  // [Nv, L]
    double* xform;    // [Nv, 9] or null
    float* jitter;    // [Nv, L, F] or null
};

// a block per cloud
__global__ void __launch_bounds__(kCloudDrawThreads) sb_cloud_draw_kernel(const CloudDrawArgs a, int64_t nv) {
    SPG_PDL_ENTRY();
    const int64_t c = blockIdx.x;
    if (c >= nv) return;
    const uint64_t key = (uint64_t)a.key[c];
    uint32_t sa, sb, resample = kPurposeResample;
    if (a.train) {
        sa = (uint32_t)key;
        sb = (uint32_t)(key >> 32);
    } else {
        const uint64_t e = (uint64_t)((int64_t)(uint32_t)key + a.test_seed_offset);
        sa = (uint32_t)e;
        sb = (uint32_t)(e >> 32);
        resample |= kPurposeEval;
    }
    const int n = a.count[c], L = a.L;
    for (int j = threadIdx.x; j < L; j += blockDim.x) {
        int r = j;  // n == L: as is; n < L: the original points first (spg.py:209-214)
        if (n > L || j >= n) r = (int)__umul64hi(draw64(a.seed, sa, sb, resample, (uint64_t)j), (uint64_t)n);
        a.sample_idx[c * L + j] = r;
    }
    if (a.xform && threadIdx.x == 0) {
        // augment_matrix (spg.py:240-253): s I, then R(angle) . M, then the two reflections; every entry of each
        // product has one non-zero term, so the float64 entries are numpy's
        double s = 1.0, cs = 1.0, sn = 0.0;
        if (a.scale > 1.0) {
            const double lo = __ddiv_rn(1.0, a.scale);
            s = __dadd_rn(lo, __dmul_rn(__dsub_rn(a.scale, lo), u53(draw64(a.seed, sa, sb, kPurposeAugment, 0))));
        }
        if (a.rotate) sincos(__dmul_rn(2.0 * M_PI, u53(draw64(a.seed, sa, sb, kPurposeAugment, 1))), &sn, &cs);
        double M[9] = {__dmul_rn(cs, s), __dmul_rn(-sn, s), 0.0, __dmul_rn(sn, s), __dmul_rn(cs, s), 0.0, 0.0, 0.0, s};
        if (a.mirror_half > 0.0) {
#pragma unroll
            for (int m = 0; m < 2; ++m)
                if (u53(draw64(a.seed, sa, sb, kPurposeAugment, 2 + m)) < a.mirror_half)
#pragma unroll
                    for (int k = 0; k < 3; ++k) M[3 * m + k] = -M[3 * m + k];
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) a.xform[c * 9 + k] = M[k];
    }
    if (a.jitter) {
        // clip(0.01 N(0, 1), +-0.05) (spg.py:255-257), Box-Muller in float64 on (1 - u53, u53)
        const int64_t LF = (int64_t)L * a.F;
        for (int64_t k = threadIdx.x; k < LF; k += blockDim.x) {
            const double u1 = __dsub_rn(1.0, u53(draw64(a.seed, sa, sb, kPurposeJitter, 2 * (uint64_t)k)));
            const double u2 = u53(draw64(a.seed, sa, sb, kPurposeJitter, 2 * (uint64_t)k + 1));
            const double g = __dmul_rn(sqrt(__dmul_rn(-2.0, log(u1))), cos(__dmul_rn(2.0 * M_PI, u2)));
            a.jitter[c * LF + k] = __double2float_rn(fmin(fmax(__dmul_rn(0.01, g), -0.05), 0.05));
        }
    }
}

struct DrawWs {
    unsigned long long *perm_keys, *centre_keys, *sorted_keys;
    int *iota, *perm_order, *centre_order;
    CubRegion cub;
    size_t bytes;
};

static int draw_layout(int64_t n, void* base, DrawWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const unsigned long long*)nullptr,
                  (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr, (int)n);
    Planner p(base);
    w->perm_keys = p.take<unsigned long long>(n);
    w->centre_keys = p.take<unsigned long long>(n);
    w->sorted_keys = p.take<unsigned long long>(n);
    w->iota = p.take<int>(n);
    w->perm_order = p.take<int>(n);
    w->centre_order = p.take<int>(n);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

struct CloudsWs {
    int* pos;
    CubRegion cub;
    size_t bytes;
};

static int clouds_layout(int64_t n, void* base, CloudsWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int*)nullptr, (int*)nullptr, (int)n);
    Planner p(base);
    w->pos = p.take<int>(n);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

static unsigned br_blocks(int64_t n) { return (unsigned)ceil_div64(n > 0 ? n : 1, BR_THREADS); }

}  // namespace spg

using namespace spg;

extern "C" {

int spg_batch_draw_workspace(int64_t n_ver, int64_t* bytes) {
    if (!bytes || n_ver < 0) return SPG_E_BADARG;
    if (too_big(n_ver)) return SPG_E_UNSUPPORTED;
    DrawWs w;
    const int rc = draw_layout(n_ver, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_batch_draw(int64_t n_ver, int64_t seed, int64_t graph_pos, int permute, int64_t n_centres, int32_t* perm,
                   int32_t* centres, void* workspace, int64_t workspace_bytes, spg_stream_t stream) {
    if (n_ver < 0 || n_centres < 0 || n_centres > n_ver || graph_pos < 0 || graph_pos > 0xffffffffll)
        return SPG_E_BADARG;
    if (too_big(n_ver)) return SPG_E_UNSUPPORTED;
    if ((permute && n_ver > 0 && !perm) || (n_centres > 0 && !centres)) return SPG_E_BADARG;
    DrawWs w;
    int rc = draw_layout(n_ver, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    permute = permute && n_ver > 0;
    if (!permute && n_centres == 0) return SPG_OK;
    cudaStream_t s = (cudaStream_t)stream;
    SPG_LAUNCH(K_SB_DRAW, s, sb_draw_kernel, br_blocks(n_ver), BR_THREADS, 0, (uint64_t)seed, (uint32_t)graph_pos,
               n_ver, permute, (int)(n_centres > 0), w.perm_keys, w.centre_keys, w.iota);
    // stable: equal keys keep vertex order, so the result is a permutation whatever the keys
    if (permute)
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const unsigned long long*)w.perm_keys, w.sorted_keys,
                (const int*)w.iota, w.perm_order, (int)n_ver, 0, 64, s);
    if (n_centres > 0)
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const unsigned long long*)w.centre_keys, w.sorted_keys,
                (const int*)w.iota, w.centre_order, (int)n_ver, 0, 64, s);
    SPG_LAUNCH(K_SB_PERM, s, sb_perm_kernel, br_blocks(permute ? n_ver : n_centres), BR_THREADS, 0,
               permute ? (const int*)w.perm_order : (const int*)nullptr, n_ver, (const int*)w.centre_order, n_centres,
               perm, centres);
    return launch_status();
}

int spg_batch_cloud_flags(const int32_t* selected, int64_t n_ver, int64_t graph_pos, const int64_t* sp_first_row,
                          const int32_t* sp_count, int64_t n_ids, int64_t minpts, int32_t* flags, int32_t* valid,
                          int64_t* first_row, int32_t* count, int64_t* key, spg_stream_t stream) {
    if (n_ver < 0 || n_ids < 0 || graph_pos < 0 || graph_pos > 0xffffffffll) return SPG_E_BADARG;
    if (too_big(n_ver)) return SPG_E_UNSUPPORTED;
    if (n_ver == 0) return SPG_OK;
    if (!selected || !flags || !valid || !first_row || !count || !key || (n_ids > 0 && (!sp_first_row || !sp_count)))
        return SPG_E_BADARG;
    SPG_LAUNCH(K_SB_FLAGS, (cudaStream_t)stream, sb_cloud_flags_kernel, br_blocks(n_ver), BR_THREADS, 0, selected,
               n_ver, (uint32_t)graph_pos, sp_first_row, sp_count, n_ids, minpts, flags, valid, first_row, count, key);
    return launch_status();
}

int spg_batch_clouds_workspace(int64_t n, int64_t* bytes) {
    if (!bytes || n < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    CloudsWs w;
    const int rc = clouds_layout(n, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_batch_clouds(const int32_t* valid, const int64_t* first_row, const int32_t* count, const int64_t* key,
                     int64_t n, void* workspace, int64_t workspace_bytes, int64_t* start_out, int32_t* count_out,
                     int64_t* key_out, spg_stream_t stream) {
    if (n < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    if (n > 0 && (!valid || !first_row || !count || !key || !start_out || !count_out || !key_out)) return SPG_E_BADARG;
    CloudsWs w;
    int rc = clouds_layout(n, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK || n == 0) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, valid, w.pos, (int)n, s);
    SPG_LAUNCH(K_SB_FLAGS, s, sb_cloud_compact_kernel, br_blocks(n), BR_THREADS, 0, valid, (const int*)w.pos, n,
               first_row, count, key, start_out, count_out, key_out);
    return launch_status();
}

int spg_batch_cloud_draw(const int64_t* key, const int32_t* count, int64_t n_clouds, int n_points, int n_attribs,
                         int64_t seed, int train, int64_t test_seed_offset, double scale, int rotate,
                         double mirror_prob, int32_t* sample_idx, double* xform, float* jitter, spg_stream_t stream) {
    if (n_clouds < 0 || n_points <= 0 || n_attribs <= 0) return SPG_E_BADARG;
    if (n_clouds > 0x7fffffffll) return SPG_E_UNSUPPORTED;
    if (n_clouds == 0) return SPG_OK;
    if (!key || !count || !sample_idx) return SPG_E_BADARG;
    CloudDrawArgs a;
    a.key = key;
    a.count = count;
    a.L = n_points;
    a.F = n_attribs;
    a.train = train;
    a.seed = (uint64_t)seed;
    a.test_seed_offset = test_seed_offset;
    a.scale = scale;
    a.mirror_half = mirror_prob / 2;
    a.rotate = rotate == 1;
    a.sample_idx = sample_idx;
    a.xform = xform;
    a.jitter = jitter;
    SPG_LAUNCH(K_SB_CLOUD_DRAW, (cudaStream_t)stream, sb_cloud_draw_kernel, (unsigned)n_clouds, kCloudDrawThreads, 0,
               a, n_clouds);
    return launch_status();
}

}  // extern "C"
