// ECC-CRF: the mean-field recurrence of ECC_CRFModule (ref: learning/modules.py:185-202) at the
// class-count widths it runs at (C <= 32, matrix filters [E, C, C], float32, no idxe).
//
// The reference evaluates the filter network and a full GraphConvFunction in every iteration and
// materialises the [E, C] products; here one launch per iteration streams the filter bank once,
// reduces in registers and applies the softmax in the same warp that owns the row.  The backward
// iteration walks the source-sorted CSR (as ecc_mat_bwd_x_kernel), so no atomics are needed and
// the summation order is fixed (deterministic).
//
// Lane mapping, one warp per row:
//   NARROW (C <= 16): lane = (h = lane>>4, o = lane&15); the half-warps take alternate rows
//                     k = 2i+h of W_e, so one load instruction reads rows 2i, 2i+1: 2C contiguous
//                     floats, whatever the alignment of C*C.
//   WIDE (16 < C <= 32): lane o, rows k = 0..C-1, C contiguous floats per load instruction.
#include <math.h>

#include "common.cuh"

namespace spg {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kCrfMaxC = 32;

template <bool NARROW>
struct CrfLanes {
    static constexpr int kRows = NARROW ? 8 : 32;  // filter rows per lane
    int h, o;
    bool col;    // lane holds a valid column o < C
    bool owner;  // lane writes column o of the row (one half only when NARROW)
    __device__ CrfLanes(int lane, int C) {
        h = NARROW ? lane >> 4 : 0;
        o = NARROW ? lane & 15 : lane;
        col = o < C;
        owner = col && h == 0;
    }
    __device__ int row(int i) const { return NARROW ? 2 * i + h : i; }
    // rows i of this lane that can exist (warp-uniform bound: both halves stop at the same i)
    __device__ static bool done(int i, int C) { return NARROW ? 2 * i >= C : i >= C; }
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
    return v;
}

// softmax over the owner lanes of a row; every lane gets its column's value (0 where !owner)
__device__ __forceinline__ float row_softmax(float z, bool owner) {
    const float m = warp_max(owner ? z : -INFINITY);
    const float ex = owner ? expf(z - m) : 0.f;
    return ex / warp_sum(ex);
}

template <bool NARROW>
__global__ void __launch_bounds__(256)
crf_fwd_kernel(const float* __restrict__ U, const float* __restrict__ Q, const float* __restrict__ W,
               const int* __restrict__ rowptr, const int* __restrict__ idxn, float* __restrict__ out,
               int n, int C, int do_softmax) {
    SPG_PDL_ENTRY();
    using L = CrfLanes<NARROW>;
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n) return;  // whole warp exits together
    const L ln(lane, C);
    const int64_t CC = (int64_t)C * C;
    const int beg = rowptr[node], end = rowptr[node + 1];
    float acc = 0.f;
    for (int e = beg; e < end; ++e) {
        const int s = __ldg(idxn + e);
        const float* We = W + (int64_t)e * CC;
        float wv[L::kRows];
#pragma unroll
        for (int i = 0; i < L::kRows; ++i) {
            if (L::done(i, C)) break;
            const int k = ln.row(i);
            wv[i] = (k < C && ln.col) ? __ldg(We + k * C + ln.o) : 0.f;
        }
        const float qv = ln.col ? __ldg(Q + (int64_t)s * C + ln.o) : 0.f;  // lane o holds Q[s, o]
#pragma unroll
        for (int i = 0; i < L::kRows; ++i) {
            if (L::done(i, C)) break;
            acc = fmaf(__shfl_sync(kFull, qv, ln.row(i)), wv[i], acc);
        }
    }
    if (NARROW) acc += __shfl_xor_sync(kFull, acc, 16);  // even + odd rows
    const int deg = end - beg;
    const int64_t at = node * C + ln.o;
    const float z = ln.col ? __ldg(U + at) - (deg > 0 ? acc / (float)deg : 0.f) : 0.f;
    const float v = do_softmax ? row_softmax(z, ln.owner) : z;
    if (ln.owner) out[at] = v;
}

template <bool NARROW>
__global__ void __launch_bounds__(256)
crf_bwd_kernel(const float* __restrict__ W, const float* __restrict__ G, const float* __restrict__ Q,
               const float* du_in, float* du_out, float* __restrict__ g_out,
               const int* __restrict__ tgt_rowptr, const int* __restrict__ src_rowptr,
               const int* __restrict__ src_perm, const int* __restrict__ edge_tgt, int n, int C) {
    SPG_PDL_ENTRY();
    using L = CrfLanes<NARROW>;
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n) return;
    const L ln(lane, C);
    const int64_t CC = (int64_t)C * C;
    const int beg = src_rowptr[node], end = src_rowptr[node + 1];
    float acc[L::kRows];  // acc[i]: partial of dQ[row(i)] over this lane's column o
#pragma unroll
    for (int i = 0; i < L::kRows; ++i) acc[i] = 0.f;
    for (int p = beg; p < end; ++p) {
        const int e = __ldg(src_perm + p);
        const int tg = __ldg(edge_tgt + e);
        const float* We = W + (int64_t)e * CC;
        float wv[L::kRows];
#pragma unroll
        for (int i = 0; i < L::kRows; ++i) {
            if (L::done(i, C)) break;
            const int k = ln.row(i);
            wv[i] = (k < C && ln.col) ? __ldg(We + k * C + ln.o) : 0.f;
        }
        const float inv = 1.f / (float)(__ldg(tgt_rowptr + tg + 1) - __ldg(tgt_rowptr + tg));
        const float gv = ln.col ? __ldg(G + (int64_t)tg * C + ln.o) * inv : 0.f;
#pragma unroll
        for (int i = 0; i < L::kRows; ++i) {
            if (L::done(i, C)) break;
            acc[i] = fmaf(wv[i], gv, acc[i]);
        }
    }
    // reduce every row over the columns o (the lanes of a half-warp, or of the warp)
    float mine = 0.f;  // dQ[o] on lane o
#pragma unroll
    for (int i = 0; i < L::kRows; ++i) {
        if (L::done(i, C)) break;
        float v = acc[i];
#pragma unroll
        for (int off = NARROW ? 8 : 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
        if (NARROW) {
            // row 2i+h is complete on every lane of half h; lane o takes row o from half o&1
            v = __shfl_sync(kFull, v, (ln.o & 1) * 16);
            if ((ln.o >> 1) == i) mine = v;
        } else if (ln.o == i) {
            mine = v;
        }
    }
    const int64_t at = node * C + ln.o;
    const float q = ln.col ? __ldg(Q + at) : 0.f;
    const float dot = warp_sum(ln.owner ? mine * q : 0.f);
    const float dz = q * (mine - dot);
    if (ln.owner) {
        du_out[at] = du_in[at] + dz;
        if (g_out) g_out[at] = -dz;
    }
}

// Row softmax (g == NULL) or its backward x * (g - <g, x>) with x the softmax output.
__global__ void __launch_bounds__(256)
crf_softmax_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ out,
                   int n, int C) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n) return;
    const bool owner = lane < C;
    const int64_t at = node * C + lane;
    const float v = owner ? __ldg(x + at) : 0.f;
    float r;
    if (g == nullptr) {
        r = row_softmax(v, owner);
    } else {
        const float gv = owner ? __ldg(g + at) : 0.f;
        r = v * (gv - warp_sum(gv * v));
    }
    if (owner) out[at] = r;
}

static inline int crf_check(int64_t n, int64_t n_edges, int C) {
    if (n < 0 || n_edges < 0 || C <= 0) return SPG_E_BADARG;
    if (C > kCrfMaxC) return SPG_E_UNSUPPORTED;
    if (n >= (1ll << 31) || n_edges >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_crf_softmax(const float* x, const float* g, float* out, int64_t n, int C, spg_stream_t stream) {
    if (int rc = crf_check(n, 0, C)) return rc;
    if (n == 0) return SPG_OK;
    if (!x || !out) return SPG_E_BADARG;
    SPG_LAUNCH(K_CRF_SOFTMAX, (cudaStream_t)stream, crf_softmax_kernel, (unsigned)ceil_div64(n * 32, 256), 256,
               0, x, g, out, (int)n, C);
    return launch_status();
}

int spg_crf_fwd_step(const float* u, const float* q_prev, const float* w, const int32_t* tgt_rowptr,
                     const int32_t* idxn, float* out, int64_t n, int64_t n_edges, int C, int do_softmax,
                     spg_stream_t stream) {
    if (int rc = crf_check(n, n_edges, C)) return rc;
    if (n == 0) return SPG_OK;
    if (!u || !q_prev || !tgt_rowptr || !out || (n_edges > 0 && (!w || !idxn))) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)ceil_div64(n * 32, 256);
    if (C <= 16) {
        SPG_LAUNCH(K_CRF_FWD, s, crf_fwd_kernel<true>, blocks, 256, 0, u, q_prev, w, tgt_rowptr, idxn, out,
                   (int)n, C, do_softmax);
    } else {
        SPG_LAUNCH(K_CRF_FWD, s, crf_fwd_kernel<false>, blocks, 256, 0, u, q_prev, w, tgt_rowptr, idxn, out,
                   (int)n, C, do_softmax);
    }
    return launch_status();
}

int spg_crf_bwd_step(const float* w, const float* gp, const float* q_prev, const float* du_in, float* du_out,
                     float* gp_out, const int32_t* tgt_rowptr, const int32_t* src_rowptr,
                     const int32_t* src_perm, const int32_t* edge_tgt, int64_t n, int64_t n_edges, int C,
                     spg_stream_t stream) {
    if (int rc = crf_check(n, n_edges, C)) return rc;
    if (n == 0) return SPG_OK;
    if (!q_prev || !du_in || !du_out || !tgt_rowptr || !src_rowptr) return SPG_E_BADARG;
    if (n_edges > 0 && (!w || !gp || !src_perm || !edge_tgt)) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)ceil_div64(n * 32, 256);
    if (C <= 16) {
        SPG_LAUNCH(K_CRF_BWD, s, crf_bwd_kernel<true>, blocks, 256, 0, w, gp, q_prev, du_in, du_out, gp_out,
                   tgt_rowptr, src_rowptr, src_perm, edge_tgt, (int)n, C);
    } else {
        SPG_LAUNCH(K_CRF_BWD, s, crf_bwd_kernel<false>, blocks, 256, 0, w, gp, q_prev, du_in, du_out, gp_out,
                   tgt_rowptr, src_rowptr, src_perm, edge_tgt, (int)n, C);
    }
    return launch_status();
}

}  // extern "C"
