// Edge-conditioned convolution: gather - per-edge product - degree-normalised
// segment reduction over a target-sorted CSR, and its two gradients.
//
// What it computes follows the reference's GraphConvFunction
// (learning/ecc/GraphConvModule.py:43-152) and its conv_aggregate kernels
// (learning/ecc/cuda_kernels.py:55-139); how it computes it does not: the
// reference materialises the [E,C] products with index_select + bmm/mul and then
// walks them with one thread per channel.  Here every kernel streams the filter
// bank exactly once with 128-bit loads, keeps the running sum in registers and
// never materialises per-edge products; gradients w.r.t. the node features use a
// source-sorted CSR so that no atomics are needed (deterministic).
//
// HBM-bound integer/float streaming work: no tensor cores on purpose.
#include "ecc_rows.cuh"

namespace spg {

// ------------------------------------------------------------------ fast paths
// C == 32, float32, no idxe.  A row of x / w(vv) / out is 128 B = 8 lanes x float4.

// Vector filters: one warp per target node (ecc_rows.cuh).  x is read through the non-coherent
// path, the filter bank is streamed.
__global__ void __launch_bounds__(256)
ecc_vv_fwd_kernel(const float4* __restrict__ x, const float4* __restrict__ w,
                  const int* __restrict__ rowptr, const int* __restrict__ idxn,
                  float4* __restrict__ out, int n_out) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n_out) return;
    const float4 acc =
        ecc_vv_row_fwd<LdNc, LdCs>((const float*)x, w, idxn, rowptr[node], rowptr[node + 1], lane);
    if (lane < kG) out[node * kG + lane] = acc;  // slot 0: sub = lane
}

// Matrix filters W_e [32,32] (4 KB per edge): one warp per target node.  A warp
// reads one W_e with 8 x 512-B fully coalesced requests; lane = (r = lane>>3,
// q = lane&7) owns rows k = 4*it + r and columns 4q..4q+3.
__global__ void __launch_bounds__(256)
ecc_mat_fwd_kernel(const float* __restrict__ x, const float4* __restrict__ w,
                   const int* __restrict__ rowptr, const int* __restrict__ idxn,
                   float4* __restrict__ out, int n_out) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n_out) return;  // whole warp exits together
    const int r = lane >> 3, q = lane & 7;
    const int beg = rowptr[node], end = rowptr[node + 1];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = beg; e < end; ++e) {
        const int s = __ldg(idxn + e);
        const float4* W = w + (int64_t)e * 256;
        float4 wv[8];
#pragma unroll
        for (int it = 0; it < 8; ++it) wv[it] = ld_stream4(W + it * 32 + lane);
        const float xv = __ldg(x + (int64_t)s * kC + lane);
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const float xk = __shfl_sync(0xffffffffu, xv, it * 4 + r);
            acc.x = fmaf(xk, wv[it].x, acc.x);
            acc.y = fmaf(xk, wv[it].y, acc.y);
            acc.z = fmaf(xk, wv[it].z, acc.z);
            acc.w = fmaf(xk, wv[it].w, acc.w);
        }
    }
    acc = slot_reduce(acc);
    if (r == 0) {
        const int deg = end - beg;
        if (deg > 0) {
            const float d = (float)deg;
            acc.x /= d;
            acc.y /= d;
            acc.z /= d;
            acc.w /= d;
        }
        out[node * kG + q] = acc;
    }
}

// grad_w[e,:] (+)= (1/deg_t) * sum_r x_r[src_e,:] * g_r[t,:]   (vector filters)
__global__ void __launch_bounds__(256)
ecc_vv_bwd_w_kernel(const float4* __restrict__ xs, const float4* __restrict__ gs,
                    int64_t x_stride4, int64_t g_stride4, int n_iter,
                    const int* __restrict__ rowptr, const int* __restrict__ idxn,
                    float4* __restrict__ grad_w, int n_out, int accumulate) {
    SPG_PDL_ENTRY();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t node = t / kG;
    const int sub = (int)(t % kG);
    if (node >= n_out) return;
    const int beg = rowptr[node], end = rowptr[node + 1];
    if (end == beg) return;
    const float inv = 1.f / (float)(end - beg);
    for (int e = beg; e < end; ++e) {
        const int s = __ldg(idxn + e);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < n_iter; ++r) {
            const float4 gv = __ldg(gs + r * g_stride4 + node * kG + sub);
            const float4 xv = __ldg(xs + r * x_stride4 + (int64_t)s * kG + sub);
            acc = fma4(xv, gv, acc);
        }
        acc.x *= inv;
        acc.y *= inv;
        acc.z *= inv;
        acc.w *= inv;
        float4* dst = grad_w + (int64_t)e * kG + sub;
        if (accumulate) {
            const float4 old = *dst;
            acc.x += old.x;
            acc.y += old.y;
            acc.z += old.z;
            acc.w += old.w;
        }
        st_stream4(dst, acc);
    }
}

// grad_W[e,k,o] (+)= (1/deg_t) * sum_r x_r[src_e,k] * g_r[t,o]   (matrix filters)
__global__ void __launch_bounds__(256)
ecc_mat_bwd_w_kernel(const float* __restrict__ xs, const float4* __restrict__ gs,
                     int64_t x_stride, int64_t g_stride4, int n_iter,
                     const int* __restrict__ rowptr, const int* __restrict__ idxn,
                     float4* __restrict__ grad_w, int n_out, int accumulate) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n_out) return;
    const int r4 = lane >> 3, q = lane & 7;
    const int beg = rowptr[node], end = rowptr[node + 1];
    if (end == beg) return;
    const float inv = 1.f / (float)(end - beg);
    for (int e = beg; e < end; ++e) {
        const int s = __ldg(idxn + e);
        float4 acc[8];
#pragma unroll
        for (int it = 0; it < 8; ++it) acc[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < n_iter; ++r) {
            float4 gv = __ldg(gs + r * g_stride4 + node * kG + q);
            gv.x *= inv;
            gv.y *= inv;
            gv.z *= inv;
            gv.w *= inv;
            const float xv = __ldg(xs + r * x_stride + (int64_t)s * kC + lane);
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                const float xk = __shfl_sync(0xffffffffu, xv, it * 4 + r4);
                acc[it].x = fmaf(xk, gv.x, acc[it].x);
                acc[it].y = fmaf(xk, gv.y, acc[it].y);
                acc[it].z = fmaf(xk, gv.z, acc[it].z);
                acc[it].w = fmaf(xk, gv.w, acc[it].w);
            }
        }
        float4* dst = grad_w + (int64_t)e * 256;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            float4 v = acc[it];
            if (accumulate) {
                const float4 old = dst[it * 32 + lane];
                v.x += old.x;
                v.y += old.y;
                v.z += old.z;
                v.w += old.w;
            }
            st_stream4(dst + it * 32 + lane, v);
        }
    }
}

// grad_x[j,:] = add0 + add1 + sum_{e out of j} w[e,:] * g[t_e,:]/deg_t  (vector filters)
// warp per source node (ecc_rows.cuh); w and g through the non-coherent path.
__global__ void __launch_bounds__(256)
ecc_vv_bwd_x_kernel(const float4* __restrict__ w, const float4* __restrict__ g,
                    const int* __restrict__ tgt_rowptr, const int* __restrict__ src_rowptr,
                    const int* __restrict__ src_perm, const int* __restrict__ edge_tgt,
                    const float4* __restrict__ add0, const float4* __restrict__ add1,
                    float4* __restrict__ grad_x, int n_in) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n_in) return;
    float4 acc = ecc_vv_row_bwd_x<LdNc, LdNc>(w, (const float*)g, tgt_rowptr, src_perm, edge_tgt,
                                              src_rowptr[node], src_rowptr[node + 1], lane);
    if (lane < kG) {  // slot 0: sub = lane
        const int64_t o = node * kG + lane;
        if (add0) acc = add4(acc, add0[o]);
        if (add1) acc = add4(acc, add1[o]);
        grad_x[o] = acc;
    }
}

// grad_x[j,k] = add0 + add1 + sum_{e out of j} sum_o W_e[k,o] * g[t_e,o]/deg_t
__global__ void __launch_bounds__(256)
ecc_mat_bwd_x_kernel(const float4* __restrict__ w, const float4* __restrict__ g,
                     const int* __restrict__ tgt_rowptr, const int* __restrict__ src_rowptr,
                     const int* __restrict__ src_perm, const int* __restrict__ edge_tgt,
                     const float* __restrict__ add0, const float* __restrict__ add1,
                     float* __restrict__ grad_x, int n_in) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t node = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (node >= n_in) return;
    const int q = lane & 7;
    const int beg = src_rowptr[node], end = src_rowptr[node + 1];
    float acc[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) acc[it] = 0.f;
    for (int p = beg; p < end; ++p) {
        const int e = __ldg(src_perm + p);
        const int tg = __ldg(edge_tgt + e);
        const float inv = 1.f / (float)(__ldg(tgt_rowptr + tg + 1) - __ldg(tgt_rowptr + tg));
        const float4* W = w + (int64_t)e * 256;
        float4 wv[8];
#pragma unroll
        for (int it = 0; it < 8; ++it) wv[it] = ld_stream4(W + it * 32 + lane);
        float4 gv = __ldg(g + (int64_t)tg * kG + q);
        gv.x *= inv;
        gv.y *= inv;
        gv.z *= inv;
        gv.w *= inv;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            acc[it] = fmaf(wv[it].x, gv.x, acc[it]);
            acc[it] = fmaf(wv[it].y, gv.y, acc[it]);
            acc[it] = fmaf(wv[it].z, gv.z, acc[it]);
            acc[it] = fmaf(wv[it].w, gv.w, acc[it]);
        }
    }
    // reduce over the 8 column groups q (lanes differing in bits 0..2)
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        acc[it] += __shfl_xor_sync(0xffffffffu, acc[it], 1);
        acc[it] += __shfl_xor_sync(0xffffffffu, acc[it], 2);
        acc[it] += __shfl_xor_sync(0xffffffffu, acc[it], 4);
    }
    // row k = 4*it + r lives in lanes with (lane>>3)==r; lane l wants row l.
    float mine = 0.f;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const float v = __shfl_sync(0xffffffffu, acc[it], (lane & 3) * 8);
        if ((lane >> 2) == it) mine = v;
    }
    const int64_t o = node * kC + lane;
    if (add0) mine += add0[o];
    if (add1) mine += add1[o];
    grad_x[o] = mine;
}

// ------------------------------------------------------------ generic kernels
// Any widths, float32/float64, optional idxe.  One thread per output element.

template <typename T>
__global__ void ecc_generic_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                       const int* __restrict__ rowptr,
                                       const int* __restrict__ idxn,
                                       const int* __restrict__ idxe, T* __restrict__ out,
                                       int64_t n_out, int c_in, int c_out, int is_mat) {
    SPG_PDL_ENTRY();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_out * c_out) return;
    const int64_t node = t / c_out;
    const int o = (int)(t % c_out);
    const int beg = rowptr[node], end = rowptr[node + 1];
    T acc = 0;
    for (int e = beg; e < end; ++e) {
        const int64_t s = idxn[e];
        const int64_t we = idxe ? idxe[e] : e;
        if (is_mat) {
            const T* W = w + we * c_in * c_out;
            T a = 0;
            for (int k = 0; k < c_in; ++k) a += x[s * c_in + k] * W[(int64_t)k * c_out + o];
            acc += a;
        } else {
            acc += x[s * c_in + o] * w[we * c_in + o];
        }
    }
    const int deg = end - beg;
    out[t] = deg > 0 ? acc / (T)deg : (T)0;
}

__device__ __forceinline__ void atomic_add_t(float* p, float v) { atomicAdd(p, v); }
__device__ __forceinline__ void atomic_add_t(double* p, double v) { atomicAdd(p, v); }

template <typename T>
__global__ void ecc_generic_bwd_w_kernel(const T* __restrict__ xs, const T* __restrict__ gs,
                                         int64_t x_stride, int64_t g_stride, int n_iter,
                                         const int* __restrict__ rowptr,
                                         const int* __restrict__ idxn,
                                         const int* __restrict__ idxe,
                                         const int* __restrict__ edge_tgt,
                                         T* __restrict__ grad_w, int64_t n_edges, int c_in,
                                         int c_out, int is_mat, int accumulate) {
    SPG_PDL_ENTRY();
    const int64_t per_edge = is_mat ? (int64_t)c_in * c_out : c_in;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_edges * per_edge) return;
    const int64_t e = t / per_edge;
    const int64_t rem = t % per_edge;
    const int k = is_mat ? (int)(rem / c_out) : (int)rem;
    const int o = is_mat ? (int)(rem % c_out) : (int)rem;
    const int64_t s = idxn[e];
    const int64_t tg = edge_tgt[e];
    const T deg = (T)(rowptr[tg + 1] - rowptr[tg]);
    T acc = 0;
    for (int r = 0; r < n_iter; ++r)
        acc += xs[r * x_stride + s * c_in + k] * (gs[r * g_stride + tg * c_out + o] / deg);
    if (idxe) {
        atomic_add_t(grad_w + (int64_t)idxe[e] * per_edge + rem, acc);
    } else if (accumulate) {
        grad_w[t] += acc;
    } else {
        grad_w[t] = acc;
    }
}

template <typename T>
__global__ void ecc_generic_bwd_x_kernel(const T* __restrict__ w, const T* __restrict__ g,
                                         const int* __restrict__ tgt_rowptr,
                                         const int* __restrict__ src_rowptr,
                                         const int* __restrict__ src_perm,
                                         const int* __restrict__ edge_tgt,
                                         const int* __restrict__ idxe, const T* __restrict__ add0,
                                         const T* __restrict__ add1, T* __restrict__ grad_x,
                                         int64_t n_in, int c_in, int c_out, int is_mat) {
    SPG_PDL_ENTRY();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_in * c_in) return;
    const int64_t node = t / c_in;
    const int k = (int)(t % c_in);
    const int beg = src_rowptr[node], end = src_rowptr[node + 1];
    T acc = 0;
    for (int p = beg; p < end; ++p) {
        const int64_t e = src_perm[p];
        const int64_t tg = edge_tgt[e];
        const int64_t we = idxe ? idxe[e] : e;
        const T deg = (T)(tgt_rowptr[tg + 1] - tgt_rowptr[tg]);
        if (is_mat) {
            const T* W = w + we * c_in * c_out + (int64_t)k * c_out;
            T a = 0;
            for (int o = 0; o < c_out; ++o) a += W[o] * (g[tg * c_out + o] / deg);
            acc += a;
        } else {
            acc += w[we * c_in + k] * (g[tg * c_out + k] / deg);
        }
    }
    if (add0) acc += add0[t];
    if (add1) acc += add1[t];
    grad_x[t] = acc;
}

static inline bool fast_ok(int c_in, int c_out, int dtype, const void* idxe) {
    return dtype == SPG_F32 && c_in == kC && c_out == kC && idxe == nullptr;
}

static inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace spg

using namespace spg;

extern "C" {

int spg_ecc_fwd(const void* x, const void* w, const int32_t* tgt_rowptr, const int32_t* idxn,
                const int32_t* idxe, void* out, int64_t n_out, int64_t n_edges, int c_in,
                int c_out, int w_is_matrix, int dtype, spg_stream_t stream) {
    if (n_out < 0 || n_edges < 0 || c_in <= 0 || c_out <= 0) return SPG_E_BADARG;
    if (n_out == 0) return SPG_OK;
    if (!x || !tgt_rowptr || !out || (n_edges > 0 && (!w || !idxn))) return SPG_E_BADARG;
    if (!w_is_matrix && c_in != c_out) return SPG_E_BADARG;
    if (dtype != SPG_F32 && dtype != SPG_F64) return SPG_E_UNSUPPORTED;
    if (n_out >= (1ll << 31) || n_edges >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    if (fast_ok(c_in, c_out, dtype, idxe) && aligned16(x) && aligned16(w) && aligned16(out)) {
        if (w_is_matrix) {
            const int64_t blocks = ceil_div64(n_out * 32, 256);
            SPG_LAUNCH(K_ECC_MAT_FWD, s, ecc_mat_fwd_kernel, (unsigned)blocks, 256, 0,
                       (const float*)x, (const float4*)w, tgt_rowptr, idxn, (float4*)out,
                       (int)n_out);
        } else {
            const int64_t blocks = ceil_div64(n_out * 32, 256);
            SPG_LAUNCH(K_ECC_VV_FWD, s, ecc_vv_fwd_kernel, (unsigned)blocks, 256, 0,
                       (const float4*)x, (const float4*)w, tgt_rowptr, idxn, (float4*)out,
                       (int)n_out);
        }
        return launch_status();
    }
    const int64_t blocks = ceil_div64(n_out * c_out, 256);
    if (dtype == SPG_F32) {
        SPG_LAUNCH(K_ECC_GEN_FWD, s, ecc_generic_fwd_kernel<float>, (unsigned)blocks, 256, 0,
                   (const float*)x, (const float*)w, tgt_rowptr, idxn, idxe, (float*)out, n_out,
                   c_in, c_out, w_is_matrix);
    } else {
        SPG_LAUNCH(K_ECC_GEN_FWD, s, ecc_generic_fwd_kernel<double>, (unsigned)blocks, 256, 0,
                   (const double*)x, (const double*)w, tgt_rowptr, idxn, idxe, (double*)out,
                   n_out, c_in, c_out, w_is_matrix);
    }
    return launch_status();
}

int spg_ecc_bwd_w(const void* xs, const void* gs, int64_t x_iter_stride, int64_t g_iter_stride,
                  int n_iter, const int32_t* tgt_rowptr, const int32_t* idxn,
                  const int32_t* idxe, const int32_t* edge_tgt, void* grad_w, int64_t n_out,
                  int64_t n_edges, int c_in, int c_out, int w_is_matrix, int accumulate,
                  int dtype, spg_stream_t stream) {
    if (n_out < 0 || n_edges < 0 || c_in <= 0 || c_out <= 0 || n_iter <= 0) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!xs || !gs || !tgt_rowptr || !idxn || !edge_tgt || !grad_w) return SPG_E_BADARG;
    if (!w_is_matrix && c_in != c_out) return SPG_E_BADARG;
    if (dtype != SPG_F32 && dtype != SPG_F64) return SPG_E_UNSUPPORTED;
    if (n_out >= (1ll << 31) || n_edges >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    if (fast_ok(c_in, c_out, dtype, idxe) && aligned16(xs) && aligned16(gs) &&
        aligned16(grad_w) && (x_iter_stride % 4 == 0) && (g_iter_stride % 4 == 0)) {
        if (w_is_matrix) {
            const int64_t blocks = ceil_div64(n_out * 32, 256);
            SPG_LAUNCH(K_ECC_MAT_BWD_W, s, ecc_mat_bwd_w_kernel, (unsigned)blocks, 256, 0,
                       (const float*)xs, (const float4*)gs, x_iter_stride, g_iter_stride / 4,
                       n_iter, tgt_rowptr, idxn, (float4*)grad_w, (int)n_out, accumulate);
        } else {
            const int64_t blocks = ceil_div64(n_out * kG, 256);
            SPG_LAUNCH(K_ECC_VV_BWD_W, s, ecc_vv_bwd_w_kernel, (unsigned)blocks, 256, 0,
                       (const float4*)xs, (const float4*)gs, x_iter_stride / 4, g_iter_stride / 4,
                       n_iter, tgt_rowptr, idxn, (float4*)grad_w, (int)n_out, accumulate);
        }
        return launch_status();
    }
    const int64_t per_edge = w_is_matrix ? (int64_t)c_in * c_out : c_in;
    const int64_t blocks = ceil_div64(n_edges * per_edge, 256);
    if (blocks >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    if (dtype == SPG_F32) {
        SPG_LAUNCH(K_ECC_GEN_BWD_W, s, ecc_generic_bwd_w_kernel<float>, (unsigned)blocks, 256, 0,
                   (const float*)xs, (const float*)gs, x_iter_stride, g_iter_stride, n_iter,
                   tgt_rowptr, idxn, idxe, edge_tgt, (float*)grad_w, n_edges, c_in, c_out,
                   w_is_matrix, accumulate);
    } else {
        SPG_LAUNCH(K_ECC_GEN_BWD_W, s, ecc_generic_bwd_w_kernel<double>, (unsigned)blocks, 256, 0,
                   (const double*)xs, (const double*)gs, x_iter_stride, g_iter_stride, n_iter,
                   tgt_rowptr, idxn, idxe, edge_tgt, (double*)grad_w, n_edges, c_in, c_out,
                   w_is_matrix, accumulate);
    }
    return launch_status();
}

int spg_ecc_bwd_x(const void* w, const void* g, const int32_t* tgt_rowptr,
                  const int32_t* src_rowptr, const int32_t* src_perm, const int32_t* edge_tgt,
                  const int32_t* idxe, const void* add0, const void* add1, void* grad_x,
                  int64_t n_in, int64_t n_edges, int c_in, int c_out, int w_is_matrix,
                  int dtype, spg_stream_t stream) {
    if (n_in < 0 || n_edges < 0 || c_in <= 0 || c_out <= 0) return SPG_E_BADARG;
    if (n_in == 0) return SPG_OK;
    if (!tgt_rowptr || !src_rowptr || !grad_x) return SPG_E_BADARG;
    if (n_edges > 0 && (!w || !g || !src_perm || !edge_tgt)) return SPG_E_BADARG;
    if (!w_is_matrix && c_in != c_out) return SPG_E_BADARG;
    if (dtype != SPG_F32 && dtype != SPG_F64) return SPG_E_UNSUPPORTED;
    if (n_in >= (1ll << 31) || n_edges >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    if (fast_ok(c_in, c_out, dtype, idxe) && aligned16(w) && aligned16(g) && aligned16(grad_x) &&
        aligned16(add0) && aligned16(add1)) {
        if (w_is_matrix) {
            const int64_t blocks = ceil_div64(n_in * 32, 256);
            SPG_LAUNCH(K_ECC_MAT_BWD_X, s, ecc_mat_bwd_x_kernel, (unsigned)blocks, 256, 0,
                       (const float4*)w, (const float4*)g, tgt_rowptr, src_rowptr, src_perm,
                       edge_tgt, (const float*)add0, (const float*)add1, (float*)grad_x,
                       (int)n_in);
        } else {
            const int64_t blocks = ceil_div64(n_in * 32, 256);
            SPG_LAUNCH(K_ECC_VV_BWD_X, s, ecc_vv_bwd_x_kernel, (unsigned)blocks, 256, 0,
                       (const float4*)w, (const float4*)g, tgt_rowptr, src_rowptr, src_perm,
                       edge_tgt, (const float4*)add0, (const float4*)add1, (float4*)grad_x,
                       (int)n_in);
        }
        return launch_status();
    }
    const int64_t blocks = ceil_div64(n_in * c_in, 256);
    if (dtype == SPG_F32) {
        SPG_LAUNCH(K_ECC_GEN_BWD_X, s, ecc_generic_bwd_x_kernel<float>, (unsigned)blocks, 256, 0,
                   (const float*)w, (const float*)g, tgt_rowptr, src_rowptr, src_perm, edge_tgt,
                   idxe, (const float*)add0, (const float*)add1, (float*)grad_x, n_in, c_in,
                   c_out, w_is_matrix);
    } else {
        SPG_LAUNCH(K_ECC_GEN_BWD_X, s, ecc_generic_bwd_x_kernel<double>, (unsigned)blocks, 256, 0,
                   (const double*)w, (const double*)g, tgt_rowptr, src_rowptr, src_perm,
                   edge_tgt, idxe, (const double*)add0, (const double*)add1, (double*)grad_x,
                   n_in, c_in, c_out, w_is_matrix);
    }
    return launch_status();
}

}  // extern "C"
