// PointNet-specific data movement: NCL clouds -> point-major rows (with the spatial
// transformer applied), segmented max-pool over the points of a superpoint with its
// argmax, the matching backward scatters, and the descriptor row scatter/gather of
// CloudEmbedder.
//
// Reference semantics: learning/pointnet.py:120-133 (transform + max_pool1d + cat),
// :147-158 (index_copy_ into zero descriptors).
#include <float.h>

#include "common.cuh"
#include "segs.cuh"

namespace spg {

constexpr int kPtChunk = 128;

// grid (B, ceil(L/128)); block 128.  smem tile [F][129].
__global__ void __launch_bounds__(kPtChunk)
cloud_rows_kernel(const float* __restrict__ clouds, const float* __restrict__ T, int add_eye,
                  float* __restrict__ rows, int64_t ld, int F, int L) {
    SPG_PDL_ENTRY();
    extern __shared__ float tile[];
    const int64_t b = blockIdx.x;
    const int l0 = blockIdx.y * kPtChunk;
    const int nl = min(kPtChunk, L - l0);
    const float* src = clouds + b * (int64_t)F * L;
    for (int f = 0; f < F; ++f)
        for (int l = threadIdx.x; l < nl; l += kPtChunk)
            tile[f * (kPtChunk + 1) + l] = src[(int64_t)f * L + l0 + l];
    __syncthreads();
    if (T && F >= 2) {
        const float eye = add_eye ? 1.f : 0.f;
        const float t00 = T[b * 4 + 0] + eye, t01 = T[b * 4 + 1], t10 = T[b * 4 + 2],
                    t11 = T[b * 4 + 3] + eye;
        for (int l = threadIdx.x; l < nl; l += kPtChunk) {
            const float x0 = tile[l], x1 = tile[(kPtChunk + 1) + l];
            // xy' = xy^T * T  (row vector times T), ref: learning/pointnet.py:123
            tile[l] = fmaf(x0, t00, x1 * t10);
            tile[(kPtChunk + 1) + l] = fmaf(x0, t01, x1 * t11);
        }
        __syncthreads();
    }
    float* dst = rows + (b * L + l0) * ld;
    const int64_t total = (int64_t)nl * ld;
    for (int64_t i = threadIdx.x; i < total; i += kPtChunk) {
        const int l = (int)(i / ld), f = (int)(i % ld);
        dst[i] = f < F ? tile[f * (kPtChunk + 1) + l] : 0.f;
    }
}

// pooled[b, c] = max over the rows of segment b, argmax[b, c] = index of the first maximum within the
// segment.  A warp owns (segment, 32 channels): lane = channel for coalesced 128-byte row reads, the
// segment's rows are strided over the 8 warps of the block and folded through shared memory.
// grid (ceil(C/32), B); block (32 x 8).
template <class Segs>
__global__ void __launch_bounds__(256)
segmax_fwd_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                  const float* __restrict__ shift, int relu, float* __restrict__ pooled,
                  int64_t ldp, int* __restrict__ argmax, Segs segs, int C) {
    SPG_PDL_ENTRY();
    __shared__ float s_v[8][32];
    __shared__ int s_i[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t b = blockIdx.y;
    const int64_t r0 = segs.begin(b);
    const int L = (int)(segs.end(b) - r0);
    float best = -FLT_MAX;
    int bi = 0;
    if (c < C) {
        const float sc = scale ? scale[c] : 1.f, sh = shift ? shift[c] : 0.f;
        const float* src = Y + r0 * ldy + c;
        for (int l = y; l < L; l += 8) {
            float v = fmaf(__ldg(src + (int64_t)l * ldy), sc, sh);
            if (relu) v = fmaxf(v, 0.f);
            if (v > best || l == y) {  // first element initialises; strict > keeps first max
                best = v;
                bi = l;
            }
        }
    }
    s_v[y][x] = best;
    s_i[y][x] = (y < L) ? bi : -1;
    __syncthreads();
    if (y == 0 && c < C) {
        float bv = s_v[0][x];
        int bidx = s_i[0][x];
        for (int j = 1; j < 8; ++j) {
            const float v = s_v[j][x];
            const int i = s_i[j][x];
            if (i >= 0 && (v > bv || (v == bv && i < bidx))) {
                bv = v;
                bidx = i;
            }
        }
        pooled[b * ldp + c] = (Segs::kMayBeEmpty && bidx < 0) ? 0.f : bv;
        argmax[b * C + c] = bidx;
    }
}

// 128-bit variant: a warp spans 128 columns (float4 per lane), 8 row lanes, 4 rows in flight per
// thread.  grid (ceil(C/128), B); block 256.  Same tie rule as the scalar kernel (first maximum).
template <class Segs>
__global__ void __launch_bounds__(256)
segmax_fwd_v4_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                     const float* __restrict__ shift, int relu, float* __restrict__ pooled,
                     int64_t ldp, int* __restrict__ argmax, Segs segs, int C) {
    SPG_PDL_ENTRY();
    __shared__ float4 s_v[8][32];
    __shared__ int4 s_i[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * 4;
    const int64_t b = blockIdx.y;
    const int64_t r0 = segs.begin(b);
    const int L = (int)(segs.end(b) - r0);
    float best[4] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    int bi[4] = {-1, -1, -1, -1};
    if (c < C) {
        float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (scale) sc[j] = scale[c + j];
            if (shift) sh[j] = shift[c + j];
        }
        const float* src = Y + r0 * ldy + c;
#pragma unroll 4
        for (int l = y; l < L; l += 8) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src + (int64_t)l * ldy));
            const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float t = fmaf(v[j], sc[j], sh[j]);
                if (relu) t = fmaxf(t, 0.f);
                if (bi[j] < 0 || t > best[j]) {  // first element initialises; strict > keeps first max
                    best[j] = t;
                    bi[j] = l;
                }
            }
        }
    }
    s_v[y][x] = make_float4(best[0], best[1], best[2], best[3]);
    s_i[y][x] = make_int4(bi[0], bi[1], bi[2], bi[3]);
    __syncthreads();
    if (y == 0 && c < C) {
        for (int j = 1; j < 8; ++j) {
            const float4 vq = s_v[j][x];
            const int4 iq = s_i[j][x];
            const float v[4] = {vq.x, vq.y, vq.z, vq.w};
            const int i[4] = {iq.x, iq.y, iq.z, iq.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (i[k] >= 0 && (bi[k] < 0 || v[k] > best[k] || (v[k] == best[k] && i[k] < bi[k]))) {
                    best[k] = v[k];
                    bi[k] = i[k];
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) pooled[b * ldp + c + k] = (Segs::kMayBeEmpty && bi[k] < 0) ? 0.f : best[k];
        *reinterpret_cast<int4*>(argmax + b * C + c) = make_int4(bi[0], bi[1], bi[2], bi[3]);
    }
}

// G[r, c] = g_pooled[b, c] if row r is the argmax of its segment b, else 0 (every row written).
template <class Segs>
__global__ void __launch_bounds__(256)
segmax_bwd_kernel(const float* __restrict__ gp, int64_t ldg, const int* __restrict__ argmax,
                  float* __restrict__ G, int64_t ldG, int64_t rows, Segs segs, int C) {
    SPG_PDL_ENTRY();
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    if (c >= C) return;
    for (int64_t r = (int64_t)blockIdx.y * 8 + y; r < rows; r += (int64_t)gridDim.y * 8) {
        const int64_t b = segs.seg_of(r);
        const int l = (int)(r - segs.begin(b));
        G[r * ldG + c] = (argmax[b * C + c] == l) ? gp[b * ldg + c] : 0.f;
    }
}

// grid B; block 128.
__global__ void __launch_bounds__(128)
stn_apply_bwd_kernel(const float* __restrict__ clouds, const float* __restrict__ dX, int64_t ld,
                     float* __restrict__ dT, int F, int L) {
    SPG_PDL_ENTRY();
    __shared__ float red[4][4];
    const int64_t b = blockIdx.x;
    const float* xy = clouds + b * (int64_t)F * L;
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
    for (int l = threadIdx.x; l < L; l += 128) {
        const float x0 = xy[l], x1 = xy[L + l];
        const float d0 = dX[(b * L + l) * ld], d1 = dX[(b * L + l) * ld + 1];
        a00 = fmaf(x0, d0, a00);
        a01 = fmaf(x0, d1, a01);
        a10 = fmaf(x1, d0, a10);
        a11 = fmaf(x1, d1, a11);
    }
    a00 = warp_sum(a00);
    a01 = warp_sum(a01);
    a10 = warp_sum(a10);
    a11 = warp_sum(a11);
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        red[w][0] = a00;
        red[w][1] = a01;
        red[w][2] = a10;
        red[w][3] = a11;
    }
    __syncthreads();
    if (threadIdx.x < 4)
        dT[b * 4 + threadIdx.x] = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] +
                                  red[3][threadIdx.x];
}

// ---- max-pool backward fused with the BatchNorm+ReLU backward of the layer that fed the pool.
// The gradient w.r.t. the pooled activation is non-zero at one point per (cloud, channel) only, so
// the batch reductions s1 = sum G*mask, s2 = sum G*mask*xhat need just the argmax rows ...
// grid (ceil(C/32), ceil(B/256)); block 32 x 8; partial layout [chunk][2][C] (as act_bwd_reduce).
template <class Segs>
__global__ void __launch_bounds__(256)
segmax_bn_bwd_reduce_kernel(const float* __restrict__ gp, int64_t ldg, const int* __restrict__ argmax,
                            const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                            const float* __restrict__ shift, const float* __restrict__ mean,
                            const float* __restrict__ var, float eps, int relu,
                            float* __restrict__ ws, int64_t B, Segs segs, int C) {
    SPG_PDL_ENTRY();
    __shared__ float s1[8][32], s2[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t b0 = (int64_t)blockIdx.y * 256, b1 = min(B, b0 + 256);
    float a1 = 0.f, a2 = 0.f;
    if (c < C) {
        const float sc = scale[c], sh = shift[c], mu = mean[c];
        const float rstd = 1.f / sqrtf(var[c] + eps);
        for (int64_t b = b0 + y; b < b1; b += 8) {
            const int l = argmax[b * C + c];
            if (Segs::kMayBeEmpty && l < 0) continue;  // empty segment: no row, no gradient
            const float yv = __ldg(Y + (segs.begin(b) + l) * ldy + c);
            float g = __ldg(gp + b * ldg + c);
            if (relu) g = relu_bwd(g, yv, sc, sh);
            a1 += g;
            a2 = fmaf(g, (yv - mu) * rstd, a2);
        }
    }
    s1[y][x] = a1;
    s2[y][x] = a2;
    __syncthreads();
    if (y == 0 && c < C) {
        float t1 = 0.f, t2 = 0.f;
        for (int j = 0; j < 8; ++j) {
            t1 += s1[j][x];
            t2 += s2[j][x];
        }
        ws[((int64_t)blockIdx.y * 2) * C + c] = t1;
        ws[((int64_t)blockIdx.y * 2 + 1) * C + c] = t2;
    }
}

// ... and dY = scale*(G*mask - s1/M - xhat*s2/M) is written directly from (g_pooled, argmax, Y):
// the dense G is never materialised.  One 128-bit lane per 4 channels; M rows in all segments.
template <class Segs>
__global__ void __launch_bounds__(256)
segmax_bn_bwd_apply_kernel(const float* __restrict__ gp, int64_t ldg, const int* __restrict__ argmax,
                           const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                           const float* __restrict__ shift, const float* __restrict__ mean,
                           const float* __restrict__ var, float eps, int relu,
                           const float* __restrict__ s1, const float* __restrict__ s2,
                           float* __restrict__ dY, int64_t lddy, int64_t M, Segs segs, int C) {
    SPG_PDL_ENTRY();
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * 4;
    if (c >= C) return;
    float sc[4], sh[4], mu[4], rs[4], m1[4], m2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sc[j] = scale[c + j];
        sh[j] = shift[c + j];
        mu[j] = mean[c + j];
        rs[j] = 1.f / sqrtf(var[c + j] + eps);
        m1[j] = s1[c + j] / (float)M;
        m2[j] = s2[c + j] / (float)M;
    }
#pragma unroll 2
    for (int64_t r = (int64_t)blockIdx.y * 8 + y; r < M; r += (int64_t)gridDim.y * 8) {
        const int64_t b = segs.seg_of(r);
        const int l = (int)(r - segs.begin(b));
        const float4 yq = __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c));
        const int4 am = __ldg(reinterpret_cast<const int4*>(argmax + b * C + c));
        // the pooled gradient row may be unaligned (ld = 256 + #global features): scalar loads, L1 hits
        const float* gr = gp + b * ldg + c;
        const float gv[4] = {__ldg(gr), __ldg(gr + 1), __ldg(gr + 2), __ldg(gr + 3)};
        const float yv[4] = {yq.x, yq.y, yq.z, yq.w};
        const int aq[4] = {am.x, am.y, am.z, am.w};
        float d[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float g = (aq[j] == l) ? gv[j] : 0.f;
            if (relu) g = relu_bwd(g, yv[j], sc[j], sh[j]);
            d[j] = bn_bwd(g, yv[j], sc[j], mu[j], rs[j], m1[j], m2[j]);
        }
        *reinterpret_cast<float4*>(dY + r * lddy + c) = make_float4(d[0], d[1], d[2], d[3]);
    }
}

__global__ void rows_scatter_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx,
                                    float* __restrict__ dst, int64_t n, int C) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * C) return;
    const int64_t r = i / C;
    dst[idx[r] * C + (i % C)] = src[i];
}

__global__ void rows_gather_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx,
                                   float* __restrict__ dst, int64_t n, int C) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * C) return;
    const int64_t r = i / C;
    dst[i] = src[idx[r] * C + (i % C)];
}

// gradient w.r.t. the point-major rows back into the reference's [B, F, L] layout (inverse of cloud_rows
// without a transformer): clouds_grad[b, f, l] = rows_grad[b*L + l, f].  grid (B, ceil(L/128)); block 128.
__global__ void __launch_bounds__(kPtChunk)
rows_to_clouds_kernel(const float* __restrict__ rows, int64_t ld, float* __restrict__ clouds, int F, int L) {
    SPG_PDL_ENTRY();
    extern __shared__ float tile[];  // [F][129]
    const int64_t b = blockIdx.x;
    const int l0 = blockIdx.y * kPtChunk;
    const int nl = min(kPtChunk, L - l0);
    const float* src = rows + (b * L + l0) * ld;
    for (int64_t i = threadIdx.x; i < (int64_t)nl * F; i += kPtChunk) {
        const int l = (int)(i / F), f = (int)(i % F);
        tile[f * (kPtChunk + 1) + l] = src[(int64_t)l * ld + f];
    }
    __syncthreads();
    float* dst = clouds + b * (int64_t)F * L;
    for (int f = 0; f < F; ++f)
        for (int l = threadIdx.x; l < nl; l += kPtChunk) dst[(int64_t)f * L + l0 + l] = tile[f * (kPtChunk + 1) + l];
}

// ------------------------------------------------------------------ ragged (CSR) segments: the xy transform
// rows_out = rows_in with columns 0,1 replaced by (x0,x1) * (T[seg] (+ I))   (pointnet.py:123)
__global__ void __launch_bounds__(256)
rows_xy_transform_kernel(const float* __restrict__ in, const float* __restrict__ T, int add_eye,
                         const int32_t* __restrict__ row_seg, float* __restrict__ out, int64_t P,
                         int64_t ld) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P * ld) return;
    const int64_t r = i / ld;
    const int f = (int)(i % ld);
    float v = in[i];
    if (f < 2) {
        const int64_t b = row_seg[r];
        const float eye = add_eye ? 1.f : 0.f;
        const float x0 = in[r * ld], x1 = in[r * ld + 1];
        v = f == 0 ? fmaf(x0, T[b * 4 + 0] + eye, x1 * T[b * 4 + 2])
                   : fmaf(x0, T[b * 4 + 1], x1 * (T[b * 4 + 3] + eye));
    }
    out[i] = v;
}

// dT[b] = sum over the rows of segment b of (x0, x1)^T (d0, d1); one warp per segment.
__global__ void __launch_bounds__(256)
rows_xy_transform_bwd_kernel(const float* __restrict__ in, int64_t ld, const float* __restrict__ dOut,
                             int64_t ldd, const int64_t* __restrict__ offsets, float* __restrict__ dT,
                             int64_t B) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B) return;
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
    for (int64_t r = offsets[b] + lane; r < offsets[b + 1]; r += 32) {
        const float x0 = in[r * ld], x1 = in[r * ld + 1], d0 = dOut[r * ldd], d1 = dOut[r * ldd + 1];
        a00 = fmaf(x0, d0, a00);
        a01 = fmaf(x0, d1, a01);
        a10 = fmaf(x1, d0, a10);
        a11 = fmaf(x1, d1, a11);
    }
    a00 = warp_sum(a00);
    a01 = warp_sum(a01);
    a10 = warp_sum(a10);
    a11 = warp_sum(a11);
    if (lane == 0) {
        dT[b * 4 + 0] = a00;
        dT[b * 4 + 1] = a01;
        dT[b * 4 + 2] = a10;
        dT[b * 4 + 3] = a11;
    }
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_cloud_rows(const float* clouds, const float* T, int add_eye, float* rows, int64_t ld,
                   int64_t B, int F, int L, spg_stream_t stream) {
    if (B < 0 || F <= 0 || L <= 0 || ld < F) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!clouds || !rows) return SPG_E_BADARG;
    if (F > 256 || B > 2147483647ll) return SPG_E_UNSUPPORTED;
    const size_t smem = sizeof(float) * (size_t)F * (kPtChunk + 1);
    if (smem > 200 * 1024) return SPG_E_UNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(cloud_rows_kernel,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    dim3 grid((unsigned)B, (unsigned)ceil_div64(L, kPtChunk));
    SPG_LAUNCH(K_CLOUD_ROWS, (cudaStream_t)stream, cloud_rows_kernel, grid, kPtChunk, smem, clouds,
               T, add_eye, rows, ld, F, L);
    return launch_status();
}

int spg_segmax_fwd(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* pooled, int64_t ldp, int32_t* argmax, int64_t B, int L, const int64_t* offsets,
                   int C, spg_stream_t stream) {
    if (B < 0 || (!offsets && L <= 0) || C <= 0 || ldy < C || ldp < C) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!Y || !pooled || !argmax) return SPG_E_BADARG;
    if (B > 65535ll * 32768) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t max_by = 65535;
    const bool vec = (C & 3) == 0 && (ldy & 3) == 0 && ((uintptr_t)Y & 15) == 0 &&
                     ((uintptr_t)argmax & 15) == 0;
    for (int64_t b0 = 0; b0 < B; b0 += max_by) {
        const int64_t nb = min(max_by, B - b0);
        // segments [b0, b0 + nb): the fixed layout moves Y, the CSR layout moves offsets
        const float* Yb = offsets ? Y : Y + b0 * L * ldy;
        const int rc = with_segs(L, offsets ? offsets + b0 : nullptr, nullptr, [&](auto segs) {
            if (vec) {
                dim3 grid((unsigned)ceil_div64(C, 128), (unsigned)nb);
                SPG_LAUNCH(K_SEGMAX_FWD, s, segmax_fwd_v4_kernel<decltype(segs)>, grid, 256, 0, Yb, ldy,
                           scale, shift, relu, pooled + b0 * ldp, ldp, argmax + b0 * C, segs, C);
            } else {
                dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)nb);
                SPG_LAUNCH(K_SEGMAX_FWD, s, segmax_fwd_kernel<decltype(segs)>, grid, 256, 0, Yb, ldy,
                           scale, shift, relu, pooled + b0 * ldp, ldp, argmax + b0 * C, segs, C);
            }
            return launch_status();
        });
        if (rc) return rc;
    }
    return SPG_OK;
}

int spg_segmax_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, float* G,
                   int64_t ldG, int64_t B, int L, const int64_t* offsets, const int32_t* row_seg,
                   int64_t rows, int C, spg_stream_t stream) {
    if (B < 0 || rows < 0 || C <= 0 || ldg < C || ldG < C) return SPG_E_BADARG;
    if (offsets ? !row_seg : (L <= 0 || rows != B * L)) return SPG_E_BADARG;
    if (rows == 0) return SPG_OK;
    if (!g_pooled || !argmax || !G) return SPG_E_BADARG;
    int64_t gy = ceil_div64(rows, 64);
    if (gy > 8 * kNumSMs) gy = 8 * kNumSMs;
    dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)gy);
    return with_segs(L, offsets, row_seg, [&](auto segs) {
        SPG_LAUNCH(K_SEGMAX_BWD, (cudaStream_t)stream, segmax_bwd_kernel<decltype(segs)>, grid, 256, 0,
                   g_pooled, ldg, argmax, G, ldG, rows, segs, C);
        return launch_status();
    });
}

int spg_segmax_bn_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, const float* Y,
                      int64_t ldy, const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, float* s12, float* dY, int64_t lddy,
                      float* workspace, int64_t B, int L, const int64_t* offsets, const int32_t* row_seg,
                      int64_t rows, int C, spg_stream_t stream) {
    if (B <= 0 || rows <= 0 || C <= 0 || !g_pooled || !argmax || !Y || !scale || !shift || !mean || !var ||
        !s12 || !dY || !workspace)
        return SPG_E_BADARG;
    if (offsets ? !row_seg : (L <= 0 || rows != B * L)) return SPG_E_BADARG;
    if ((C & 3) || (ldy & 3) || (lddy & 3)) return SPG_E_UNSUPPORTED;
    if (((uintptr_t)argmax | (uintptr_t)Y | (uintptr_t)dY) & 15) return SPG_E_ALIGN;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t chunks = ceil_div64(B, 256);
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    return with_segs(L, offsets, row_seg, [&](auto segs) {
        dim3 g1((unsigned)ceil_div64(C, 32), (unsigned)chunks);
        SPG_LAUNCH(K_SEGMAX_BWD, s, segmax_bn_bwd_reduce_kernel<decltype(segs)>, g1, 256, 0, g_pooled, ldg,
                   argmax, Y, ldy, scale, shift, mean, var, eps, relu, workspace, B, segs, C);
        int rc = launch_status();
        if (rc) return rc;
        rc = colsum_merge(K_SEGMAX_BWD, workspace, chunks, 2 * C, s12, s);
        if (rc) return rc;
        int64_t gy = ceil_div64(rows, 32);
        if (gy > 16 * kNumSMs) gy = 16 * kNumSMs;
        dim3 g2((unsigned)ceil_div64(C, 128), (unsigned)gy);
        SPG_LAUNCH(K_SEGMAX_BWD, s, segmax_bn_bwd_apply_kernel<decltype(segs)>, g2, 256, 0, g_pooled, ldg,
                   argmax, Y, ldy, scale, shift, mean, var, eps, relu, s12, s12 + C, dY, lddy, rows, segs, C);
        return launch_status();
    });
}

int spg_stn_apply_bwd(const float* clouds, const float* dXrows, int64_t ld, float* dT, int64_t B,
                      int F, int L, spg_stream_t stream) {
    if (B < 0 || F < 2 || L <= 0 || ld < 2) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!clouds || !dXrows || !dT) return SPG_E_BADARG;
    if (B > 2147483647ll) return SPG_E_UNSUPPORTED;
    SPG_LAUNCH(K_STN_APPLY_BWD, (cudaStream_t)stream, stn_apply_bwd_kernel, (unsigned)B, 128, 0,
               clouds, dXrows, ld, dT, F, L);
    return launch_status();
}

int spg_rows_scatter(const float* src, const int64_t* idx, float* dst, int64_t n_src, int C,
                     spg_stream_t stream) {
    if (n_src < 0 || C <= 0) return SPG_E_BADARG;
    if (n_src == 0) return SPG_OK;
    if (!src || !idx || !dst) return SPG_E_BADARG;
    SPG_LAUNCH(K_ROWS_SCATTER, (cudaStream_t)stream, rows_scatter_kernel,
               (unsigned)ceil_div64(n_src * C, 256), 256, 0, src, idx, dst, n_src, C);
    return launch_status();
}

int spg_rows_gather(const float* src, const int64_t* idx, float* dst, int64_t n_dst, int C,
                    spg_stream_t stream) {
    if (n_dst < 0 || C <= 0) return SPG_E_BADARG;
    if (n_dst == 0) return SPG_OK;
    if (!src || !idx || !dst) return SPG_E_BADARG;
    SPG_LAUNCH(K_ROWS_GATHER, (cudaStream_t)stream, rows_gather_kernel,
               (unsigned)ceil_div64(n_dst * C, 256), 256, 0, src, idx, dst, n_dst, C);
    return launch_status();
}

int spg_rows_to_clouds(const float* rows, int64_t ld, float* clouds, int64_t B, int F, int L,
                       spg_stream_t stream) {
    if (B < 0 || F <= 0 || L <= 0 || ld < F) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!rows || !clouds) return SPG_E_BADARG;
    const size_t smem = sizeof(float) * (size_t)F * (kPtChunk + 1);
    if (smem > 48 * 1024 || B > 2147483647ll) return SPG_E_UNSUPPORTED;
    dim3 grid((unsigned)B, (unsigned)ceil_div64(L, kPtChunk));
    SPG_LAUNCH(K_CLOUD_ROWS, (cudaStream_t)stream, rows_to_clouds_kernel, grid, kPtChunk, smem, rows, ld, clouds, F,
               L);
    return launch_status();
}

int spg_rows_xy_transform(const float* rows_in, const float* T, int add_eye, const int32_t* row_seg,
                          float* rows_out, int64_t P, int64_t ld, spg_stream_t stream) {
    if (P < 0 || ld < 2) return SPG_E_BADARG;
    if (P == 0) return SPG_OK;
    if (!rows_in || !T || !row_seg || !rows_out) return SPG_E_BADARG;
    SPG_LAUNCH(K_CLOUD_ROWS, (cudaStream_t)stream, rows_xy_transform_kernel, (unsigned)ceil_div64(P * ld, 256),
               256, 0, rows_in, T, add_eye, row_seg, rows_out, P, ld);
    return launch_status();
}

int spg_rows_xy_transform_bwd(const float* rows_in, int64_t ld, const float* d_rows_out, int64_t ld_d,
                              const int64_t* offsets, float* dT, int64_t B, spg_stream_t stream) {
    if (B < 0 || ld < 2 || ld_d < 2) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!rows_in || !d_rows_out || !offsets || !dT) return SPG_E_BADARG;
    SPG_LAUNCH(K_STN_APPLY_BWD, (cudaStream_t)stream, rows_xy_transform_bwd_kernel,
               (unsigned)ceil_div64(B * 32, 256), 256, 0, rows_in, ld, d_rows_out, ld_d, offsets, dT, B);
    return launch_status();
}

}  // extern "C"
