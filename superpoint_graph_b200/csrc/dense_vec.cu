// 128-bit vectorised variants of the column reductions / element-wise passes of dense.cu.
// Used when C % 4 == 0 and all pointers / leading dimensions are 16-byte aligned (always true
// for the PointNet / filter-network layers); dense.cu keeps the scalar kernels for odd shapes.
// A warp covers 128 consecutive columns of one row (512 B), 8 row lanes per CTA, 256 rows per
// CTA, 4 independent float4 loads in flight per thread and tensor.
// DROP kernels apply dropout (philox.cuh): C % 4 == 0 and c % 4 == 0, so the float4 at (r, c) is
// exactly the Philox group (r*C + c) >> 2 and its lane j uses word j.
#include "common.cuh"
#include "philox.cuh"

namespace spg {

constexpr int kVecRows = 256;

__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// Lane mapping shared by all kernels of this file.  A row of C floats is C/4 float4 lanes; for
// C >= 128 a warp spans 128 columns of one row, for narrower power-of-two rows (C = 64, 32, ...)
// the warp is folded over 32/(C/4) consecutive rows so that no lane idles (half of the PointNet
// layers are 64 wide).  x: float4 column lane, sub: row within the warp's row group.
struct LaneMap {
    int cpl;   // float4 lanes per row handled by one warp
    int rpw;   // rows per warp step
    int x, sub;
};
__host__ __device__ __forceinline__ int lanes_per_row(int C) {
    const int q = C >> 2;
    return (q < 32 && (q & (q - 1)) == 0) ? q : 32;
}
__device__ __forceinline__ LaneMap lane_map(int C) {
    LaneMap m;
    const int lane = threadIdx.x & 31;
    m.cpl = lanes_per_row(C);
    m.rpw = 32 / m.cpl;
    m.x = lane % m.cpl;
    m.sub = lane / m.cpl;
    return m;
}
__device__ __forceinline__ float4 fold_rows(float4 a, int cpl) {
    for (int o = cpl; o < 32; o <<= 1) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
        a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
        a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
    }
    return a;
}

template <bool DROP>
__global__ void __launch_bounds__(256)
act_bwd_reduce_v4_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                         int64_t ldy, const float* __restrict__ scale,
                         const float* __restrict__ shift, const float* __restrict__ mean,
                         const float* __restrict__ var, float eps, int relu,
                         float* __restrict__ ws, int64_t M, int C, float p,
                         const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    __shared__ float4 s1[8][32], s2[8][32];
    const LaneMap lm = lane_map(C);
    const int x = lm.x, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * 4;
    const int64_t r0 = (int64_t)blockIdx.y * kVecRows;
    const int64_t r1 = min(M, r0 + kVecRows);
    float4 a1 = f4zero(), a2 = f4zero();
    if (c < C) {
        const float4 sc = *reinterpret_cast<const float4*>(scale + c);
        const float4 sh = *reinterpret_cast<const float4*>(shift + c);
        const float4 mu = *reinterpret_cast<const float4*>(mean + c);
        const float4 vr = *reinterpret_cast<const float4*>(var + c);
        const float4 rs = make_float4(1.f / sqrtf(vr.x + eps), 1.f / sqrtf(vr.y + eps),
                                      1.f / sqrtf(vr.z + eps), 1.f / sqrtf(vr.w + eps));
        const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll 4
        for (int64_t r = r0 + y * lm.rpw + lm.sub; r < r1; r += 8 * lm.rpw) {
            const float4 yv = __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c));
            float4 g = __ldg(reinterpret_cast<const float4*>(G + r * ldg + c));
            if constexpr (DROP) {
                const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)((r * C + c) >> 2));
                g.x = drop1(d, w.v[0], g.x);
                g.y = drop1(d, w.v[1], g.y);
                g.z = drop1(d, w.v[2], g.z);
                g.w = drop1(d, w.v[3], g.w);
            }
            if (relu) {
                if (!(fmaf(yv.x, sc.x, sh.x) > 0.f)) g.x = 0.f;
                if (!(fmaf(yv.y, sc.y, sh.y) > 0.f)) g.y = 0.f;
                if (!(fmaf(yv.z, sc.z, sh.z) > 0.f)) g.z = 0.f;
                if (!(fmaf(yv.w, sc.w, sh.w) > 0.f)) g.w = 0.f;
            }
            a1.x += g.x; a1.y += g.y; a1.z += g.z; a1.w += g.w;
            a2.x = fmaf(g.x, (yv.x - mu.x) * rs.x, a2.x);
            a2.y = fmaf(g.y, (yv.y - mu.y) * rs.y, a2.y);
            a2.z = fmaf(g.z, (yv.z - mu.z) * rs.z, a2.z);
            a2.w = fmaf(g.w, (yv.w - mu.w) * rs.w, a2.w);
        }
    }
    a1 = fold_rows(a1, lm.cpl);
    a2 = fold_rows(a2, lm.cpl);
    s1[y][threadIdx.x & 31] = a1;
    s2[y][threadIdx.x & 31] = a2;
    __syncthreads();
    if (y == 0 && lm.sub == 0 && c < C) {
        float4 t1 = f4zero(), t2 = f4zero();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 u = s1[j][x], v = s2[j][x];
            t1.x += u.x; t1.y += u.y; t1.z += u.z; t1.w += u.w;
            t2.x += v.x; t2.y += v.y; t2.z += v.z; t2.w += v.w;
        }
        *reinterpret_cast<float4*>(ws + ((int64_t)blockIdx.y * 2) * C + c) = t1;
        *reinterpret_cast<float4*>(ws + ((int64_t)blockIdx.y * 2 + 1) * C + c) = t2;
    }
}

__global__ void __launch_bounds__(256)
colsum_v4_kernel(const float* __restrict__ X, int64_t ldx, int64_t M, int C,
                 float* __restrict__ ws) {
    SPG_PDL_ENTRY();
    __shared__ float4 s[8][32];
    const LaneMap lm = lane_map(C);
    const int x = lm.x, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * 4;
    const int64_t r0 = (int64_t)blockIdx.y * kVecRows;
    const int64_t r1 = min(M, r0 + kVecRows);
    float4 a = f4zero();
    if (c < C) {
#pragma unroll 4
        for (int64_t r = r0 + y * lm.rpw + lm.sub; r < r1; r += 8 * lm.rpw) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(X + r * ldx + c));
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
    }
    a = fold_rows(a, lm.cpl);
    s[y][threadIdx.x & 31] = a;
    __syncthreads();
    if (y == 0 && lm.sub == 0 && c < C) {
        float4 t = f4zero();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 u = s[j][x];
            t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
        }
        *reinterpret_cast<float4*>(ws + (int64_t)blockIdx.y * C + c) = t;
    }
}

// out[c] = sum_k ws[k*C + c], one warp per column, fp64 accumulation, fixed order.
__global__ void __launch_bounds__(128)
colsum_merge_kernel(const float* __restrict__ ws, int64_t chunks, int C, float* __restrict__ out) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (c >= C) return;
    double a = 0.0;
    for (int64_t k = lane; k < chunks; k += 32) a += (double)__ldg(ws + k * C + c);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) out[c] = (float)a;
}

template <bool DROP>
__global__ void __launch_bounds__(256)
act_bwd_apply_v4_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                        int64_t ldy, const float* __restrict__ scale,
                        const float* __restrict__ shift, const float* __restrict__ mean,
                        const float* __restrict__ var, float eps, int relu, int has_bn,
                        const float* __restrict__ s1, const float* __restrict__ s2,
                        float* __restrict__ dY, int64_t lddy, int64_t M, int C, float p,
                        const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    const LaneMap lm = lane_map(C);
    const int x = lm.x, y = (threadIdx.x >> 5) * lm.rpw + lm.sub;
    const int rows_per_block = 8 * lm.rpw;
    const int c = (blockIdx.x * 32 + x) * 4;
    if (c >= C) return;
    float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
    float mu[4] = {0.f, 0.f, 0.f, 0.f}, rs[4] = {1.f, 1.f, 1.f, 1.f};
    float m1[4] = {0.f, 0.f, 0.f, 0.f}, m2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (scale) sc[j] = scale[c + j];
        if (shift) sh[j] = shift[c + j];
        if (has_bn) {
            mu[j] = mean[c + j];
            rs[j] = 1.f / sqrtf(var[c + j] + eps);
            m1[j] = s1[c + j] / (float)M;
            m2[j] = s2[c + j] / (float)M;
        }
    }
    const DropParams dp = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll 4
    for (int64_t r = (int64_t)blockIdx.y * rows_per_block + y; r < M;
         r += (int64_t)gridDim.y * rows_per_block) {
        float4 yq = f4zero();
        if (Y) yq = __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c));
        const float4 gq = __ldg(reinterpret_cast<const float4*>(G + r * ldg + c));
        const float yv[4] = {yq.x, yq.y, yq.z, yq.w};
        float g[4] = {gq.x, gq.y, gq.z, gq.w};
        if constexpr (DROP) {
            const Philox4 w = dropout_words(dp.seed, dp.ctr, (uint64_t)((r * C + c) >> 2));
#pragma unroll
            for (int j = 0; j < 4; ++j) g[j] = drop1(dp, w.v[j], g[j]);
        }
        float d[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (relu && !(fmaf(yv[j], sc[j], sh[j]) > 0.f)) g[j] = 0.f;
            d[j] = has_bn ? sc[j] * (g[j] - m1[j] - (yv[j] - mu[j]) * rs[j] * m2[j]) : g[j];
        }
        *reinterpret_cast<float4*>(dY + r * lddy + c) = make_float4(d[0], d[1], d[2], d[3]);
    }
}

template <bool DROP>
__global__ void __launch_bounds__(256)
affine_act_v4_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                     const float* __restrict__ shift, int relu, float* __restrict__ out,
                     int64_t ldo, int64_t M, int C, float p, const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    const LaneMap lm = lane_map(C);
    const int x = lm.x, y = (threadIdx.x >> 5) * lm.rpw + lm.sub;
    const int rows_per_block = 8 * lm.rpw;
    const int c = (blockIdx.x * 32 + x) * 4;
    if (c >= C) return;
    float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (scale) sc[j] = scale[c + j];
        if (shift) sh[j] = shift[c + j];
    }
    const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll 4
    for (int64_t r = (int64_t)blockIdx.y * rows_per_block + y; r < M;
         r += (int64_t)gridDim.y * rows_per_block) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c));
        float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[j] = fmaf(v[j], sc[j], sh[j]);
            if (relu) v[j] = fmaxf(v[j], 0.f);
        }
        if constexpr (DROP) {
            const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)((r * C + c) >> 2));
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = drop1(d, w.v[j], v[j]);
        }
        *reinterpret_cast<float4*>(out + r * ldo + c) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

int colsum_merge(int kid, const float* ws, int64_t chunks, int C, float* out, cudaStream_t s) {
    SPG_LAUNCH(kid, s, colsum_merge_kernel, (unsigned)ceil_div64(C, 4), 128, 0, ws, chunks, C, out);
    return launch_status();
}

static inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }
static inline bool ld4(int64_t ld) { return (ld & 3) == 0; }

// CTAs along the rows of the element-wise passes.  The masked (DROP) passes are bound by the Philox
// latency, not by bandwidth: they get one row step per thread where the cap allows.
static inline unsigned row_grid(int64_t M, int C, bool drop) {
    int64_t g = ceil_div64(M, drop ? 8 * (32 / lanes_per_row(C)) : 32);
    if (g > 16 * kNumSMs) g = 16 * kNumSMs;
    return (unsigned)(g < 1 ? 1 : g);
}

bool vec_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                        const float* scale, const float* shift, const float* mean,
                        const float* var, float eps, int relu, float* s12, float* ws,
                        int64_t M, int C, float p, const int64_t* slot, cudaStream_t s, int* rc) {
    if ((C & 3) || !ld4(ldg) || !ld4(ldy) || !al16(G) || !al16(Y) || !al16(scale) ||
        !al16(shift) || !al16(mean) || !al16(var) || !al16(ws))
        return false;
    const int64_t chunks = ceil_div64(M, kVecRows);
    if (chunks > 65535) return false;
    const bool drop = slot != nullptr;
    dim3 grid((unsigned)ceil_div64(C, 128), (unsigned)chunks);
    SPG_LAUNCH(drop ? K_DROPOUT_BWD_REDUCE : K_ACT_BWD_REDUCE, s,
               (drop ? act_bwd_reduce_v4_kernel<true> : act_bwd_reduce_v4_kernel<false>), grid, 256,
               0, G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, ws, M, C, p, slot);
    *rc = launch_status();
    if (*rc) return true;
    // the [chunk][2][C] partials are 2*chunks rows of C: even rows -> s1, odd rows -> s2
    *rc = colsum_merge(drop ? K_DROPOUT_BWD_REDUCE_FINAL : K_ACT_BWD_REDUCE_FINAL, ws, chunks, 2 * C, s12, s);
    return true;
}

bool vec_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* ws,
                cudaStream_t s, int* rc) {
    if ((C & 3) || !ld4(ldx) || !al16(X) || !al16(ws)) return false;
    const int64_t chunks = ceil_div64(M, kVecRows);
    if (chunks > 65535) return false;
    dim3 grid((unsigned)ceil_div64(C, 128), (unsigned)chunks);
    SPG_LAUNCH(K_COLSUM_PARTIAL, s, colsum_v4_kernel, grid, 256, 0, X, ldx, M, C, ws);
    *rc = launch_status();
    if (*rc) return true;
    *rc = colsum_merge(K_COLSUM_FINAL, ws, chunks, C, out, s);
    return true;
}

bool vec_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, int has_bn, const float* s1,
                       const float* s2, float* dY, int64_t lddy, int64_t M, int C, float p,
                       const int64_t* slot, cudaStream_t s, int* rc) {
    if ((C & 3) || !ld4(ldg) || !ld4(lddy) || !al16(G) || !al16(dY)) return false;
    if (Y && (!ld4(ldy) || !al16(Y))) return false;
    const bool drop = slot != nullptr;
    dim3 grid((unsigned)ceil_div64(C, 128), row_grid(M, C, drop));
    SPG_LAUNCH(drop ? K_DROPOUT_BWD_APPLY : K_ACT_BWD_APPLY, s,
               (drop ? act_bwd_apply_v4_kernel<true> : act_bwd_apply_v4_kernel<false>), grid, 256,
               0, G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, has_bn, s1, s2, dY, lddy, M,
               C, p, slot);
    *rc = launch_status();
    return true;
}

bool vec_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                    float* out, int64_t ldo, int64_t M, int C, float p, const int64_t* slot,
                    cudaStream_t s, int* rc) {
    if ((C & 3) || !ld4(ldy) || !ld4(ldo) || !al16(Y) || !al16(out)) return false;
    const bool drop = slot != nullptr;
    dim3 grid((unsigned)ceil_div64(C, 128), row_grid(M, C, drop));
    SPG_LAUNCH(drop ? K_DROPOUT_FWD : K_AFFINE_ACT, s,
               (drop ? affine_act_v4_kernel<true> : affine_act_v4_kernel<false>), grid, 256, 0, Y,
               ldy, scale, shift, relu, out, ldo, M, C, p, slot);
    *rc = launch_status();
    return true;
}

}  // namespace spg
