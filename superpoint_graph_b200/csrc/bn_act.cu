// The BatchNorm/ReLU activation passes and column sums under every dense layer, for any width:
//   affine_act      out = drop(relu?(Y*scale + shift))
//   act_bwd_reduce  per-chunk partials of s1 = sum g, s2 = sum g*xhat    (g = relu'(.) * drop'(G))
//   act_bwd_apply   dY = BatchNorm/ReLU backward of G
//   colsum_partial  per-chunk partials of sum X
// The reductions' [chunk][C] partials are merged in fp64 by colsum_merge.
//
// Each kernel is written once on V, the floats per lane.  V = 4 (128-bit loads) when C % 4 == 0 and
// every row and pointer is 16-byte aligned, which holds for the PointNet / filter-network layers; V = 1
// otherwise.  Lane x covers columns (blockIdx.x*32 + x)*V .. +V, 8 warps per CTA.  With V = 4 a warp
// spans 128 columns of one row, and narrower power-of-two rows (C = 64, 32, ...) fold the warp over
// 32/(C/4) consecutive rows so that no lane idles (half of the PointNet layers are 64 wide); with V = 1
// a warp spans 32 columns of one row.
// DROP: dropout with probability p, mask from `slot` (philox.cuh).  With V = 4, C % 4 == 0 and
// c % 4 == 0, so the float4 at (r, c) is exactly the Philox group (r*C + c) >> 2 and one call gives
// its four words; with V = 1 every element makes its own call (drop_at).
#include <initializer_list>

#include "common.cuh"
#include "philox.cuh"

namespace spg {

// Rows per reduction chunk.  The masked V = 1 sums spend a Philox call per element: shorter chunks,
// more CTAs.
__host__ __device__ constexpr int chunk_rows(int V, bool drop) { return V == 4 || drop ? 256 : 1024; }

// Unroll count of the row loops: 4 for V = 4.  V = 1 is left to the compiler's own choice: nvcc
// ignores a pragma with a count of 0 (and would warn about it).
__host__ __device__ constexpr int row_unroll(int V) { return V == 4 ? 4 : 0; }
#pragma nv_diag_suppress 20168

// float4 lanes of a row that one warp covers: C/4 for narrow power-of-two rows, else 32
__host__ __device__ __forceinline__ int lanes_per_row(int C) {
    const int q = C >> 2;
    return (q < 32 && (q & (q - 1)) == 0) ? q : 32;
}

// x: column lane, sub: row within the warp's group of rpw rows, cpl: column lanes per row.
struct LaneMap {
    int cpl, rpw, x, sub;
};
template <int V>
__device__ __forceinline__ LaneMap lane_map(int C) {
    LaneMap m;
    const int lane = threadIdx.x & 31;
    m.cpl = V == 4 ? lanes_per_row(C) : 32;
    m.rpw = 32 / m.cpl;
    m.x = lane % m.cpl;
    m.sub = lane / m.cpl;
    return m;
}

// The V floats of one lane, and their loads and stores.  NC: load through the read-only data cache
// (__ldg).  The reductions stream their rows that way; the element-wise passes do so at V = 4 only:
// at V = 1 the compiler unrolls their row loop over plain loads but not over __ldg.
template <int V>
struct alignas(4 * V) Vf {
    float v[V];
};
template <int V, bool NC = false>
__device__ __forceinline__ Vf<V> vld(const float* p) {
    Vf<V> a;
    if constexpr (V == 4) {
        const float4* q4 = reinterpret_cast<const float4*>(p);
        const float4 q = NC ? __ldg(q4) : *q4;
        a.v[0] = q.x; a.v[1] = q.y; a.v[2] = q.z; a.v[3] = q.w;
    } else {
        a.v[0] = NC ? __ldg(p) : *p;
    }
    return a;
}
template <int V>
__device__ __forceinline__ void vst(float* p, const Vf<V>& a) {
    if constexpr (V == 4)
        *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
    else
        *p = a.v[0];
}

// a = drop'(a) for the V elements at row r, columns c ..
template <int V>
__device__ __forceinline__ void drop_lane(const DropParams& d, int64_t r, int C, int c, Vf<V>& a) {
    if constexpr (V == 4) {
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)((r * C + c) >> 2));
#pragma unroll
        for (int j = 0; j < 4; ++j) a.v[j] = drop1(d, w.v[j], a.v[j]);
    } else {
        a.v[0] = drop_at(d, r * C + c, a.v[0]);
    }
}

// The gradient's V elements at row r, columns c .. (p = G + r*ldg + c), read through the read-only
// cache, with drop' if DROP.  The reduction masks the float4 before splitting it: masking the split
// values made nvcc allocate the masked V = 4 reduction differently, a third slower on an H100.
template <int V, bool DROP>
__device__ __forceinline__ Vf<V> vld_grad(const float* p, const DropParams& d, int64_t r, int C, int c) {
    if constexpr (V == 4) {
        float4 q = __ldg(reinterpret_cast<const float4*>(p));
        if constexpr (DROP) {
            const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)((r * C + c) >> 2));
            q.x = drop1(d, w.v[0], q.x);
            q.y = drop1(d, w.v[1], q.y);
            q.z = drop1(d, w.v[2], q.z);
            q.w = drop1(d, w.v[3], q.w);
        }
        return Vf<V>{{q.x, q.y, q.z, q.w}};
    } else {
        Vf<V> a = vld<V, true>(p);
        if constexpr (DROP) a.v[0] = drop_at(d, r * C + c, a.v[0]);
        return a;
    }
}

// sum over the rows a warp folds together (V = 4, cpl < 32)
template <int V>
__device__ __forceinline__ void fold_rows(Vf<V>& a, int cpl) {
    for (int o = cpl; o < 32; o <<= 1)
#pragma unroll
        for (int j = 0; j < V; ++j) a.v[j] += __shfl_xor_sync(0xffffffffu, a.v[j], o);
}

template <int V, bool DROP>
__global__ void __launch_bounds__(256)
affine_act_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                  const float* __restrict__ shift, int relu, float* __restrict__ out, int64_t ldo,
                  int64_t M, int C, float p, const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    const LaneMap lm = lane_map<V>(C);
    const int x = lm.x, y = (threadIdx.x >> 5) * lm.rpw + lm.sub;
    const int rows_per_block = 8 * lm.rpw;
    const int c = (blockIdx.x * 32 + x) * V;
    if (c >= C) return;
    float sc[V], sh[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
        sc[j] = scale ? scale[c + j] : 1.f;
        sh[j] = shift ? shift[c + j] : 0.f;
    }
    const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll row_unroll(V)
    for (int64_t r = (int64_t)blockIdx.y * rows_per_block + y; r < M;
         r += (int64_t)gridDim.y * rows_per_block) {
        Vf<V> v = vld<V, V == 4>(Y + r * ldy + c);
#pragma unroll
        for (int j = 0; j < V; ++j) {
            v.v[j] = fmaf(v.v[j], sc[j], sh[j]);
            if (relu) v.v[j] = fmaxf(v.v[j], 0.f);
        }
        if constexpr (DROP) drop_lane<V>(d, r, C, c, v);
        vst<V>(out + r * ldo + c, v);
    }
}

template <int V, bool DROP>
__global__ void __launch_bounds__(256)
act_bwd_reduce_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                      int64_t ldy, const float* __restrict__ scale,
                      const float* __restrict__ shift, const float* __restrict__ mean,
                      const float* __restrict__ var, float eps, int relu, float* __restrict__ ws,
                      int64_t M, int C, float p, const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    __shared__ Vf<V> s1[8][32], s2[8][32];
    constexpr int kRows = chunk_rows(V, DROP);
    const LaneMap lm = lane_map<V>(C);
    const int x = lm.x, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * V;
    const int64_t r0 = (int64_t)blockIdx.y * kRows;
    const int64_t r1 = min(M, r0 + kRows);
    Vf<V> a1 = {}, a2 = {};
    if (c < C) {
        const Vf<V> sc = vld<V>(scale + c), sh = vld<V>(shift + c), mu = vld<V>(mean + c);
        const Vf<V> vr = vld<V>(var + c);
        float rs[V];
#pragma unroll
        for (int j = 0; j < V; ++j) rs[j] = 1.f / sqrtf(vr.v[j] + eps);
        const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll row_unroll(V)
        for (int64_t r = r0 + y * lm.rpw + lm.sub; r < r1; r += 8 * lm.rpw) {
            const Vf<V> yv = vld<V, true>(Y + r * ldy + c);
            Vf<V> g = vld_grad<V, DROP>(G + r * ldg + c, d, r, C, c);
            if (relu)
#pragma unroll
                for (int j = 0; j < V; ++j) g.v[j] = relu_bwd(g.v[j], yv.v[j], sc.v[j], sh.v[j]);
#pragma unroll
            for (int j = 0; j < V; ++j) a1.v[j] += g.v[j];
#pragma unroll
            for (int j = 0; j < V; ++j) a2.v[j] = fmaf(g.v[j], (yv.v[j] - mu.v[j]) * rs[j], a2.v[j]);
        }
    }
    fold_rows<V>(a1, lm.cpl);
    fold_rows<V>(a2, lm.cpl);
    s1[y][threadIdx.x & 31] = a1;
    s2[y][threadIdx.x & 31] = a2;
    __syncthreads();
    if (y == 0 && lm.sub == 0 && c < C) {
        Vf<V> t1 = {}, t2 = {};
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int j = 0; j < V; ++j) {
                t1.v[j] += s1[k][x].v[j];
                t2.v[j] += s2[k][x].v[j];
            }
        vst<V>(ws + ((int64_t)blockIdx.y * 2) * C + c, t1);
        vst<V>(ws + ((int64_t)blockIdx.y * 2 + 1) * C + c, t2);
    }
}

template <int V, bool DROP>
__global__ void __launch_bounds__(256)
act_bwd_apply_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                     int64_t ldy, const float* __restrict__ scale, const float* __restrict__ shift,
                     const float* __restrict__ mean, const float* __restrict__ var, float eps,
                     int relu, int has_bn, const float* __restrict__ s1,
                     const float* __restrict__ s2, float* __restrict__ dY, int64_t lddy, int64_t M,
                     int C, float p, const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    const LaneMap lm = lane_map<V>(C);
    const int x = lm.x, y = (threadIdx.x >> 5) * lm.rpw + lm.sub;
    const int rows_per_block = 8 * lm.rpw;
    const int c = (blockIdx.x * 32 + x) * V;
    if (c >= C) return;
    float sc[V], sh[V], mu[V], rs[V], m1[V], m2[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
        sc[j] = scale ? scale[c + j] : 1.f;
        sh[j] = shift ? shift[c + j] : 0.f;
        mu[j] = 0.f, rs[j] = 1.f, m1[j] = 0.f, m2[j] = 0.f;
        if (has_bn) {
            mu[j] = mean[c + j];
            rs[j] = 1.f / sqrtf(var[c + j] + eps);
            m1[j] = s1[c + j] / (float)M;
            m2[j] = s2[c + j] / (float)M;
        }
    }
    const DropParams dp = DROP ? drop_params(slot, p) : DropParams{};
#pragma unroll row_unroll(V)
    for (int64_t r = (int64_t)blockIdx.y * rows_per_block + y; r < M;
         r += (int64_t)gridDim.y * rows_per_block) {
        const Vf<V> yv = Y ? vld<V, V == 4>(Y + r * ldy + c) : Vf<V>{};
        Vf<V> g = vld<V, V == 4>(G + r * ldg + c);
        if constexpr (DROP) drop_lane<V>(dp, r, C, c, g);
        Vf<V> d;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const float gj = relu ? relu_bwd(g.v[j], yv.v[j], sc[j], sh[j]) : g.v[j];
            d.v[j] = has_bn ? bn_bwd(gj, yv.v[j], sc[j], mu[j], rs[j], m1[j], m2[j]) : gj;
        }
        vst<V>(dY + r * lddy + c, d);
    }
}

template <int V>
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ X, int64_t ldx, int64_t M, int C,
                      float* __restrict__ ws) {
    SPG_PDL_ENTRY();
    __shared__ Vf<V> s[8][32];
    constexpr int kRows = chunk_rows(V, false);
    const LaneMap lm = lane_map<V>(C);
    const int x = lm.x, y = threadIdx.x >> 5;
    const int c = (blockIdx.x * 32 + x) * V;
    const int64_t r0 = (int64_t)blockIdx.y * kRows;
    const int64_t r1 = min(M, r0 + kRows);
    Vf<V> a = {};
    if (c < C) {
#pragma unroll row_unroll(V)
        for (int64_t r = r0 + y * lm.rpw + lm.sub; r < r1; r += 8 * lm.rpw) {
            const Vf<V> v = vld<V, true>(X + r * ldx + c);
#pragma unroll
            for (int j = 0; j < V; ++j) a.v[j] += v.v[j];
        }
    }
    fold_rows<V>(a, lm.cpl);
    s[y][threadIdx.x & 31] = a;
    __syncthreads();
    if (y == 0 && lm.sub == 0 && c < C) {
        Vf<V> t = {};
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int j = 0; j < V; ++j) t.v[j] += s[k][x].v[j];
        vst<V>(ws + (int64_t)blockIdx.y * C + c, t);
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

int colsum_merge(int kid, const float* ws, int64_t chunks, int C, float* out, cudaStream_t s) {
    SPG_LAUNCH(kid, s, colsum_merge_kernel, (unsigned)ceil_div64(C, 4), 128, 0, ws, chunks, C, out);
    return launch_status();
}

// V = 4 if C % 4 == 0, every leading dimension is a multiple of 4 and every pointer is 16-byte
// aligned (NULL counts as aligned); else V = 1.
static int width(int C, std::initializer_list<int64_t> lds, std::initializer_list<const void*> ptrs) {
    if (C & 3) return 1;
    for (const int64_t ld : lds)
        if (ld & 3) return 1;
    for (const void* q : ptrs)
        if ((uintptr_t)q & 15) return 1;
    return 4;
}

// CTAs along the rows of the element-wise passes.  The masked passes are bound by the Philox latency,
// not by bandwidth: they get one row step per thread where the cap allows.
static unsigned rows_grid(int64_t M, int C, int V, bool drop) {
    const int rows_per_step = 8 * (V == 4 ? 32 / lanes_per_row(C) : 1);
    int64_t g = ceil_div64(M, drop ? rows_per_step : V == 4 ? 32 : 64);
    const int64_t cap = (V == 4 ? 16 : 8) * kNumSMs;
    if (g > cap) g = cap;
    return (unsigned)(g < 1 ? 1 : g);
}

// kernel template K instantiated for width V and dropout on or off
#define SPG_ACT_KERNEL(K, V, drop) \
    ((V) == 4 ? ((drop) ? K<4, true> : K<4, false>) : ((drop) ? K<1, true> : K<1, false>))

}  // namespace spg

using namespace spg;

extern "C" {

int spg_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* out, int64_t ldo, int64_t M, int C, float p, const int64_t* drop_slot,
                   spg_stream_t stream) {
    if (M < 0 || C <= 0 || (drop_slot && !(p >= 0.f))) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!Y || !out || ldy < C || ldo < C) return SPG_E_BADARG;
    const bool drop = drop_slot != nullptr;
    const int V = width(C, {ldy, ldo}, {Y, out});
    dim3 grid((unsigned)ceil_div64(C, 32 * V), rows_grid(M, C, V, drop));
    SPG_LAUNCH(drop ? K_DROPOUT_FWD : K_AFFINE_ACT, (cudaStream_t)stream,
               SPG_ACT_KERNEL(affine_act_kernel, V, drop), grid, 256, 0, Y, ldy, scale, shift, relu,
               out, ldo, M, C, p, drop_slot);
    return launch_status();
}

int spg_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* workspace,
               spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !X || !out || !workspace || ldx < C) return SPG_E_BADARG;
    int V = width(C, {ldx}, {X, workspace});
    if (ceil_div64(M, chunk_rows(4, false)) > 65535) V = 1;
    const int64_t chunks = ceil_div64(M, chunk_rows(V, false));
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div64(C, 32 * V), (unsigned)chunks);
    SPG_LAUNCH(K_COLSUM_PARTIAL, s, (V == 4 ? colsum_partial_kernel<4> : colsum_partial_kernel<1>), grid,
               256, 0, X, ldx, M, C, workspace);
    const int rc = launch_status();
    if (rc) return rc;
    return colsum_merge(K_COLSUM_FINAL, workspace, chunks, C, out, s);
}

int spg_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, float* s12, float* workspace,
                       int64_t M, int C, float p, const int64_t* drop_slot, spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !G || !Y || !scale || !shift || !mean || !var || !s12 ||
        !workspace || (drop_slot && !(p >= 0.f)))
        return SPG_E_BADARG;
    const bool drop = drop_slot != nullptr;
    int V = width(C, {ldg, ldy}, {G, Y, scale, shift, mean, var, workspace});
    if (ceil_div64(M, chunk_rows(4, drop)) > 65535) V = 1;
    const int64_t chunks = ceil_div64(M, chunk_rows(V, drop));
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div64(C, 32 * V), (unsigned)chunks);
    SPG_LAUNCH(drop ? K_DROPOUT_BWD_REDUCE : K_ACT_BWD_REDUCE, s,
               SPG_ACT_KERNEL(act_bwd_reduce_kernel, V, drop), grid, 256, 0, G, ldg, Y, ldy, scale,
               shift, mean, var, eps, relu, workspace, M, C, p, drop_slot);
    const int rc = launch_status();
    if (rc) return rc;
    // the [chunk][2][C] partials are 2*chunks rows of C: even rows -> s1, odd rows -> s2
    return colsum_merge(drop ? K_DROPOUT_BWD_REDUCE_FINAL : K_ACT_BWD_REDUCE_FINAL, workspace, chunks,
                        2 * C, s12, s);
}

int spg_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                      const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, int has_bn, const float* s1,
                      const float* s2, float* dY, int64_t lddy, int64_t M, int C, float p,
                      const int64_t* drop_slot, spg_stream_t stream) {
    if (M < 0 || C <= 0 || (drop_slot && !(p >= 0.f))) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!G || !dY) return SPG_E_BADARG;
    if ((relu || has_bn) && !Y) return SPG_E_BADARG;
    if (has_bn && (!scale || !shift || !mean || !var || !s1 || !s2)) return SPG_E_BADARG;
    const bool drop = drop_slot != nullptr;
    const int V = width(C, {ldg, lddy, Y ? ldy : 0}, {G, dY, Y});
    dim3 grid((unsigned)ceil_div64(C, 32 * V), rows_grid(M, C, V, drop));
    SPG_LAUNCH(drop ? K_DROPOUT_BWD_APPLY : K_ACT_BWD_APPLY, (cudaStream_t)stream,
               SPG_ACT_KERNEL(act_bwd_apply_kernel, V, drop), grid, 256, 0, G, ldg, Y, ldy, scale,
               shift, mean, var, eps, relu, has_bn, s1, s2, dY, lddy, M, C, p, drop_slot);
    return launch_status();
}

}  // extern "C"
