// GroupNorm over point segments: nn.GroupNorm(G, C) of the reference's norm='layer' | 'group' PointNets and
// spatial transformers, followed by ReLU and training-mode dropout, on point-major rows [rows, C]:
//   gn_fwd  mean [S, G, 2], rstd [S, G] of every (segment, group) and a = drop(relu?((y - mean)*rstd*gamma + beta))
//   gn_bwd  dY = rstd*(gh - mean(gh) - xhat*mean(gh*xhat)), gh = g*gamma, g = relu'(.)*drop'(G), and per-CTA
//           partials of d_beta = sum g, d_gamma = sum g*xhat, merged in fp64 by colsum_merge
// The statistics of (segment b, group g) run over the rows of b and the C/G columns of g, biased variance.
// A conv layer's segments are the clouds (FixedSegs{L} or CsrSegs); an FC layer's are its rows (FixedSegs{1}).
//
// A warp owns one segment at a time; the warps stride over the segments in a fixed order, so that every sum
// has one order and the backward writes a bounded number of partial rows (one per CTA).  Within a segment,
// lane x covers the V columns (k*cpl + x)*V .. +V of column chunk k, and narrow power-of-two rows fold the
// warp over 32/(C/V) rows, as in bn_act.cu.  The forward reads the segment three times (sum, centred sum of
// squares, apply); the second and third reads come from L1/L2 at point-cloud segment sizes.  The sums of the
// statistics are fp64, so that a group whose mean is large against its spread keeps its variance, and the
// mean is kept as a pair of floats (hi, lo = mean - hi): y - hi is exact for y near the mean, so the centred
// value (y - hi) - lo keeps float precision relative to the spread, not to the mean.
// DROP: dropout with probability p, mask of `slot` at logical index r*C + c (philox.cuh), as affine_act.
#include <initializer_list>

#include "common.cuh"
#include "philox.cuh"
#include "segs.cuh"

namespace spg {

constexpr int kGnWarps = 4;    // warps per CTA
constexpr int kGnMaxC = 1024;  // shared memory: (2C + 2G) doubles + 2C floats per warp in the backward

template <int V>
struct GnV {
    float v[V];
};

template <int V>
__device__ __forceinline__ GnV<V> gn_ld(const float* p) {
    GnV<V> a;
    if constexpr (V == 4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(p));
        a.v[0] = q.x; a.v[1] = q.y; a.v[2] = q.z; a.v[3] = q.w;
    } else {
        a.v[0] = __ldg(p);
    }
    return a;
}

template <int V>
__device__ __forceinline__ void gn_st(float* p, const GnV<V>& a) {
    if constexpr (V == 4)
        *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
    else
        *p = a.v[0];
}

// a = drop'(a) for the V elements at row r, columns c ..  (V = 4: c % 4 == 0 and C % 4 == 0, so the four
// elements are exactly one Philox group)
template <int V>
__device__ __forceinline__ void gn_drop(const DropParams& d, int64_t r, int C, int c, GnV<V>& a) {
    if constexpr (V == 4) {
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)((r * C + c) >> 2));
#pragma unroll
        for (int j = 0; j < 4; ++j) a.v[j] = drop1(d, w.v[j], a.v[j]);
    } else {
        a.v[0] = drop_at(d, r * C + c, a.v[0]);
    }
}

// nv: V-wide column lanes of a row; cpl of them per warp row, rpw rows per warp step, `chunks` column chunks.
struct GnLanes {
    int nv, cpl, rpw, x, sub, chunks;
};

template <int V>
__device__ __forceinline__ GnLanes gn_lanes(int C) {
    GnLanes m;
    const int lane = threadIdx.x & 31;
    m.nv = C / V;
    m.cpl = (m.nv < 32 && (m.nv & (m.nv - 1)) == 0) ? m.nv : 32;
    m.rpw = 32 / m.cpl;
    m.x = lane % m.cpl;
    m.sub = lane / m.cpl;
    m.chunks = (m.nv + m.cpl - 1) / m.cpl;
    return m;
}

// 1/x for a row count x >= 1: the fast float reciprocal refined by two Newton steps (no call to the slow
// paths of IEEE division, which would give the kernels a stack frame)
__device__ __forceinline__ double gn_recip(double x) {
    double r = (double)__fdividef(1.f, (float)x);
    r = r * fma(-x, r, 2.0);
    return r * fma(-x, r, 2.0);
}

// sum over the rows a warp folds together
template <class T>
__device__ __forceinline__ T gn_fold(T a, int cpl) {
    for (int o = cpl; o < 32; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    return a;
}

// out[g] = scale * sum over the columns c of group g of col[c] (* wt[c] if wt), fp64, one fixed order
__device__ __forceinline__ void gn_group_sums(const double* col, const float* __restrict__ wt, int G, int gs,
                                              double scale, double* out) {
    const int lane = threadIdx.x & 31;
    for (int g = 0; g < G; ++g) {
        double a = 0.0;
        for (int j = lane; j < gs; j += 32) {
            const int c = g * gs + j;
            a += wt ? col[c] * (double)__ldg(wt + c) : col[c];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) out[g] = a * scale;
    }
    __syncwarp();
}

// col[c] = sum over the n rows of Yb of y (CENTRED: of (y - mu[group of c])^2), fp64.
template <int V, bool CENTRED>
__device__ __forceinline__ void gn_col_sums(const GnLanes& lm, const float* __restrict__ Yb, int64_t ldy, int n,
                                            int gs, const double* mu, double* col) {
    for (int k = 0; k < lm.chunks; ++k) {
        const int cv = k * lm.cpl + lm.x;
        const int c = cv * V;
        const bool active = cv < lm.nv;
        double m[V], a[V];
#pragma unroll
        for (int j = 0; j < V; ++j) {
            m[j] = (CENTRED && active) ? mu[(c + j) / gs] : 0.0;
            a[j] = 0.0;
        }
        if (active) {
            for (int l = lm.sub; l < n; l += lm.rpw) {
                const GnV<V> y = gn_ld<V>(Yb + (int64_t)l * ldy + c);
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    if (CENTRED) {
                        const double t = (double)y.v[j] - m[j];
                        a[j] = fma(t, t, a[j]);
                    } else {
                        a[j] += (double)y.v[j];
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < V; ++j) a[j] = gn_fold(a[j], lm.cpl);
        if (active && lm.sub == 0)
#pragma unroll
            for (int j = 0; j < V; ++j) col[c + j] = a[j];
    }
    __syncwarp();
}

// grid: gn_grid(S) CTAs of kGnWarps warps; dynamic smem gn_fwd_smem(C, G).
template <class Segs, int V, bool DROP>
__global__ void __launch_bounds__(kGnWarps * 32, 4)
gn_fwd_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ gamma,
              const float* __restrict__ beta, float eps, int relu, float* __restrict__ out, int64_t ldo,
              float* __restrict__ mean, float* __restrict__ rstd, int64_t S, Segs segs, int C, int G, float p,
              const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    extern __shared__ double gn_smem[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double* col = gn_smem + (int64_t)w * (C + 2 * G);  // per-column sums of the current segment
    double* gmu = col + C;                              // group means
    double* grs = gmu + G;                              // group variances, then the float rstd
    const int gs = C / G;
    const GnLanes lm = gn_lanes<V>(C);
    const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
    for (int64_t b = (int64_t)blockIdx.x * kGnWarps + w; b < S; b += (int64_t)gridDim.x * kGnWarps) {
        const int64_t r0 = segs.begin(b);
        const int n = (int)(segs.end(b) - r0);
        if (Segs::kMayBeEmpty && n == 0) {  // no rows: nothing to normalise, statistics 0
            for (int g = lane; g < G; g += 32) mean[2 * (b * G + g)] = mean[2 * (b * G + g) + 1] = rstd[b * G + g] = 0.f;
            continue;
        }
        const float* Yb = Y + r0 * ldy;
        const double inv_cnt = gn_recip((double)n * gs);
        gn_col_sums<V, false>(lm, Yb, ldy, n, gs, nullptr, col);
        gn_group_sums(col, nullptr, G, gs, inv_cnt, gmu);
        gn_col_sums<V, true>(lm, Yb, ldy, n, gs, gmu, col);
        gn_group_sums(col, nullptr, G, gs, inv_cnt, grs);
        for (int g = lane; g < G; g += 32) {
            const float hi = (float)gmu[g], rs = rsqrtf((float)grs[g] + eps);
            mean[2 * (b * G + g)] = hi;
            mean[2 * (b * G + g) + 1] = (float)(gmu[g] - (double)hi);
            rstd[b * G + g] = rs;
            grs[g] = rs;
        }
        __syncwarp();
        for (int k = 0; k < lm.chunks; ++k) {
            const int cv = k * lm.cpl + lm.x;
            const int c = cv * V;
            if (cv >= lm.nv) continue;
            float mh[V], ml[V], a[V], bt[V];
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const int g = (c + j) / gs;
                mh[j] = (float)gmu[g];
                ml[j] = (float)(gmu[g] - (double)mh[j]);
                a[j] = (float)grs[g] * __ldg(gamma + c + j);
                bt[j] = __ldg(beta + c + j);
            }
            for (int l = lm.sub; l < n; l += lm.rpw) {
                GnV<V> v = gn_ld<V>(Yb + (int64_t)l * ldy + c);
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    v.v[j] = fmaf((v.v[j] - mh[j]) - ml[j], a[j], bt[j]);
                    if (relu) v.v[j] = fmaxf(v.v[j], 0.f);
                }
                if constexpr (DROP) gn_drop<V>(d, r0 + l, C, c, v);
                gn_st<V>(out + (r0 + l) * ldo + c, v);
            }
        }
        __syncwarp();  // the next segment's sums overwrite gmu / grs
    }
}

// grid: gn_grid(S) CTAs; dynamic smem gn_bwd_smem(C, G); ws [gridDim.x][2C] = per-CTA (sum g | sum g*xhat).
template <class Segs, int V, bool DROP>
__global__ void __launch_bounds__(kGnWarps * 32, 4)
gn_bwd_kernel(const float* __restrict__ Gr, int64_t ldg, const float* __restrict__ Y, int64_t ldy,
              const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
              const float* __restrict__ beta, int relu, float* __restrict__ dY, int64_t lddy,
              float* __restrict__ ws, int64_t S, Segs segs, int C, int G, float p,
              const int64_t* __restrict__ slot) {
    SPG_PDL_ENTRY();
    extern __shared__ double gn_smem[];
    const int w = threadIdx.x >> 5;
    double* s1 = gn_smem + (int64_t)w * (2 * C + 2 * G);  // sum g, sum g*xhat of the current segment
    double* s2 = s1 + C;
    double* m1 = s2 + C;  // mean(gh), mean(gh*xhat) of every group
    double* m2 = m1 + G;
    float* acc = reinterpret_cast<float*>(gn_smem + (int64_t)kGnWarps * (2 * C + 2 * G));  // [warp][2C]
    float* acc1 = acc + (int64_t)w * 2 * C;
    float* acc2 = acc1 + C;
    for (int i = threadIdx.x; i < kGnWarps * 2 * C; i += blockDim.x) acc[i] = 0.f;
    __syncthreads();
    const int gs = C / G;
    const GnLanes lm = gn_lanes<V>(C);
    const DropParams d = DROP ? drop_params(slot, p) : DropParams{};
    for (int64_t b = (int64_t)blockIdx.x * kGnWarps + w; b < S; b += (int64_t)gridDim.x * kGnWarps) {
        const int64_t r0 = segs.begin(b);
        const int n = (int)(segs.end(b) - r0);
        if (Segs::kMayBeEmpty && n == 0) continue;  // no rows, no gradient
        const double inv_cnt = gn_recip((double)n * gs);
        // pass 1: column sums of g and g*xhat (-> d_beta, d_gamma and the group means of gh, gh*xhat)
        for (int k = 0; k < lm.chunks; ++k) {
            const int cv = k * lm.cpl + lm.x;
            const int c = cv * V;
            const bool active = cv < lm.nv;
            float mh[V], ml[V], rs[V], a[V], bt[V], t1[V], t2[V];
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const int g = active ? (c + j) / gs : 0;
                mh[j] = __ldg(mean + 2 * (b * G + g));
                ml[j] = __ldg(mean + 2 * (b * G + g) + 1);
                rs[j] = __ldg(rstd + b * G + g);
                a[j] = active ? rs[j] * __ldg(gamma + c + j) : 0.f;
                bt[j] = active ? __ldg(beta + c + j) : 0.f;
                t1[j] = t2[j] = 0.f;
            }
            if (active) {
                for (int l = lm.sub; l < n; l += lm.rpw) {
                    const int64_t r = r0 + l;
                    const GnV<V> y = gn_ld<V>(Y + r * ldy + c);
                    GnV<V> g = gn_ld<V>(Gr + r * ldg + c);
                    if constexpr (DROP) gn_drop<V>(d, r, C, c, g);
#pragma unroll
                    for (int j = 0; j < V; ++j) {
                        const float yc = (y.v[j] - mh[j]) - ml[j];
                        const float gj = (!relu || fmaf(yc, a[j], bt[j]) > 0.f) ? g.v[j] : 0.f;
                        t1[j] += gj;
                        t2[j] = fmaf(gj, yc * rs[j], t2[j]);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < V; ++j) {
                t1[j] = gn_fold(t1[j], lm.cpl);
                t2[j] = gn_fold(t2[j], lm.cpl);
            }
            if (active && lm.sub == 0)
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    s1[c + j] = t1[j];
                    s2[c + j] = t2[j];
                    acc1[c + j] += t1[j];
                    acc2[c + j] += t2[j];
                }
        }
        __syncwarp();
        gn_group_sums(s1, gamma, G, gs, inv_cnt, m1);
        gn_group_sums(s2, gamma, G, gs, inv_cnt, m2);
        // pass 2: dY
        for (int k = 0; k < lm.chunks; ++k) {
            const int cv = k * lm.cpl + lm.x;
            const int c = cv * V;
            if (cv >= lm.nv) continue;
            float mh[V], ml[V], rs[V], a[V], bt[V], gm[V], q1[V], q2[V];
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const int g = (c + j) / gs;
                mh[j] = __ldg(mean + 2 * (b * G + g));
                ml[j] = __ldg(mean + 2 * (b * G + g) + 1);
                rs[j] = __ldg(rstd + b * G + g);
                gm[j] = __ldg(gamma + c + j);
                a[j] = rs[j] * gm[j];
                bt[j] = __ldg(beta + c + j);
                q1[j] = (float)m1[g];
                q2[j] = (float)m2[g];
            }
            for (int l = lm.sub; l < n; l += lm.rpw) {
                const int64_t r = r0 + l;
                const GnV<V> y = gn_ld<V>(Y + r * ldy + c);
                GnV<V> g = gn_ld<V>(Gr + r * ldg + c);
                if constexpr (DROP) gn_drop<V>(d, r, C, c, g);
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    const float yc = (y.v[j] - mh[j]) - ml[j];
                    const float gj = (!relu || fmaf(yc, a[j], bt[j]) > 0.f) ? g.v[j] : 0.f;
                    g.v[j] = rs[j] * (gj * gm[j] - q1[j] - yc * rs[j] * q2[j]);
                }
                gn_st<V>(dY + r * lddy + c, g);
            }
        }
        __syncwarp();  // the next segment's sums overwrite s1, s2, m1, m2
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float t1 = 0.f, t2 = 0.f;
#pragma unroll
        for (int k = 0; k < kGnWarps; ++k) {
            t1 += acc[(int64_t)k * 2 * C + c];
            t2 += acc[(int64_t)k * 2 * C + C + c];
        }
        ws[(int64_t)blockIdx.x * 2 * C + c] = t1;
        ws[(int64_t)blockIdx.x * 2 * C + C + c] = t2;
    }
}

static int64_t gn_grid(int64_t S) {
    const int64_t g = ceil_div64(S, kGnWarps);
    const int64_t cap = 16 * kNumSMs;
    return g < 1 ? 1 : g > cap ? cap : g;
}

static size_t gn_fwd_smem(int C, int G) { return sizeof(double) * kGnWarps * (size_t)(C + 2 * G); }
static size_t gn_bwd_smem(int C, int G) {
    return sizeof(double) * kGnWarps * (size_t)(2 * C + 2 * G) + sizeof(float) * kGnWarps * (size_t)(2 * C);
}

// V = 4 if C % 4 == 0, every leading dimension is a multiple of 4 and every pointer is 16-byte aligned
static int gn_width(int C, std::initializer_list<int64_t> lds, std::initializer_list<const void*> ptrs) {
    if (C & 3) return 1;
    for (const int64_t ld : lds)
        if (ld & 3) return 1;
    for (const void* q : ptrs)
        if ((uintptr_t)q & 15) return 1;
    return 4;
}

// opts `kernel` into smem bytes of dynamic shared memory where that is above the default 48 KB
template <class K>
static int gn_smem_attr(K kernel, size_t smem) {
    if (smem <= 48 * 1024) return SPG_OK;
    return (int)cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// kernel template K instantiated for segment layout S, width V and dropout on or off
#define SPG_GN_KERNEL(K, S, V, drop) \
    ((V) == 4 ? ((drop) ? K<S, 4, true> : K<S, 4, false>) : ((drop) ? K<S, 1, true> : K<S, 1, false>))

static int gn_check(int64_t B, int L, const int64_t* offsets, int C, int G) {
    if (B < 0 || (!offsets && L <= 0) || C <= 0 || G <= 0 || C % G) return SPG_E_BADARG;
    if (C > kGnMaxC) return SPG_E_UNSUPPORTED;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int64_t spg_group_norm_partials(int64_t B) { return gn_grid(B); }

int spg_group_norm_fwd(const float* Y, int64_t ldy, const float* gamma, const float* beta, float eps, int relu,
                       float* out, int64_t ldo, float* mean, float* rstd, int64_t B, int L,
                       const int64_t* offsets, int C, int groups, float p, const int64_t* drop_slot,
                       spg_stream_t stream) {
    int rc = gn_check(B, L, offsets, C, groups);
    if (rc) return rc;
    if (drop_slot && !(p >= 0.f)) return SPG_E_BADARG;
    if (B == 0) return SPG_OK;
    if (!Y || !gamma || !beta || !out || !mean || !rstd || ldy < C || ldo < C) return SPG_E_BADARG;
    const bool drop = drop_slot != nullptr;
    const int V = gn_width(C, {ldy, ldo}, {Y, out});
    const size_t smem = gn_fwd_smem(C, groups);
    const int64_t grid = gn_grid(B);
    cudaStream_t s = (cudaStream_t)stream;
    return with_segs(L, offsets, nullptr, [&](auto segs) {
        auto kernel = SPG_GN_KERNEL(gn_fwd_kernel, decltype(segs), V, drop);
        const int e = gn_smem_attr(kernel, smem);
        if (e) return e;
        SPG_LAUNCH(K_GN_FWD, s, kernel, (unsigned)grid, kGnWarps * 32, smem, Y, ldy, gamma, beta, eps, relu, out,
                   ldo, mean, rstd, B, segs, C, groups, p, drop_slot);
        return launch_status();
    });
}

int spg_group_norm_bwd(const float* G, int64_t ldg, const float* Y, int64_t ldy, const float* mean,
                       const float* rstd, const float* gamma, const float* beta, int relu, float* dY,
                       int64_t lddy, float* dbg, float* workspace, int64_t B, int L, const int64_t* offsets,
                       int C, int groups, float p, const int64_t* drop_slot, spg_stream_t stream) {
    int rc = gn_check(B, L, offsets, C, groups);
    if (rc) return rc;
    if (drop_slot && !(p >= 0.f)) return SPG_E_BADARG;
    if (!G || !Y || !mean || !rstd || !gamma || !beta || !dY || !dbg || !workspace) return SPG_E_BADARG;
    if (ldg < C || ldy < C || lddy < C) return SPG_E_BADARG;
    const bool drop = drop_slot != nullptr;
    const int V = gn_width(C, {ldg, ldy, lddy}, {G, Y, dY});
    const size_t smem = gn_bwd_smem(C, groups);
    const int64_t grid = gn_grid(B);
    cudaStream_t s = (cudaStream_t)stream;
    return with_segs(L, offsets, nullptr, [&](auto segs) {
        auto kernel = SPG_GN_KERNEL(gn_bwd_kernel, decltype(segs), V, drop);
        int e = gn_smem_attr(kernel, smem);
        if (e) return e;
        SPG_LAUNCH(K_GN_BWD, s, kernel, (unsigned)grid, kGnWarps * 32, smem, G, ldg, Y, ldy, mean, rstd, gamma,
                   beta, relu, dY, lddy, workspace, B, segs, C, groups, p, drop_slot);
        e = launch_status();
        if (e) return e;
        // the [CTA][2C] partials -> dbg = [d_beta | d_gamma]
        return colsum_merge(K_GN_BWD_FINAL, workspace, grid, 2 * C, dbg, s);
    });
}

}  // extern "C"
