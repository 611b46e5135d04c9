// Training-mode dropout of a fused Linear/Conv1d [+BatchNorm] [+ReLU] layer (ref: learning/pointnet.py:109-110,
// learning/graphnet.py:54-55: nn.Dropout after the activation).
//
// The mask is a pure function of (seed, ctr, i) with i = m*C + c the logical index of element (m, c) of the
// [M, C] activation: Philox4x32-10 with key (seed_lo, seed_hi) and counter (i>>2 low word, i>>34, ctr_lo,
// ctr_hi), word i & 3; kept iff word >= floor(p * 2^32), kept elements scaled by 1/(1-p), p >= 1 drops all.
// It depends on neither grid size, leading dimension nor launch order, so the backward regenerates it instead
// of storing it.  (seed, ctr) live in device memory: spg_dropout_rng_next copies the device generator state
// into a per-site slot and advances the counter, every other kernel reads the slot — nothing about the stream
// position is baked into launch parameters, so replays of a captured CUDA graph draw fresh masks.
#include "common.cuh"
#include "philox.cuh"

namespace spg {

constexpr int kDropRows = 256;  // rows per partial of the backward column sums

struct DropParams {
    uint64_t seed, ctr;
    uint32_t thr;
    bool all;   // p >= 1: every element dropped
    float inv;  // 1 / (1 - p)
};

__device__ __forceinline__ DropParams drop_params(const int64_t* slot, float p) {
    DropParams d;
    d.seed = (uint64_t)slot[0];
    d.ctr = (uint64_t)slot[1];
    d.thr = dropout_threshold(p);
    d.all = !(p < 1.f);
    d.inv = d.all ? 0.f : 1.f / (1.f - p);
    return d;
}

__device__ __forceinline__ bool kept(const DropParams& d, uint32_t w) { return !d.all && w >= d.thr; }

__device__ __forceinline__ uint32_t word_of(const Philox4& w, int64_t i) {
    const int k = (int)(i & 3);
    return k == 0 ? w.v[0] : k == 1 ? w.v[1] : k == 2 ? w.v[2] : w.v[3];
}

// G * m / (1-p) for one element (a select, so that p = 1 or an infinite gradient gives 0, never NaN)
__device__ __forceinline__ float drop1(const DropParams& d, uint32_t w, float g) { return kept(d, w) ? g * d.inv : 0.f; }

__global__ void dropout_rng_next_kernel(int64_t* state, int64_t* slot, int64_t key_xor) {
    SPG_PDL_ENTRY();
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        slot[0] = state[0] ^ key_xor;
        slot[1] = state[1];
        state[1] = state[1] + 1;
    }
}

// out = dropout(relu?(Y*scale+shift)); vec: C % 4 == 0 and 16-byte aligned rows (one float4 = one group).
__global__ void __launch_bounds__(256)
dropout_fwd_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                   const float* __restrict__ shift, int relu, float p, const int64_t* __restrict__ slot,
                   float* __restrict__ out, int64_t ldo, int64_t M, int C, int vec) {
    SPG_PDL_ENTRY();
    const DropParams d = drop_params(slot, p);
    const int64_t n = M * C, groups = (n + 3) >> 2;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (int64_t)gridDim.x * blockDim.x) {
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)q);
        const int64_t i0 = q << 2;
        if (vec) {
            const int64_t m = i0 / C;
            const int c = (int)(i0 - m * C);
            const float4 y = __ldg(reinterpret_cast<const float4*>(Y + m * ldy + c));
            float v[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float sc = scale ? __ldg(scale + c + j) : 1.f, sh = shift ? __ldg(shift + c + j) : 0.f;
                float a = fmaf(v[j], sc, sh);
                if (relu) a = fmaxf(a, 0.f);
                v[j] = drop1(d, w.v[j], a);
            }
            *reinterpret_cast<float4*>(out + m * ldo + c) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            for (int j = 0; j < 4 && i0 + j < n; ++j) {
                const int64_t i = i0 + j, m = i / C;
                const int c = (int)(i - m * C);
                float a = fmaf(Y[m * ldy + c], scale ? scale[c] : 1.f, shift ? shift[c] : 0.f);
                if (relu) a = fmaxf(a, 0.f);
                out[m * ldo + c] = drop1(d, w.v[j], a);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
dropout_mask_kernel(const int64_t* __restrict__ slot, float p, int64_t M, int C, uint8_t* __restrict__ mask) {
    SPG_PDL_ENTRY();
    const DropParams d = drop_params(slot, p);
    const int64_t n = M * C, groups = (n + 3) >> 2;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (int64_t)gridDim.x * blockDim.x) {
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)q);
        for (int j = 0; j < 4 && (q << 2) + j < n; ++j) mask[(q << 2) + j] = kept(d, w.v[j]) ? 1 : 0;
    }
}

// Per-column loop state of the BatchNorm/ReLU backward (rstd from the batch variance).
struct BnCol {
    float sc, sh, mu, rs;
};
__device__ __forceinline__ BnCol bn_col(const float* scale, const float* shift, const float* mean, const float* var,
                                        float eps, int c) {
    BnCol b;
    b.sc = scale[c];
    b.sh = shift[c];
    b.mu = mean[c];
    b.rs = 1.f / sqrtf(var[c] + eps);
    return b;
}

// Pass 1 of the masked BatchNorm backward: per 256-row chunk, partial s1 = sum g, s2 = sum g*xhat with
// g = relu_mask * G*m/(1-p); ws[chunk][2][C].  VEC: a thread owns 4 columns (one Philox group) of a row,
// 32 threads x 8 row lanes cover 128 columns; scalar: 32 columns x 8 row lanes, one Philox call per element.
template <bool VEC>
__global__ void __launch_bounds__(256)
dropout_bwd_reduce_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y, int64_t ldy,
                          const float* __restrict__ scale, const float* __restrict__ shift,
                          const float* __restrict__ mean, const float* __restrict__ var, float eps, int relu,
                          float p, const int64_t* __restrict__ slot, float* __restrict__ ws, int64_t M, int C) {
    SPG_PDL_ENTRY();
    constexpr int W = VEC ? 4 : 1;
    __shared__ float s1[8][32 * W], s2[8][32 * W];
    const DropParams d = drop_params(slot, p);
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c0 = (blockIdx.x * 32 + x) * W;
    const int64_t r0 = (int64_t)blockIdx.y * kDropRows, r1 = min(M, r0 + kDropRows);
    float a1[W], a2[W];
#pragma unroll
    for (int j = 0; j < W; ++j) a1[j] = a2[j] = 0.f;
    if (c0 < C) {
        BnCol b[W];
#pragma unroll
        for (int j = 0; j < W; ++j) b[j] = bn_col(scale, shift, mean, var, eps, c0 + j);
        for (int64_t r = r0 + y; r < r1; r += 8) {
            float yv[W], g[W];
            const int64_t i0 = r * C + c0;
            const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)(i0 >> 2));
            if constexpr (VEC) {
                const float4 yq = __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c0));
                const float4 gq = __ldg(reinterpret_cast<const float4*>(G + r * ldg + c0));
                yv[0] = yq.x; yv[1] = yq.y; yv[2] = yq.z; yv[3] = yq.w;
                g[0] = gq.x; g[1] = gq.y; g[2] = gq.z; g[3] = gq.w;
            } else {
                yv[0] = __ldg(Y + r * ldy + c0);
                g[0] = __ldg(G + r * ldg + c0);
            }
#pragma unroll
            for (int j = 0; j < W; ++j) {
                float gj = drop1(d, VEC ? w.v[j] : word_of(w, i0), g[j]);
                if (relu && !(fmaf(yv[j], b[j].sc, b[j].sh) > 0.f)) gj = 0.f;
                a1[j] += gj;
                a2[j] = fmaf(gj, (yv[j] - b[j].mu) * b[j].rs, a2[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < W; ++j) {
        s1[y][x * W + j] = a1[j];
        s2[y][x * W + j] = a2[j];
    }
    __syncthreads();
    if (y == 0 && c0 < C) {
#pragma unroll
        for (int j = 0; j < W; ++j) {
            float t1 = 0.f, t2 = 0.f;
            for (int k = 0; k < 8; ++k) {
                t1 += s1[k][x * W + j];
                t2 += s2[k][x * W + j];
            }
            ws[((int64_t)blockIdx.y * 2) * C + c0 + j] = t1;
            ws[((int64_t)blockIdx.y * 2 + 1) * C + c0 + j] = t2;
        }
    }
}

// s12[k] = sum over chunks of ws[chunk][k], k < 2C: one warp per column, fp64 accumulation, fixed order.
__global__ void __launch_bounds__(128)
dropout_bwd_merge_kernel(const float* __restrict__ ws, int64_t chunks, int n, float* __restrict__ s12) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (k >= n) return;
    double a = 0.0;
    for (int64_t j = lane; j < chunks; j += 32) a += (double)__ldg(ws + j * n + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) s12[k] = (float)a;
}

// Pass 2: dY = scale*(g - s1/M - xhat*s2/M) (BN) or g (no BN), g = relu_mask * G*m/(1-p).  Y may be NULL
// when there is neither BatchNorm nor ReLU.  In place (dY == G) is allowed.
template <bool VEC>
__global__ void __launch_bounds__(256)
dropout_bwd_apply_kernel(const float* G, int64_t ldg, const float* __restrict__ Y, int64_t ldy,
                         const float* __restrict__ scale, const float* __restrict__ shift,
                         const float* __restrict__ mean, const float* __restrict__ var, float eps, int relu,
                         int has_bn, const float* __restrict__ s1, const float* __restrict__ s2, float p,
                         const int64_t* __restrict__ slot, float* dY, int64_t lddy, int64_t M, int C) {
    SPG_PDL_ENTRY();
    constexpr int W = VEC ? 4 : 1;
    const DropParams d = drop_params(slot, p);
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c0 = (blockIdx.x * 32 + x) * W;
    if (c0 >= C) return;
    float sc[W], sh[W], mu[W], rs[W], m1[W], m2[W];
#pragma unroll
    for (int j = 0; j < W; ++j) {
        const int c = c0 + j;
        sc[j] = scale ? scale[c] : 1.f;
        sh[j] = shift ? shift[c] : 0.f;
        mu[j] = has_bn ? mean[c] : 0.f;
        rs[j] = has_bn ? 1.f / sqrtf(var[c] + eps) : 1.f;
        m1[j] = has_bn ? s1[c] / (float)M : 0.f;
        m2[j] = has_bn ? s2[c] / (float)M : 0.f;
    }
    for (int64_t r = (int64_t)blockIdx.y * 8 + y; r < M; r += (int64_t)gridDim.y * 8) {
        const int64_t i0 = r * C + c0;
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)(i0 >> 2));
        float yv[W], g[W];
        if constexpr (VEC) {
            const float4 yq = Y ? __ldg(reinterpret_cast<const float4*>(Y + r * ldy + c0)) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 gq = *reinterpret_cast<const float4*>(G + r * ldg + c0);
            yv[0] = yq.x; yv[1] = yq.y; yv[2] = yq.z; yv[3] = yq.w;
            g[0] = gq.x; g[1] = gq.y; g[2] = gq.z; g[3] = gq.w;
        } else {
            yv[0] = Y ? Y[r * ldy + c0] : 0.f;
            g[0] = G[r * ldg + c0];
        }
        float o[W];
#pragma unroll
        for (int j = 0; j < W; ++j) {
            float gj = drop1(d, VEC ? w.v[j] : word_of(w, i0), g[j]);
            if (relu && !(fmaf(yv[j], sc[j], sh[j]) > 0.f)) gj = 0.f;
            o[j] = has_bn ? sc[j] * (gj - m1[j] - (yv[j] - mu[j]) * rs[j] * m2[j]) : gj;
        }
        if constexpr (VEC) {
            *reinterpret_cast<float4*>(dY + r * lddy + c0) = make_float4(o[0], o[1], o[2], o[3]);
        } else {
            dY[r * lddy + c0] = o[0];
        }
    }
}

static inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

static inline unsigned flat_grid(int64_t groups) {
    int64_t g = ceil_div64(groups, 256);
    if (g > 16 * kNumSMs) g = 16 * kNumSMs;
    return (unsigned)(g < 1 ? 1 : g);
}

static inline unsigned apply_rows_grid(int64_t M) {
    int64_t g = ceil_div64(M, 64);
    if (g > 8 * kNumSMs) g = 8 * kNumSMs;
    return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_dropout_rng_next(int64_t* state, int64_t* slot, int64_t key_xor, spg_stream_t stream) {
    if (!state || !slot) return SPG_E_BADARG;
    SPG_LAUNCH(K_DROPOUT_RNG_NEXT, (cudaStream_t)stream, dropout_rng_next_kernel, 1, 32, 0, state, slot, key_xor);
    return launch_status();
}

int spg_dropout_fwd(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu, float p,
                    const int64_t* slot, float* out, int64_t ldo, int64_t M, int C, spg_stream_t stream) {
    if (M < 0 || C <= 0 || !(p >= 0.f)) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!Y || !out || !slot || ldy < C || ldo < C) return SPG_E_BADARG;
    const int vec = (C % 4 == 0) && ldy % 4 == 0 && ldo % 4 == 0 && al16(Y) && al16(out);
    SPG_LAUNCH(K_DROPOUT_FWD, (cudaStream_t)stream, dropout_fwd_kernel, flat_grid(ceil_div64(M * C, 4)), 256, 0,
               Y, ldy, scale, shift, relu, p, slot, out, ldo, M, C, vec);
    return launch_status();
}

int spg_dropout_mask(const int64_t* slot, float p, int64_t M, int C, uint8_t* mask, spg_stream_t stream) {
    if (M < 0 || C <= 0 || !(p >= 0.f)) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!slot || !mask) return SPG_E_BADARG;
    SPG_LAUNCH(K_DROPOUT_MASK, (cudaStream_t)stream, dropout_mask_kernel, flat_grid(ceil_div64(M * C, 4)), 256, 0,
               slot, p, M, C, mask);
    return launch_status();
}

int spg_dropout_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy, const float* scale,
                           const float* shift, const float* mean, const float* var, float eps, int relu, float p,
                           const int64_t* slot, float* s12, float* workspace, int64_t M, int C,
                           spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !(p >= 0.f) || !G || !Y || !scale || !shift || !mean || !var || !slot || !s12 ||
        !workspace || ldg < C || ldy < C)
        return SPG_E_BADARG;
    const int64_t chunks = ceil_div64(M, kDropRows);
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const bool vec = C % 4 == 0 && ldg % 4 == 0 && ldy % 4 == 0 && al16(G) && al16(Y);
    if (vec) {
        dim3 grid((unsigned)ceil_div64(C, 128), (unsigned)chunks);
        SPG_LAUNCH(K_DROPOUT_BWD_REDUCE, s, dropout_bwd_reduce_kernel<true>, grid, 256, 0, G, ldg, Y, ldy, scale,
                   shift, mean, var, eps, relu, p, slot, workspace, M, C);
    } else {
        dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)chunks);
        SPG_LAUNCH(K_DROPOUT_BWD_REDUCE, s, dropout_bwd_reduce_kernel<false>, grid, 256, 0, G, ldg, Y, ldy, scale,
                   shift, mean, var, eps, relu, p, slot, workspace, M, C);
    }
    int rc = launch_status();
    if (rc) return rc;
    SPG_LAUNCH(K_DROPOUT_BWD_REDUCE_FINAL, s, dropout_bwd_merge_kernel, (unsigned)ceil_div64(2 * C, 4), 128, 0,
               workspace, chunks, 2 * C, s12);
    return launch_status();
}

int spg_dropout_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy, const float* scale,
                          const float* shift, const float* mean, const float* var, float eps, int relu, int has_bn,
                          const float* s1, const float* s2, float p, const int64_t* slot, float* dY, int64_t lddy,
                          int64_t M, int C, spg_stream_t stream) {
    if (M < 0 || C <= 0 || !(p >= 0.f)) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!G || !dY || !slot || ldg < C || lddy < C) return SPG_E_BADARG;
    if ((relu || has_bn) && (!Y || ldy < C)) return SPG_E_BADARG;
    if (has_bn && (!scale || !shift || !mean || !var || !s1 || !s2)) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const bool vec = C % 4 == 0 && ldg % 4 == 0 && lddy % 4 == 0 && al16(G) && al16(dY) &&
                     (!Y || (ldy % 4 == 0 && al16(Y)));
    if (vec) {
        dim3 grid((unsigned)ceil_div64(C, 128), apply_rows_grid(M));
        SPG_LAUNCH(K_DROPOUT_BWD_APPLY, s, dropout_bwd_apply_kernel<true>, grid, 256, 0, G, ldg, Y, ldy, scale,
                   shift, mean, var, eps, relu, has_bn, s1, s2, p, slot, dY, lddy, M, C);
    } else {
        dim3 grid((unsigned)ceil_div64(C, 32), apply_rows_grid(M));
        SPG_LAUNCH(K_DROPOUT_BWD_APPLY, s, dropout_bwd_apply_kernel<false>, grid, 256, 0, G, ldg, Y, ldy, scale,
                   shift, mean, var, eps, relu, has_bn, s1, s2, p, slot, dY, lddy, M, C);
    }
    return launch_status();
}

}  // extern "C"
