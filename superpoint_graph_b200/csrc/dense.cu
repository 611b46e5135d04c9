// Dense fp32 building blocks of the PointNet / filter-network / classifier layers:
// a tiled FMA GEMM with the producing layer's "BatchNorm apply + ReLU" fused into
// the operand load, deterministic batch statistics, and the BatchNorm/ReLU backward.
//
// Reference semantics: nn.Conv1d(kernel 1) / nn.Linear / nn.BatchNorm1d / nn.ReLU as
// stacked by learning/pointnet.py:27-53,83-118 and learning/graphnet.py:17-34.  The
// reference round-trips every [Nv*L, C] activation through memory three times per
// layer (conv, BN, ReLU); here only the raw pre-norm output of a layer is ever
// stored and the normalisation + activation happen while the next GEMM loads it.
//
// This file is the exact-fp32 engine (parity reference on device and the path for
// small / odd shapes).  The large point-wise layers are served by the wgmma
// 3xTF32 kernel in tc_gemm.cu when it applies.
#include "common.cuh"

namespace spg {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4;
constexpr int LDA_S = BM + 4, LDB_S = BN + 4;

struct GemmArgs {
    const float* A;
    int64_t lda;
    const float* B;
    int64_t ldb;
    const float* bias;
    float* C;
    int64_t ldc;
    int64_t M, N, K;
    const float *a_scale, *a_shift;
    int a_relu;
    const float *b_scale, *b_shift;
    int b_relu;
    int64_t k_chunk;
    int a_vec, b_vec, c_vec, split;
    float* stats;        // optional [row_tiles, N, 3] = (count, mean, M2) of C per 128-row tile
    int64_t stats_tile0;  // first row-tile index of this launch (tall problems are slabbed)
};

template <bool A_KMAJOR, bool B_KMAJOR>
__global__ void __launch_bounds__(256) gemm_kernel(const GemmArgs p) {
    SPG_PDL_ENTRY();
    __shared__ __align__(16) float As[BK * LDA_S];
    __shared__ __align__(16) float Bs[BK * LDB_S];
    const int t = threadIdx.x;
    const int tx = t & 15, ty = t >> 4;
    const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
    const int64_t kbeg = (int64_t)blockIdx.z * p.k_chunk;
    const int64_t kend = min(p.K, kbeg + p.k_chunk);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float ra[8], rb[4];

    auto load_a = [&](int64_t k0) {
        if (A_KMAJOR) {
            const int kq = t & 3;
            const int64_t kk = k0 + kq * 4;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int64_t row = m0 + (t >> 2) + 64 * i;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                if (row < p.M) {
                    const float* src = p.A + row * p.lda + kk;
                    if (p.a_vec && kk + 3 < kend) {
                        const float4 q = __ldg(reinterpret_cast<const float4*>(src));
                        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            if (kk + j < kend) v[j] = __ldg(src + j);
                    }
                    if (p.a_scale || p.a_shift || p.a_relu) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            if (kk + j < kend) {
                                const float sc = p.a_scale ? __ldg(p.a_scale + kk + j) : 1.f;
                                const float sh = p.a_shift ? __ldg(p.a_shift + kk + j) : 0.f;
                                float u = fmaf(v[j], sc, sh);
                                if (p.a_relu) u = fmaxf(u, 0.f);
                                v[j] = u;
                            }
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) ra[i * 4 + j] = v[j];
            }
        } else {
            const int m4 = t & 31;
            const int64_t m = m0 + m4 * 4;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int64_t k = k0 + (t >> 5) + 8 * i;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                if (k < kend) {
                    const float* src = p.A + k * p.lda + m;
                    if (p.a_vec && m + 3 < p.M) {
                        const float4 q = __ldg(reinterpret_cast<const float4*>(src));
                        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            if (m + j < p.M) v[j] = __ldg(src + j);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) ra[i * 4 + j] = v[j];
            }
        }
    };
    auto store_a = [&]() {
        if (A_KMAJOR) {
            const int kq = t & 3;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int rl = (t >> 2) + 64 * i;
#pragma unroll
                for (int j = 0; j < 4; ++j) As[(kq * 4 + j) * LDA_S + rl] = ra[i * 4 + j];
            }
        } else {
            const int m4 = t & 31;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int kl = (t >> 5) + 8 * i;
                *reinterpret_cast<float4*>(&As[kl * LDA_S + m4 * 4]) =
                    make_float4(ra[i * 4], ra[i * 4 + 1], ra[i * 4 + 2], ra[i * 4 + 3]);
            }
        }
    };
    auto load_b = [&](int64_t k0) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (B_KMAJOR) {
            const int kq = t & 3;
            const int64_t kk = k0 + kq * 4;
            const int64_t n = n0 + (t >> 2);
            if (n < p.N) {
                const float* src = p.B + n * p.ldb + kk;
                if (p.b_vec && kk + 3 < kend) {
                    const float4 q = __ldg(reinterpret_cast<const float4*>(src));
                    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (kk + j < kend) v[j] = __ldg(src + j);
                }
            }
        } else {
            const int n4 = t & 15;
            const int64_t n = n0 + n4 * 4;
            const int64_t k = k0 + (t >> 4);
            if (k < kend) {
                const float* src = p.B + k * p.ldb + n;
                if (p.b_vec && n + 3 < p.N) {
                    const float4 q = __ldg(reinterpret_cast<const float4*>(src));
                    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (n + j < p.N) v[j] = __ldg(src + j);
                }
                if (p.b_scale || p.b_shift || p.b_relu) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (n + j < p.N) {
                            const float sc = p.b_scale ? __ldg(p.b_scale + n + j) : 1.f;
                            const float sh = p.b_shift ? __ldg(p.b_shift + n + j) : 0.f;
                            float u = fmaf(v[j], sc, sh);
                            if (p.b_relu) u = fmaxf(u, 0.f);
                            v[j] = u;
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) rb[j] = v[j];
    };
    auto store_b = [&]() {
        if (B_KMAJOR) {
            const int kq = t & 3, nl = t >> 2;
#pragma unroll
            for (int j = 0; j < 4; ++j) Bs[(kq * 4 + j) * LDB_S + nl] = rb[j];
        } else {
            const int n4 = t & 15, kl = t >> 4;
            *reinterpret_cast<float4*>(&Bs[kl * LDB_S + n4 * 4]) =
                make_float4(rb[0], rb[1], rb[2], rb[3]);
        }
    };

    if (kbeg < kend) {
        load_a(kbeg);
        load_b(kbeg);
    }
    for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
        store_a();
        store_b();
        __syncthreads();
        if (k0 + BK < kend) {
            load_a(k0 + BK);
            load_b(k0 + BK);
        }
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk * LDA_S + ty * TM]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk * LDA_S + ty * TM + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk * LDB_S + tx * TN]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

    // epilogue
    float* Cout = p.C;
    int64_t ldc = p.ldc;
    if (p.split > 1) {
        Cout = p.C + (int64_t)blockIdx.z * p.M * p.N;  // C is the workspace here
        ldc = p.N;
    }
    const int64_t n = n0 + tx * TN;
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.bias && p.split == 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (n + j < p.N) bv[j] = __ldg(p.bias + n + j);
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t m = m0 + ty * TM + i;
        if (m >= p.M) continue;
        float* dst = Cout + m * ldc + n;
        if ((p.c_vec || p.split > 1) && n + 3 < p.N &&
            ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
            *reinterpret_cast<float4*>(dst) = make_float4(acc[i][0] + bv[0], acc[i][1] + bv[1],
                                                          acc[i][2] + bv[2], acc[i][3] + bv[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n + j < p.N) dst[j] = acc[i][j] + bv[j];
        }
    }
    // fused batch statistics of this 128-row tile: two passes over the registers (sum -> mean,
    // then sum of squared deviations), merged over tiles by colstats_merge (Chan, fp64).
    if (p.stats) {
        float* red = As;            // [16][64]
        float* mean_s = As + 1024;  // [64]
        __syncthreads();
        float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < TM; ++i)
            if (m0 + ty * TM + i < p.M)
#pragma unroll
                for (int j = 0; j < 4; ++j) cs[j] += acc[i][j] + bv[j];
#pragma unroll
        for (int j = 0; j < 4; ++j) red[ty * 64 + tx * 4 + j] = cs[j];
        __syncthreads();
        const float nvalid = (float)min((int64_t)BM, p.M - m0);
        if (t < 64) {
            float tot = 0.f;
#pragma unroll
            for (int r = 0; r < 16; ++r) tot += red[r * 64 + t];
            mean_s[t] = tot / nvalid;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) cs[j] = 0.f;
#pragma unroll
        for (int i = 0; i < TM; ++i)
            if (m0 + ty * TM + i < p.M)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float d = acc[i][j] + bv[j] - mean_s[tx * 4 + j];
                    cs[j] = fmaf(d, d, cs[j]);
                }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) red[ty * 64 + tx * 4 + j] = cs[j];
        __syncthreads();
        if (t < 64 && n0 + t < p.N) {
            float m2 = 0.f;
#pragma unroll
            for (int r = 0; r < 16; ++r) m2 += red[r * 64 + t];
            float* o = p.stats + ((p.stats_tile0 + blockIdx.y) * p.N + n0 + t) * 3;
            o[0] = nvalid;
            o[1] = mean_s[t];
            o[2] = m2;
        }
    }
}

// C[m,n] = sum_z ws[z,m,n] (+ bias[n]).  Block = 64 elements x 4 partial groups: every group sums a
// strided quarter of the partials with 8 independent loads in flight, a fixed-order shared-memory
// combine keeps the result deterministic.
__global__ void __launch_bounds__(256)
gemm_splitk_reduce_kernel(const float* __restrict__ ws, int split, int64_t M, int64_t N,
                          const float* __restrict__ bias, float* __restrict__ C, int64_t ldc) {
    SPG_PDL_ENTRY();
    __shared__ float part[4][64];
    const int x = threadIdx.x & 63, y = threadIdx.x >> 6;
    const int64_t i = (int64_t)blockIdx.x * 64 + x;
    const int64_t stride = M * N;
    float s = 0.f;
    if (i < stride) {
        int z = y;
        for (; z + 28 < split; z += 32) {
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = __ldg(ws + (int64_t)(z + 4 * u) * stride + i);
#pragma unroll
            for (int u = 0; u < 8; ++u) s += v[u];
        }
        for (; z < split; z += 4) s += __ldg(ws + (int64_t)z * stride + i);
    }
    part[y][x] = s;
    __syncthreads();
    if (y == 0 && i < stride) {
        float t = (part[0][x] + part[1][x]) + (part[2][x] + part[3][x]);
        const int64_t m = i / N, n = i % N;
        if (bias) t += bias[n];
        C[m * ldc + n] = t;
    }
}

// ---------------------------------------------------------------- column reductions
constexpr int kChunkRows = 1024;

// per (chunk, column): count, mean, M2 (Welford), merged over the 8 row lanes (Chan).
__global__ void __launch_bounds__(256)
colstats_partial_kernel(const float* __restrict__ Y, int64_t ldy, int64_t M, int C,
                        float* __restrict__ ws) {
    SPG_PDL_ENTRY();
    __shared__ float s_n[8][32], s_mean[8][32], s_m2[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t r0 = (int64_t)blockIdx.y * kChunkRows;
    const int64_t r1 = min(M, r0 + kChunkRows);
    float n = 0.f, mean = 0.f, m2 = 0.f;
    if (c < C) {
        for (int64_t r = r0 + y; r < r1; r += 8) {
            const float v = __ldg(Y + r * ldy + c);
            n += 1.f;
            const float d = v - mean;
            mean += d / n;
            m2 = fmaf(d, v - mean, m2);
        }
    }
    s_n[y][x] = n;
    s_mean[y][x] = mean;
    s_m2[y][x] = m2;
    __syncthreads();
    if (y == 0 && c < C) {
        float na = s_n[0][x], ma = s_mean[0][x], qa = s_m2[0][x];
        for (int j = 1; j < 8; ++j) {
            const float nb = s_n[j][x], mb = s_mean[j][x], qb = s_m2[j][x];
            if (nb > 0.f) {
                const float nn = na + nb, d = mb - ma;
                ma += d * (nb / nn);
                qa += qb + d * d * (na * nb / nn);
                na = nn;
            }
        }
        float* o = ws + ((int64_t)blockIdx.y * C + c) * 3;
        o[0] = na;
        o[1] = ma;
        o[2] = qa;
    }
}

// Merge of (count, mean, M2) partials, deterministic and division-free in the inner loops:
//   N = sum n_k, mean = sum n_k*mean_k / N, M2 = sum (M2_k + n_k*(mean_k - mean)^2)    (fp64 sums).
// Block = 32 columns x 32 lanes, 256 partials per block (8 per thread, kept in registers between
// the two passes); grid.y > 1 writes block-level partials (same triple format) for a second level.
constexpr int kMergePerBlock = 256;

// optional BatchNorm fold executed by the last merge level (saves a launch per layer)
struct FoldArgs {
    const float *gamma, *beta;
    float *scale, *shift, *rmean, *rvar;
    long long* nbt;
    float eps, momentum, unbias;
    int enabled;
};

__global__ void __launch_bounds__(1024)
colstats_final_kernel(const float* __restrict__ ws, int64_t chunks, int C,
                      float* __restrict__ mean, float* __restrict__ var,
                      float* __restrict__ out_partials, const FoldArgs f) {
    SPG_PDL_ENTRY();
    __shared__ double s_a[32][33], s_b[32][33];
    __shared__ double s_mean[32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t k0 = (int64_t)blockIdx.y * kMergePerBlock;
    float pn[8], pm[8], pq[8];
    double sn = 0.0, snm = 0.0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const int64_t k = k0 + y + 32 * u;
        pn[u] = 0.f;
        pm[u] = 0.f;
        pq[u] = 0.f;
        if (c < C && k < chunks) {
            const float* o = ws + (k * C + c) * 3;
            pn[u] = o[0];
            pm[u] = o[1];
            pq[u] = o[2];
        }
        sn += (double)pn[u];
        snm += (double)pn[u] * (double)pm[u];
    }
    s_a[y][x] = sn;
    s_b[y][x] = snm;
    __syncthreads();
    if (y == 0) {
        double a = 0.0, b = 0.0;
        for (int j = 0; j < 32; ++j) {
            a += s_a[j][x];
            b += s_b[j][x];
        }
        s_a[0][x] = a;
        s_mean[x] = a > 0.0 ? b / a : 0.0;
    }
    __syncthreads();
    const double ntot = s_a[0][x], mu = s_mean[x];
    double q = 0.0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const double d = (double)pm[u] - mu;
        q += (double)pq[u] + (double)pn[u] * d * d;
    }
    __syncthreads();
    s_b[y][x] = q;
    __syncthreads();
    if (y == 0 && c < C) {
        double qq = 0.0;
        for (int j = 0; j < 32; ++j) qq += s_b[j][x];
        if (out_partials) {
            float* o = out_partials + ((int64_t)blockIdx.y * C + c) * 3;
            o[0] = (float)ntot;
            o[1] = (float)mu;
            o[2] = (float)qq;
        } else {
            const float mu_f = (float)mu;
            const float var_f = ntot > 0.0 ? (float)(qq / ntot) : 0.f;
            mean[c] = mu_f;
            var[c] = var_f;
            if (f.enabled) {
                const float rstd = 1.f / sqrtf(var_f + f.eps);
                const float sc = (f.gamma ? f.gamma[c] : 1.f) * rstd;
                f.scale[c] = sc;
                f.shift[c] = (f.beta ? f.beta[c] : 0.f) - mu_f * sc;
                if (f.rmean) f.rmean[c] = (1.f - f.momentum) * f.rmean[c] + f.momentum * mu_f;
                if (f.rvar) f.rvar[c] = (1.f - f.momentum) * f.rvar[c] + f.momentum * var_f * f.unbias;
                if (c == 0 && f.nbt) f.nbt[0] += 1;
            }
        }
    }
}

// two-level driver; `partials` must have room for ceil(n/256) extra triples per column at its end
static int colstats_merge_launch(float* partials, int64_t n, int C, float* mean, float* var,
                                 cudaStream_t s, const FoldArgs& fold) {
    FoldArgs nofold;
    nofold.enabled = 0;
    nofold.gamma = nofold.beta = nullptr;
    nofold.scale = nofold.shift = nofold.rmean = nofold.rvar = nullptr;
    nofold.nbt = nullptr;
    nofold.eps = nofold.momentum = nofold.unbias = 0.f;
    const unsigned gx = (unsigned)ceil_div64(C, 32);
    const int64_t P = ceil_div64(n, kMergePerBlock);
    if (P > 65535) return SPG_E_UNSUPPORTED;
    if (P == 1) {
        SPG_LAUNCH(K_COLSTATS_FINAL, s, colstats_final_kernel, dim3(gx, 1), 1024, 0, partials, n, C,
                   mean, var, (float*)nullptr, fold);
        return launch_status();
    }
    float* lvl2 = partials + n * C * 3;
    SPG_LAUNCH(K_COLSTATS_FINAL, s, colstats_final_kernel, dim3(gx, (unsigned)P), 1024, 0, partials, n,
               C, mean, var, lvl2, nofold);
    int rc = launch_status();
    if (rc) return rc;
    if (P > kMergePerBlock) return SPG_E_UNSUPPORTED;
    SPG_LAUNCH(K_COLSTATS_FINAL, s, colstats_final_kernel, dim3(gx, 1), 1024, 0, lvl2, P, C, mean, var,
               (float*)nullptr, fold);
    return launch_status();
}

static FoldArgs no_fold() {
    FoldArgs f;
    f.enabled = 0;
    f.gamma = f.beta = nullptr;
    f.scale = f.shift = f.rmean = f.rvar = nullptr;
    f.nbt = nullptr;
    f.eps = f.momentum = f.unbias = 0.f;
    return f;
}

__global__ void bn_fold_kernel(const float* __restrict__ mean, const float* __restrict__ var,
                               const float* __restrict__ gamma, const float* __restrict__ beta,
                               float eps, float* __restrict__ scale, float* __restrict__ shift,
                               float* __restrict__ rmean, float* __restrict__ rvar,
                               long long* __restrict__ nbt, float momentum, float unbias, int C) {
    SPG_PDL_ENTRY();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c == 0 && nbt) nbt[0] += 1;
    if (c >= C) return;
    const float mu = mean[c], v = var[c];
    const float rstd = 1.f / sqrtf(v + eps);
    const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    const float sc = g * rstd;
    scale[c] = sc;
    shift[c] = b - mu * sc;
    if (rmean) rmean[c] = (1.f - momentum) * rmean[c] + momentum * mu;
    if (rvar) rvar[c] = (1.f - momentum) * rvar[c] + momentum * v * unbias;
}

__global__ void __launch_bounds__(256)
affine_act_kernel(const float* __restrict__ Y, int64_t ldy, const float* __restrict__ scale,
                  const float* __restrict__ shift, int relu, float* __restrict__ out, int64_t ldo,
                  int64_t M, int C) {
    SPG_PDL_ENTRY();
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    if (c >= C) return;
    const float sc = scale ? scale[c] : 1.f, sh = shift ? shift[c] : 0.f;
    for (int64_t r = (int64_t)blockIdx.y * 8 + y; r < M; r += (int64_t)gridDim.y * 8) {
        float v = fmaf(Y[r * ldy + c], sc, sh);
        if (relu) v = fmaxf(v, 0.f);
        out[r * ldo + c] = v;
    }
}

__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ X, int64_t ldx, int64_t M, int C,
                      float* __restrict__ ws) {
    SPG_PDL_ENTRY();
    __shared__ float s[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t r0 = (int64_t)blockIdx.y * kChunkRows;
    const int64_t r1 = min(M, r0 + kChunkRows);
    float a = 0.f;
    if (c < C)
        for (int64_t r = r0 + y; r < r1; r += 8) a += __ldg(X + r * ldx + c);
    s[y][x] = a;
    __syncthreads();
    if (y == 0 && c < C) {
        float t = 0.f;
        for (int j = 0; j < 8; ++j) t += s[j][x];
        ws[(int64_t)blockIdx.y * C + c] = t;
    }
}

// out[c] = sum over chunks of ws[k*stride + c*inner + off] accumulated in double.
__global__ void colsum_final_kernel(const float* __restrict__ ws, int64_t chunks, int C,
                                    float* __restrict__ out) {
    SPG_PDL_ENTRY();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double a = 0.0;
    for (int64_t k = 0; k < chunks; ++k) a += (double)ws[k * C + c];
    out[c] = (float)a;
}

__global__ void __launch_bounds__(256)
act_bwd_reduce_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                      int64_t ldy, const float* __restrict__ scale,
                      const float* __restrict__ shift, const float* __restrict__ mean,
                      const float* __restrict__ var, float eps, int relu, float* __restrict__ ws,
                      int64_t M, int C) {
    SPG_PDL_ENTRY();
    __shared__ float s1[8][32], s2[8][32];
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    const int64_t r0 = (int64_t)blockIdx.y * kChunkRows;
    const int64_t r1 = min(M, r0 + kChunkRows);
    float a1 = 0.f, a2 = 0.f;
    if (c < C) {
        const float sc = scale[c], sh = shift[c], mu = mean[c];
        const float rstd = 1.f / sqrtf(var[c] + eps);
        for (int64_t r = r0 + y; r < r1; r += 8) {
            const float yv = __ldg(Y + r * ldy + c);
            float g = __ldg(G + r * ldg + c);
            if (relu && !(fmaf(yv, sc, sh) > 0.f)) g = 0.f;
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

__global__ void act_bwd_reduce_final_kernel(const float* __restrict__ ws, int64_t chunks, int C,
                                            float* __restrict__ s1, float* __restrict__ s2) {
    SPG_PDL_ENTRY();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double a1 = 0.0, a2 = 0.0;
    for (int64_t k = 0; k < chunks; ++k) {
        a1 += (double)ws[(k * 2) * C + c];
        a2 += (double)ws[(k * 2 + 1) * C + c];
    }
    s1[c] = (float)a1;
    s2[c] = (float)a2;
}

__global__ void __launch_bounds__(256)
act_bwd_apply_kernel(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Y,
                     int64_t ldy, const float* __restrict__ scale, const float* __restrict__ shift,
                     const float* __restrict__ mean, const float* __restrict__ var, float eps,
                     int relu, int has_bn, const float* __restrict__ s1,
                     const float* __restrict__ s2, float* __restrict__ dY, int64_t lddy, int64_t M,
                     int C) {
    SPG_PDL_ENTRY();
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + x;
    if (c >= C) return;
    const float sc = (has_bn || scale) ? (scale ? scale[c] : 1.f) : 1.f;
    const float sh = shift ? shift[c] : 0.f;
    float mu = 0.f, rstd = 1.f, m1 = 0.f, m2 = 0.f;
    if (has_bn) {
        mu = mean[c];
        rstd = 1.f / sqrtf(var[c] + eps);
        m1 = s1[c] / (float)M;
        m2 = s2[c] / (float)M;
    }
    for (int64_t r = (int64_t)blockIdx.y * 8 + y; r < M; r += (int64_t)gridDim.y * 8) {
        const float yv = Y ? Y[r * ldy + c] : 0.f;
        float g = G[r * ldg + c];
        if (relu && !(fmaf(yv, sc, sh) > 0.f)) g = 0.f;
        float d = g;
        if (has_bn) d = sc * (g - m1 - (yv - mu) * rstd * m2);
        dY[r * lddy + c] = d;
    }
}

static inline bool a16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace spg

using namespace spg;

extern "C" {

int spg_gemm(const float* A, int64_t lda, int a_kmajor, const float* B, int64_t ldb, int b_kmajor,
             const float* bias, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
             const float* a_scale, const float* a_shift, int a_relu, const float* b_scale,
             const float* b_shift, int b_relu, int split_k, float* workspace, float* stats_ws,
             spg_stream_t stream) {
    if (M < 0 || N < 0 || K < 0) return SPG_E_BADARG;
    if (stats_ws && split_k > 1) return SPG_E_UNSUPPORTED;
    if (M == 0 || N == 0) return SPG_OK;
    if (!A || !B || !C) return SPG_E_BADARG;
    if ((a_scale || a_shift || a_relu) && !a_kmajor) return SPG_E_UNSUPPORTED;
    if ((b_scale || b_shift || b_relu) && b_kmajor) return SPG_E_UNSUPPORTED;
    if (split_k < 1) split_k = 1;
    if (split_k > 1 && !workspace) return SPG_E_BADARG;
    if (lda < (a_kmajor ? K : M) || ldb < (b_kmajor ? K : N) || ldc < N) return SPG_E_BADARG;
    GemmArgs p;
    p.A = A; p.lda = lda; p.B = B; p.ldb = ldb; p.bias = bias;
    p.C = split_k > 1 ? workspace : C;
    p.ldc = ldc; p.M = M; p.N = N; p.K = K;
    p.a_scale = a_scale; p.a_shift = a_shift; p.a_relu = a_relu;
    p.b_scale = b_scale; p.b_shift = b_shift; p.b_relu = b_relu;
    int64_t kc = ceil_div64(K > 0 ? K : 1, split_k);
    kc = ceil_div64(kc, BK) * BK;
    p.k_chunk = kc;
    p.split = split_k;
    p.a_vec = a16(A) && (lda % 4 == 0);
    p.b_vec = a16(B) && (ldb % 4 == 0);
    p.c_vec = a16(C) && (ldc % 4 == 0);
    p.stats = stats_ws;
    p.stats_tile0 = 0;
    const int64_t gy = ceil_div64(M, BM), gx = ceil_div64(N, BN);
    if (gy > 65535 * 32ll) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    // blockIdx.y is limited to 65535: fold very tall problems by looping over row slabs.
    const int64_t max_gy = 65535;
    for (int64_t y0 = 0; y0 < gy; y0 += max_gy) {
        GemmArgs q = p;
        const int64_t rows0 = y0 * BM;
        const int64_t gyi = min(max_gy, gy - y0);
        q.M = min(M - rows0, gyi * BM);
        q.stats_tile0 = y0;
        if (a_kmajor) q.A = A + rows0 * lda; else q.A = A + rows0;
        if (split_k > 1) {
            if (gy > max_gy) return SPG_E_UNSUPPORTED;
        } else {
            q.C = C + rows0 * ldc;
        }
        dim3 grid((unsigned)gx, (unsigned)gyi, (unsigned)split_k);
        if (a_kmajor && b_kmajor) {
            SPG_LAUNCH(K_GEMM, s, (gemm_kernel<true, true>), grid, 256, 0, q);
        } else if (a_kmajor && !b_kmajor) {
            SPG_LAUNCH(K_GEMM, s, (gemm_kernel<true, false>), grid, 256, 0, q);
        } else if (!a_kmajor && b_kmajor) {
            SPG_LAUNCH(K_GEMM, s, (gemm_kernel<false, true>), grid, 256, 0, q);
        } else {
            SPG_LAUNCH(K_GEMM, s, (gemm_kernel<false, false>), grid, 256, 0, q);
        }
        int rc = launch_status();
        if (rc) return rc;
    }
    if (split_k > 1) {
        const int64_t blocks = ceil_div64(M * N, 64);
        SPG_LAUNCH(K_GEMM_SPLITK_REDUCE, s, gemm_splitk_reduce_kernel, (unsigned)blocks, 256, 0,
                   workspace, split_k, M, N, bias, C, ldc);
        return launch_status();
    }
    return SPG_OK;
}

// workspace bound for the column reductions (the vectorised kernels use 256-row chunks)
int spg_splitk_reduce(const float* partials, int split, int64_t M, int64_t N, const float* bias,
                      float* C, int64_t ldc, spg_stream_t stream) {
    if (!partials || !C || split < 1 || M <= 0 || N <= 0 || ldc < N) return SPG_E_BADARG;
    const int64_t blocks = ceil_div64(M * N, 64);
    SPG_LAUNCH(K_GEMM_SPLITK_REDUCE, (cudaStream_t)stream, gemm_splitk_reduce_kernel,
               (unsigned)blocks, 256, 0, partials, split, M, N, bias, C, ldc);
    return launch_status();
}

int64_t spg_colstats_chunks(int64_t M) { return M <= 0 ? 1 : ceil_div64(M, 256); }
static inline int64_t scalar_chunks(int64_t M) { return M <= 0 ? 1 : ceil_div64(M, kChunkRows); }

int spg_colstats(const float* Y, int64_t ldy, int64_t M, int C, float* mean, float* var,
                 float* workspace, spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !Y || !mean || !var || !workspace || ldy < C) return SPG_E_BADARG;
    const int64_t chunks = scalar_chunks(M);
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)chunks);
    SPG_LAUNCH(K_COLSTATS_PARTIAL, s, colstats_partial_kernel, grid, 256, 0, Y, ldy, M, C,
               workspace);
    int rc = launch_status();
    if (rc) return rc;
    return colstats_merge_launch(workspace, chunks, C, mean, var, s, no_fold());
}

int64_t spg_gemm_stats_tiles(int64_t M) { return M <= 0 ? 1 : ceil_div64(M, BM); }

int spg_colstats_merge(float* partials, int64_t n_partials, int C, float* mean, float* var,
                       spg_stream_t stream) {
    if (n_partials <= 0 || C <= 0 || !partials || !mean || !var) return SPG_E_BADARG;
    return colstats_merge_launch(partials, n_partials, C, mean, var, (cudaStream_t)stream, no_fold());
}

int spg_colstats_merge_fold(float* partials, int64_t n_partials, int C, float* mean, float* var,
                            const float* gamma, const float* beta, float eps, float* scale,
                            float* shift, float* running_mean, float* running_var,
                            int64_t* num_batches_tracked, float momentum, int64_t M,
                            spg_stream_t stream) {
    if (n_partials <= 0 || C <= 0 || !partials || !mean || !var || !scale || !shift) return SPG_E_BADARG;
    FoldArgs f;
    f.enabled = 1;
    f.gamma = gamma; f.beta = beta; f.scale = scale; f.shift = shift;
    f.rmean = running_mean; f.rvar = running_var; f.nbt = (long long*)num_batches_tracked;
    f.eps = eps; f.momentum = momentum;
    f.unbias = M > 1 ? (float)((double)M / (double)(M - 1)) : 1.f;
    return colstats_merge_launch(partials, n_partials, C, mean, var, (cudaStream_t)stream, f);
}

int spg_bn_fold(const float* mean, const float* var, const float* gamma, const float* beta,
                float eps, float* scale, float* shift, float* running_mean, float* running_var,
                int64_t* num_batches_tracked, float momentum, int64_t M, int C,
                spg_stream_t stream) {
    if (C <= 0 || !mean || !var || !scale || !shift) return SPG_E_BADARG;
    const float unbias = M > 1 ? (float)((double)M / (double)(M - 1)) : 1.f;
    SPG_LAUNCH(K_BN_FOLD, (cudaStream_t)stream, bn_fold_kernel, (unsigned)ceil_div64(C, 128), 128,
               0, mean, var, gamma, beta, eps, scale, shift, running_mean, running_var,
               (long long*)num_batches_tracked, momentum, unbias, C);
    return launch_status();
}

static inline unsigned rows_grid(int64_t M) {
    int64_t g = ceil_div64(M, 64);
    if (g > 8 * kNumSMs) g = 8 * kNumSMs;
    if (g < 1) g = 1;
    return (unsigned)g;
}

int spg_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* out, int64_t ldo, int64_t M, int C, spg_stream_t stream) {
    if (M < 0 || C <= 0) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!Y || !out || ldy < C || ldo < C) return SPG_E_BADARG;
    {
        int rc = 0;
        if (vec_affine_act(Y, ldy, scale, shift, relu, out, ldo, M, C, (cudaStream_t)stream, &rc))
            return rc;
    }
    dim3 grid((unsigned)ceil_div64(C, 32), rows_grid(M));
    SPG_LAUNCH(K_AFFINE_ACT, (cudaStream_t)stream, affine_act_kernel, grid, 256, 0, Y, ldy, scale,
               shift, relu, out, ldo, M, C);
    return launch_status();
}

int spg_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* workspace,
               spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !X || !out || !workspace || ldx < C) return SPG_E_BADARG;
    {
        int rc = 0;
        if (vec_colsum(X, ldx, M, C, out, workspace, (cudaStream_t)stream, &rc)) return rc;
    }
    const int64_t chunks = scalar_chunks(M);
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)chunks);
    SPG_LAUNCH(K_COLSUM_PARTIAL, s, colsum_partial_kernel, grid, 256, 0, X, ldx, M, C, workspace);
    int rc = launch_status();
    if (rc) return rc;
    SPG_LAUNCH(K_COLSUM_FINAL, s, colsum_final_kernel, (unsigned)ceil_div64(C, 128), 128, 0,
               workspace, chunks, C, out);
    return launch_status();
}

int spg_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, float* s1, float* s2,
                       float* workspace, int64_t M, int C, spg_stream_t stream) {
    if (M <= 0 || C <= 0 || !G || !Y || !scale || !shift || !mean || !var || !s1 || !s2 ||
        !workspace)
        return SPG_E_BADARG;
    if (s2 == s1 + C) {
        int rc = 0;
        if (vec_act_bwd_reduce(G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, s1, s2,
                               workspace, M, C, (cudaStream_t)stream, &rc))
            return rc;
    }
    const int64_t chunks = scalar_chunks(M);
    if (chunks > 65535) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div64(C, 32), (unsigned)chunks);
    SPG_LAUNCH(K_ACT_BWD_REDUCE, s, act_bwd_reduce_kernel, grid, 256, 0, G, ldg, Y, ldy, scale,
               shift, mean, var, eps, relu, workspace, M, C);
    int rc = launch_status();
    if (rc) return rc;
    SPG_LAUNCH(K_ACT_BWD_REDUCE_FINAL, s, act_bwd_reduce_final_kernel,
               (unsigned)ceil_div64(C, 128), 128, 0, workspace, chunks, C, s1, s2);
    return launch_status();
}

int spg_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                      const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, int has_bn, const float* s1,
                      const float* s2, float* dY, int64_t lddy, int64_t M, int C,
                      spg_stream_t stream) {
    if (M < 0 || C <= 0) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!G || !dY) return SPG_E_BADARG;
    if ((relu || has_bn) && !Y) return SPG_E_BADARG;
    if (has_bn && (!scale || !shift || !mean || !var || !s1 || !s2)) return SPG_E_BADARG;
    {
        int rc = 0;
        if (vec_act_bwd_apply(G, ldg, Y, ldy, scale, shift, mean, var, eps, relu, has_bn, s1, s2,
                              dY, lddy, M, C, (cudaStream_t)stream, &rc))
            return rc;
    }
    dim3 grid((unsigned)ceil_div64(C, 32), rows_grid(M));
    SPG_LAUNCH(K_ACT_BWD_APPLY, (cudaStream_t)stream, act_bwd_apply_kernel, grid, 256, 0, G, ldg, Y,
               ldy, scale, shift, mean, var, eps, relu, has_bn, s1, s2, dY, lddy, M, C);
    return launch_status();
}

}  // extern "C"
