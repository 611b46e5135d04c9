// Hopper (wgmma) 3xTF32 GEMM for the point-wise layers: persistent, warp-specialised, weights resident
// in SMEM (loaded by TMA), with the BatchNorm bookkeeping of the training step fused on both sides.
//
//     C[M,N] = f(A)[M,K] * B[N,K]^T + bias
//
// in fp32-equivalent precision through error-compensated 3xTF32 splitting
// (x = hi + lo with hi = tf32(x), lo = tf32(x - hi);  A*B ~= Ahi*Bhi + Alo*Bhi + Ahi*Blo, all three
// accumulated in the same fp32 register accumulator; single-pass TF32 cannot hold the 1e-4 parity bound
// through five layers + BatchNorm, 3xTF32 is at ~1e-6).
//
// A CTA (one per SM) owns an N-slice of NS <= 128 output channels whose pre-split weight image
// (hi+lo, <= 128 KB) is brought into shared memory ONCE by cp.async.bulk.tensor (TMA, one 2-D box
// per (K-chunk, hi|lo) block of the image, completion on an mbarrier), and then walks over 128-row tiles:
//
//   warps 0-7   consumers: two warpgroups, each issues wgmma.mma_async m64 x NS x k8 over its 64 rows of
//               the tile (12 per K chunk), then runs the epilogue straight from the register accumulator:
//               +bias -> C, plus ONE of the fused column reductions
//                 STATS : batch statistics of C (pivoted sums kept per warp across tiles)
//                 BNRED : BatchNorm-backward sums of the layer BELOW (C is its dL/d(act)):
//                         s1 = sum gz, s2 = sum gz*xhat with gz = relu'(y2) * C
//               The two warpgroups take turns (ping-pong, two named barriers): warpgroup 1 issues a tile's
//               MMAs once warpgroup 0 has issued its own for that tile, warpgroup 0 those of the next tile
//               once warpgroup 1 is done, so each one's epilogue runs under the other's MMAs.
//   warps 8-15  producers: coalesced 128-bit loads of A (next chunks prefetched in registers), fused
//               prologue, tf32 hi/lo split, SWIZZLE_128B K-major tiles.  Producer warpgroup p fills
//               the 64-row half p of every tile into its own 2..4-stage ring, read by consumer warpgroup
//               p alone: a warpgroup in its epilogue holds back none of the other one's stages.
//                 AFFINE : f = relu(a*scale + shift)          (forward: BN apply + ReLU)
//                 BNBWD  : f = scale*(gz - s1/M - xhat*s2/M)  (backward: A = dL/d(act),
//                          A2 = raw output y of the layer; optional side store of f)
//
// The column reductions leave ONE partial per CTA and column (pivoted sums are carried across the
// CTA's tiles); a companion kernel (tc_merge_kernel, same C-ABI call) folds the <= kNumSMs partials per
// column in a fixed order (deterministic) into mean/var/scale/shift/running statistics or s1/s2.
//
// Reference semantics: nn.Conv1d(k=1)+BatchNorm1d+ReLU stacks of learning/pointnet.py:27-37,83-96
// and their autograd backward.
#include <cuda.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "tc_common.cuh"

namespace spg {

constexpr int T2_BM = 128;
constexpr int T2_KC = 32;
constexpr int T2_MAX_STAGES = 4;  // the A ring gets as many stages as fit next to the resident weights
constexpr int T2_EPI_WARPS = 8, T2_PROD_WARPS = 8;  // consumers: two warpgroups of 64 rows each
constexpr int T2_THREADS = (T2_EPI_WARPS + T2_PROD_WARPS) * 32;  // 512
constexpr int T2_A_BYTES = T2_BM * T2_KC * 4;                    // 16 KB (hi or lo)
constexpr int T2_STAGE_BYTES = 2 * T2_A_BYTES;                   // one stage of both rings
constexpr int T2_HALF_A_BYTES = T2_A_BYTES / 2;                  // 64 rows: one warpgroup's hi or lo
constexpr int T2_HALF_STAGE_BYTES = 2 * T2_HALF_A_BYTES;         // one stage of one warpgroup's ring

enum { PRO_AFFINE = 0, PRO_BNBWD = 1 };
enum { EPI_NONE = 0, EPI_STATS = 1, EPI_BNRED = 2 };

struct Tc2Args {
    const float* A;
    int64_t lda;
    const float* A2;  // PRO_BNBWD: raw output Y of the layer (same [M,K] coordinates as A)
    int64_t lda2;
    const float* bias;
    float* C;
    int64_t ldc;
    int64_t M;
    int N, K;
    const float *a_scale, *a_shift;  // AFFINE: prologue; BNBWD: scale/shift of this layer's BatchNorm
    int a_relu;
    const float *a_mean, *a_var, *a_s12;  // BNBWD: batch mean/var [K], s1|s2 [2K]
    float a_eps;
    float* dy_out;  // BNBWD: optional side store of f(A) (slice 0 only), ld = lddy
    int64_t lddy;
    int epi;        // EPI_*
    float* part;    // per-CTA partials [gridDim.x][N][3 | 2]
    // EPI_STATS outputs (+ optional fold)
    float *mean_out, *var_out;
    FoldArgs fold;
    // EPI_BNRED inputs (layer below) and output
    const float* e_y;
    int64_t e_ldy;
    const float *e_scale, *e_shift, *e_mean, *e_var;
    float e_eps;
    int e_relu;
    float* e_s12;  // [2N]
    int nstages;   // A-ring depth (2..4)
};

// Named barriers 1 and 2 order the consumer warpgroups' MMA phases (0 is __syncthreads)
constexpr int T2_TURN_BAR = 1;
constexpr int T2_TURN_THREADS = 2 * 128;
__device__ __forceinline__ void turn_wait(int id) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(T2_TURN_THREADS) : "memory");
}
__device__ __forceinline__ void turn_pass(int id) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(T2_TURN_THREADS) : "memory");
}

// Predicated global stores that the compiler may not take for writes to shared memory (C and the dY side
// store: nothing in the kernel reads them back, so column sums in shared memory need no reload after them)
__device__ __forceinline__ void st_global2(float* ptr, float2 v, bool pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}" ::"l"(ptr),
        "f"(v.x), "f"(v.y), "r"((int)pred));
}
__device__ __forceinline__ void st_global4(float* ptr, float4 v, bool pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p st.global.v4.f32 [%0], {%1, %2, %3, %4};\n\t}" ::"l"(ptr),
        "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"((int)pred));
}

// Column sums of a block of 4 columns over the 8 lanes that hold them (the lanes with the same lane % 4; lane
// r = lane / 4 holds rows r and r + 8): v[2k], v[2k + 1] are this lane's two partial sums of block column k.
// Reduce-scatter in three halving steps over lane distance 4, 8 and 16.  Every sum is formed from the same
// pairs, in the same order, as a butterfly (x += shfl_xor(x, 4), 8, 16) on each value forms it, so it is
// bitwise what that butterfly leaves in every lane.  Lane r gets sum v[4(r & 1) + 2((r >> 1) & 1) + (r >> 2)].
__device__ __forceinline__ float reduce_scatter8(const float (&v)[8], int r) {
    const bool b0 = r & 1, b1 = r & 2, b2 = r & 4;
    float w[4], x[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float keep = b0 ? v[i + 4] : v[i], send = b0 ? v[i] : v[i + 4];
        w[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float keep = b1 ? w[i + 2] : w[i], send = b1 ? w[i] : w[i + 2];
        x[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    const float keep = b2 ? x[1] : x[0], send = b2 ? x[0] : x[1];
    return keep + __shfl_xor_sync(0xffffffffu, send, 16);
}

// 2-D TMA load global -> shared, completion counted on an mbarrier (coordinates: {x = innermost, y})
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(map), "r"(x), "r"(y), "r"(bar)
        : "memory");
}

template <int NS, int PRO>
__global__ void __launch_bounds__(T2_THREADS, 1)
tc_gemm2_kernel(const Tc2Args p, const __grid_constant__ CUtensorMap wmap) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // the dynamic segment starts 1024-byte aligned (declared alignment; static data is padded up to
    // it): SWIZZLE_128B atoms need that, and no spare bytes are reserved for a manual round-up
    uint8_t* smem = smem_raw;
    if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();
    __shared__ __align__(8) uint64_t bars[4 * T2_MAX_STAGES + 1];

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const int nk = p.K / T2_KC;
    const int n0 = blockIdx.y * NS;  // first output channel of this CTA's slice
    const int64_t tiles = (p.M + T2_BM - 1) / T2_BM;
    const int nst = p.nstages;
    // two A rings, one per 64-row half of the tile: ring h = nst stages of [hi|lo][64 rows][128 B]
    auto ring = [&](int h) { return smem_u32(smem) + (uint32_t)(h * nst) * T2_HALF_STAGE_BYTES; };
    uint8_t* wres = smem + (size_t)nst * T2_STAGE_BYTES;  // resident weights: [nk][hi|lo][NS][128 B]

    const uint32_t bars_u32 = smem_u32(&bars[0]);
    auto bar_full = [&](int h, int s) { return bars_u32 + 8u * (uint32_t)(h * T2_MAX_STAGES + s); };
    auto bar_empty = [&](int h, int s) { return bars_u32 + 8u * (uint32_t)((2 + h) * T2_MAX_STAGES + s); };
    const uint32_t bar_w = bars_u32 + 8u * (4 * T2_MAX_STAGES);

    if (t == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int s = 0; s < T2_MAX_STAGES; ++s) {
                mbar_init(bar_full(h, s), T2_PROD_WARPS / 2);  // one elected arrival per producer warp of h
                mbar_init(bar_empty(h, s), T2_EPI_WARPS / 2);  // one elected arrival per consumer warp of h
            }
        mbar_init(bar_w, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
    }
    // Everything above (barrier init, descriptor prefetch) overlaps the previous kernel of the stream;
    // nothing below this line runs before that kernel's results are visible.
    SPG_PDL_ENTRY();
    if (t == 0) {
        // resident weight slice by TMA: rows [n0, n0+NS) of every (chunk, hi|lo) block of the image
        // (a block is [N rows][128 B], already in the SWIZZLE_128B layout the MMA reads)
        mbar_expect_tx(bar_w, (uint32_t)(nk * 2 * NS * T2_KC * 4));
        const uint32_t wres_u = smem_u32(wres);
        for (int blk = 0; blk < nk * 2; ++blk)
            tma_load_2d(wres_u + (uint32_t)blk * (NS * T2_KC * 4), &wmap, 0, blk * p.N + n0, bar_w);
    }
    // Producer threads put their first A chunks in flight before anything else: the global-load
    // latency then overlaps the resident-weight load and the CTA-wide barrier below.
    // Register-level prefetch ring: PF chunks of A are in flight per thread (the global-load
    // latency under load is far longer than one chunk's transform + MMA).  The BNBWD
    // prologue streams two operands, so its ring is half as deep (same register budget).
    constexpr int PF = PRO == PRO_BNBWD ? 2 : 4;
    constexpr int NOPS = PRO == PRO_BNBWD ? 2 : 1;
    float4 q[PF][NOPS][4];
    const int pt = t - T2_EPI_WARPS * 32;  // producer thread id 0..255 (negative: consumers)
    const int ph = pt >> 7, pq = pt & 127;  // producer warpgroup = half of the tile it fills, thread in it
    auto load = [&](int64_t tile, int kc, float4 (&dst)[NOPS][4]) {
        const int64_t m0 = tile * T2_BM;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int row = ph * 64 + (pq >> 3) + 16 * j, c16 = pq & 7;
            const bool ok = tile < tiles && m0 + row < p.M;
            dst[0][j] = ok ? __ldg(reinterpret_cast<const float4*>(p.A + (m0 + row) * p.lda + kc * T2_KC + c16 * 4))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            if (PRO == PRO_BNBWD)
                dst[NOPS - 1][j] =
                    ok ? __ldg(reinterpret_cast<const float4*>(p.A2 + (m0 + row) * p.lda2 + kc * T2_KC + c16 * 4))
                       : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto advance = [&](int64_t& tl, int& k) {
        if (++k == nk) {
            k = 0;
            tl += gridDim.x;
        }
    };
    // load cursor (runs PF-1 items ahead of the consume cursor)
    int64_t ltile = blockIdx.x;
    int lkc = 0;
    if (pt >= 0) {
#pragma unroll
        for (int d = 0; d < PF - 1; ++d) {
            load(ltile, lkc, q[d]);
            advance(ltile, lkc);
        }
    }
    // per-channel vectors of the fused prologue / epilogue, once per CTA
    float* sc_s = reinterpret_cast<float*>(wres + (size_t)nk * 2 * NS * T2_KC * 4);
    float* sh_s = sc_s + p.K;
    float* cy_s = sh_s + p.K;   // BNBWD: coefficient of y
    float* c0_s = cy_s + p.K;   // BNBWD: constant term
    float* bias_s = c0_s + p.K;
    float* ev_s = bias_s + NS;  // BNRED: [4][NS] = scale2, shift2, mean2, rstd2 of the layer below
    float* acc_s = ev_s + 4 * NS;  // column accumulators [8 consumer warps][NS][4]
    for (int i = t; i < p.K; i += T2_THREADS) {
        const float sc = p.a_scale ? p.a_scale[i] : 1.f;
        sc_s[i] = sc;
        sh_s[i] = p.a_shift ? p.a_shift[i] : 0.f;
        if (PRO == PRO_BNBWD) {
            // dY = sc*(gz - s1/M - (y-mu)*rstd*s2/M) = sc*gz + cy*y + c0
            const float mu = p.a_mean[i], rstd = 1.f / sqrtf(p.a_var[i] + p.a_eps);
            const float m1 = p.a_s12[i] / (float)p.M, m2 = p.a_s12[p.K + i] / (float)p.M;
            cy_s[i] = -sc * rstd * m2;
            c0_s[i] = sc * (rstd * m2 * mu - m1);
        }
    }
    for (int i = t; i < NS; i += T2_THREADS) {
        bias_s[i] = p.bias ? p.bias[n0 + i] : 0.f;
        if (p.epi == EPI_BNRED) {
            ev_s[i] = p.e_scale ? p.e_scale[n0 + i] : 1.f;
            ev_s[NS + i] = p.e_shift ? p.e_shift[n0 + i] : 0.f;
            ev_s[2 * NS + i] = p.e_mean[n0 + i];
            ev_s[3 * NS + i] = 1.f / sqrtf(p.e_var[n0 + i] + p.e_eps);
        }
    }
    for (int i = t; i < T2_EPI_WARPS * NS * 4; i += T2_THREADS) acc_s[i] = 0.f;
    __syncthreads();

    if (warp >= T2_EPI_WARPS) {
        // ================================ producers ================================
        const bool pro = PRO == PRO_BNBWD || p.a_scale || p.a_shift || p.a_relu;
        int64_t tile = blockIdx.x;
        int kc = 0;
        uint32_t it = 0;
        const int c16 = pq & 7;  // 16-byte chunk of the 128-byte K row (same for all 4 rows)
        uint32_t soff[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) soff[j] = sw128_off((pq >> 3) + 16 * j, c16);
        const uint32_t ring_u = ring(ph);
        const bool side_store = PRO == PRO_BNBWD && p.dy_out != nullptr && blockIdx.y == 0;
        auto st_shared4 = [](uint32_t addr, uint4 v) {
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y),
                         "r"(v.z), "r"(v.w)
                         : "memory");
        };
        auto consume = [&](float4 (&cur)[NOPS][4], float4 (&far)[NOPS][4]) {
            const int s = it % nst;
            const uint32_t use = it / nst;
            load(ltile, lkc, far);  // item it+PF-1
            advance(ltile, lkc);
            const int col = kc * T2_KC + c16 * 4;
            const float4 sc = *reinterpret_cast<const float4*>(sc_s + col);
            const float4 sh = *reinterpret_cast<const float4*>(sh_s + col);
            float4 cy = make_float4(0.f, 0.f, 0.f, 0.f), c0 = cy;
            if (PRO == PRO_BNBWD) {
                cy = *reinterpret_cast<const float4*>(cy_s + col);
                c0 = *reinterpret_cast<const float4*>(c0_s + col);
            }
            if (use > 0) mbar_wait(bar_empty(ph, s), (use - 1) & 1);
            const uint32_t stage = ring_u + (uint32_t)s * T2_HALF_STAGE_BYTES;
            const int64_t m0 = tile * T2_BM + ph * 64;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float4 v = cur[0][j];
                const int64_t row = m0 + (pq >> 3) + 16 * j;
                if (pro && row < p.M) {
                    if (PRO == PRO_BNBWD) {
                        const float4 y = cur[NOPS - 1][j];
                        if (p.a_relu) {
                            if (!(fmaf(y.x, sc.x, sh.x) > 0.f)) v.x = 0.f;
                            if (!(fmaf(y.y, sc.y, sh.y) > 0.f)) v.y = 0.f;
                            if (!(fmaf(y.z, sc.z, sh.z) > 0.f)) v.z = 0.f;
                            if (!(fmaf(y.w, sc.w, sh.w) > 0.f)) v.w = 0.f;
                        }
                        v.x = fmaf(sc.x, v.x, fmaf(cy.x, y.x, c0.x));
                        v.y = fmaf(sc.y, v.y, fmaf(cy.y, y.y, c0.y));
                        v.z = fmaf(sc.z, v.z, fmaf(cy.z, y.z, c0.z));
                        v.w = fmaf(sc.w, v.w, fmaf(cy.w, y.w, c0.w));
                        st_global4(p.dy_out + row * p.lddy + col, v, side_store);
                    } else {
                        v.x = fmaf(v.x, sc.x, sh.x);
                        v.y = fmaf(v.y, sc.y, sh.y);
                        v.z = fmaf(v.z, sc.z, sh.z);
                        v.w = fmaf(v.w, sc.w, sh.w);
                        if (p.a_relu) {
                            v.x = fmaxf(v.x, 0.f);
                            v.y = fmaxf(v.y, 0.f);
                            v.z = fmaxf(v.z, 0.f);
                            v.w = fmaxf(v.w, 0.f);
                        }
                    }
                }
                uint4 hi, lo;
                hi.x = to_tf32(v.x);
                hi.y = to_tf32(v.y);
                hi.z = to_tf32(v.z);
                hi.w = to_tf32(v.w);
                lo.x = to_tf32(v.x - __uint_as_float(hi.x));
                lo.y = to_tf32(v.y - __uint_as_float(hi.y));
                lo.z = to_tf32(v.z - __uint_as_float(hi.z));
                lo.w = to_tf32(v.w - __uint_as_float(hi.w));
                st_shared4(stage + soff[j], hi);
                st_shared4(stage + T2_HALF_A_BYTES + soff[j], lo);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_full(ph, s));
            advance(tile, kc);
            ++it;
        };
        while (tile < tiles) {
#pragma unroll
            for (int u = 0; u < PF; ++u) {
                consume(q[u], q[(u + PF - 1) % PF]);
                if (tile >= tiles) break;
            }
        }
    } else {
        // ======================= consumers: wgmma + epilogue from registers =======================
        const int g = warp >> 2, wl = warp & 3;  // warpgroup (64-row half of the tile), warp in it
        const int r = lane >> 2, cq = 2 * (lane & 3);
        float* acc_w = acc_s + warp * (NS * 4);
        const uint32_t wres_u32 = smem_u32(wres);
        const uint32_t ring_u = ring(g);
        float acc[NS / 2];
        float n_w = 0.f;  // STATS: rows this warp has reduced so far (the count of every one of its columns)
        uint32_t it = 0;
        mbar_wait(bar_w, 0);  // resident weights have landed (TMA complete_tx)
        for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            // warpgroup 1 waits for warpgroup 0 to have issued this tile's MMAs, warpgroup 0 (after its first
            // tile) for warpgroup 1 to have issued the previous tile's
            if (g == 1 || tile != blockIdx.x) turn_wait(T2_TURN_BAR + g);
            for (int kc = 0; kc < nk; ++kc, ++it) {
                const int s = it % nst;
                mbar_wait(bar_full(g, s), (it / nst) & 1);
                const uint32_t a_hi = ring_u + (uint32_t)s * T2_HALF_STAGE_BYTES;
                const uint32_t a_lo = a_hi + T2_HALF_A_BYTES;
                const uint32_t b_hi = wres_u32 + (uint32_t)(kc * 2) * (NS * T2_KC * 4);
                const uint32_t b_lo = b_hi + NS * T2_KC * 4;
                wg_reg_fence(acc);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < T2_KC / 8; ++ks) {
                    const uint32_t ko = ks * 32;
                    const uint64_t dah = wg_desc_k_sw128(a_hi + ko), dal = wg_desc_k_sw128(a_lo + ko);
                    const uint64_t dbh = wg_desc_k_sw128(b_hi + ko), dbl = wg_desc_k_sw128(b_lo + ko);
                    wgmma_tf32<NS>(acc, dah, dbh, (kc | ks) ? 1u : 0u);
                    wgmma_tf32<NS>(acc, dal, dbh, 1u);
                    wgmma_tf32<NS>(acc, dah, dbl, 1u);
                }
                wg_commit();
                wg_wait<0>();
                wg_reg_fence(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty(g, s));
            }
            // the other warpgroup's turn: warpgroup 1 takes this tile, warpgroup 0 the next one (if there is one;
            // both walk the same tiles, so warpgroup 0 always waits for this)
            if (g == 0 || tile + gridDim.x < tiles) turn_pass(T2_TURN_BAR + (g ^ 1));
            // ---- epilogue: this thread holds rows ra = row0 + r and rb = ra + 8, column pairs 8j + cq
            const int64_t row0 = tile * T2_BM + g * 64 + wl * 16;
            const int nv = (int)max((int64_t)0, min((int64_t)16, p.M - row0));
            const bool va = r < nv, vb = r + 8 < nv;
            float* ca = p.C + (row0 + r) * p.ldc + n0;
            float* cb = ca + 8 * p.ldc;
            // STATS: the pivot of a column is the first value the warp saw in it, stored (lanes r == 0) at the
            // first tile with a valid row and read by the whole warp at the later ones
            const bool have_pivot = n_w > 0.f;
            if (p.epi == EPI_STATS) __syncwarp();
            const bool reduce = p.epi == EPI_BNRED || (p.epi == EPI_STATS && nv > 0);
            // Blocks of 2 column pairs = the 4 columns 8(j0 + u) + cq + e, u < 2, e < 2, of this lane (block
            // column k = 2u + e); lane r folds sum vr = 4(r & 1) + 2((r >> 1) & 1) + (r >> 2) of each block, i.e.
            // the first (vr even) or second sum of block column vr / 2 (see reduce_scatter8)
            const int vr = 4 * (r & 1) + 2 * ((r >> 1) & 1) + (r >> 2);
            // BNRED reads the layer below's y for YB column pairs (two blocks; one at NS = 128, where the 64
            // accumulators leave no room for more) ahead of their reductions
            constexpr int YB = NS == 128 ? 2 : 4;
#pragma unroll
            for (int j1 = 0; j1 < NS / 8; j1 += YB) {
                float2 ya[YB], yb[YB];
                if (p.epi == EPI_BNRED) {
#pragma unroll
                    for (int u = 0; u < YB; ++u) {
                        const int64_t col = n0 + 8 * (j1 + u) + cq;
                        ya[u] = va ? __ldg(reinterpret_cast<const float2*>(p.e_y + (row0 + r) * p.e_ldy + col))
                                   : make_float2(0.f, 0.f);
                        yb[u] = vb ? __ldg(reinterpret_cast<const float2*>(p.e_y + (row0 + r + 8) * p.e_ldy + col))
                                   : make_float2(0.f, 0.f);
                    }
                }
#pragma unroll
                for (int j0 = j1; j0 < j1 + YB; j0 += 2) {
                    float v[8];    // per block column k: the two sums over this thread's rows, at 2k and 2k + 1
                    float piv[4];  // STATS: pivot of block column k
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int j = j0 + u;
                        const int c = 8 * j + cq;
                        const float2 oa = make_float2(acc[4 * j] + bias_s[c], acc[4 * j + 1] + bias_s[c + 1]);
                        const float2 ob = make_float2(acc[4 * j + 2] + bias_s[c], acc[4 * j + 3] + bias_s[c + 1]);
                        st_global2(ca + c, oa, va);
                        st_global2(cb + c, ob, vb);
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int k = 2 * u + e;
                            if (p.epi == EPI_BNRED) {
                                // BatchNorm-backward sums of the layer below: gz = relu'(y) * g
                                const float esc = ev_s[c + e], esh = ev_s[NS + c + e];
                                const float emu = ev_s[2 * NS + c + e], ers = ev_s[3 * NS + c + e];
                                const float2 y0p = ya[j - j1], y1p = yb[j - j1];
                                const float y0 = e ? y0p.y : y0p.x, y1 = e ? y1p.y : y1p.x;
                                float g0 = va ? (e ? oa.y : oa.x) : 0.f, g1 = vb ? (e ? ob.y : ob.x) : 0.f;
                                if (p.e_relu) {
                                    if (!(fmaf(y0, esc, esh) > 0.f)) g0 = 0.f;
                                    if (!(fmaf(y1, esc, esh) > 0.f)) g1 = 0.f;
                                }
                                v[2 * k] = g0 + g1;
                                v[2 * k + 1] = fmaf(g1, (y1 - emu) * ers, g0 * ((y0 - emu) * ers));
                            } else if (p.epi == EPI_STATS && nv > 0) {
                                // pivoted sums over the valid rows of this warp's 16-row group
                                const float x0 = e ? oa.y : oa.x, x1 = e ? ob.y : ob.x;
                                const float first = __shfl_sync(0xffffffffu, x0, lane & 3);
                                piv[k] = have_pivot ? acc_w[(c + e) * 4 + 3] : first;
                                const float d0 = va ? x0 - piv[k] : 0.f;
                                const float d1 = vb ? x1 - piv[k] : 0.f;
                                v[2 * k] = d0 + d1;
                                v[2 * k + 1] = fmaf(d1, d1, d0 * d0);
                            }
                        }
                    }
                    if (reduce) {
                        // lanes with the same lane % 4 hold the same columns: fold the 8 row pairs
                        const float sum = reduce_scatter8(v, r);
                        const int k = vr >> 1;  // block column
                        // BNRED: s1, s2 in o[0], o[1]; STATS: the pivoted sums in o[1], o[2] (o[0]: count, o[3]: pivot)
                        acc_w[(8 * (j0 + (k >> 1)) + cq + (k & 1)) * 4 + (p.epi == EPI_STATS) + (vr & 1)] += sum;
                        if (p.epi == EPI_STATS && r == 0 && !have_pivot) {
#pragma unroll
                            for (int q = 0; q < 4; ++q) acc_w[(8 * (j0 + (q >> 1)) + cq + (q & 1)) * 4 + 3] = piv[q];
                        }
                    }
                }
            }
            if (p.epi == EPI_STATS && nv > 0) n_w += (float)nv;
        }
        if (p.epi == EPI_STATS && r == 0) {
#pragma unroll
            for (int j = 0; j < NS / 8; ++j) {
                acc_w[(8 * j + cq) * 4] = n_w;
                acc_w[(8 * j + cq + 1) * 4] = n_w;
            }
        }
    }

    __syncthreads();
    if (p.epi == EPI_NONE) return;

    // ---------------- column reductions: CTA partial, then the merge kernel folds -------------
    if (t < NS) {
        if (p.epi == EPI_STATS) {
            // Chan merge of the 8 row groups (each: n, pivot + d1/n, d2 - d1^2/n), fixed order
            double n = 0.0, mean = 0.0, m2 = 0.0;
#pragma unroll
            for (int wq = 0; wq < T2_EPI_WARPS; ++wq) {
                const float* o = acc_s + wq * (NS * 4) + t * 4;
                const double nb = (double)o[0];
                if (nb > 0.0) {
                    const double mb = (double)o[3] + (double)o[1] / nb;
                    const double qb = fmax((double)o[2] - (double)o[1] * (double)o[1] / nb, 0.0);
                    const double tot = n + nb, delta = mb - mean;
                    m2 += qb + delta * delta * n * nb / tot;
                    mean += delta * nb / tot;
                    n = tot;
                }
            }
            float* o = p.part + ((int64_t)blockIdx.x * p.N + n0 + t) * 3;
            o[0] = (float)n;
            o[1] = (float)mean;
            o[2] = (float)m2;
        } else {
            float a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int wq = 0; wq < T2_EPI_WARPS; ++wq) {
                a1 += acc_s[wq * (NS * 4) + t * 4];
                a2 += acc_s[wq * (NS * 4) + t * 4 + 1];
            }
            float* o = p.part + ((int64_t)blockIdx.x * p.N + n0 + t) * 2;
            o[0] = a1;
            o[1] = a2;
        }
    }
}

// Second (tiny) kernel of a fused reduction: one warp per column folds the <= kNumSMs per-CTA partials in
// a fixed order (deterministic) and writes mean/var (+ BatchNorm fold, running statistics) or s1|s2.
// (An in-kernel grid barrier would need a cooperative launch, which must wait until the WHOLE grid fits
// on the GPU and thereby serialises against the weight-gradient kernels of the side stream.)
__global__ void __launch_bounds__(256) tc_merge_kernel(const Tc2Args p, int P) {
    SPG_PDL_ENTRY();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 8 + warp;
    if (c >= p.N) return;
    {
        if (p.epi == EPI_STATS) {
            double sn = 0.0, snm = 0.0;
            float pn[5], pm[5], pq[5];  // P <= kNumSMs <= 160 -> <= 5 partials per lane
#pragma unroll
            for (int u = 0; u < 5; ++u) {
                const int k = lane + 32 * u;
                pn[u] = pm[u] = pq[u] = 0.f;
                if (k < P) {
                    const float* o = p.part + ((int64_t)k * p.N + c) * 3;
                    pn[u] = __ldcg(o);
                    pm[u] = __ldcg(o + 1);
                    pq[u] = __ldcg(o + 2);
                }
                sn += (double)pn[u];
                snm += (double)pn[u] * (double)pm[u];
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                sn += __shfl_xor_sync(0xffffffffu, sn, o);
                snm += __shfl_xor_sync(0xffffffffu, snm, o);
            }
            const double mu = sn > 0.0 ? snm / sn : 0.0;
            double qq = 0.0;
#pragma unroll
            for (int u = 0; u < 5; ++u) {
                const double d = (double)pm[u] - mu;
                qq += (double)pq[u] + (double)pn[u] * d * d;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) qq += __shfl_xor_sync(0xffffffffu, qq, o);
            if (lane == 0) {
                const float mu_f = (float)mu;
                const float var_f = sn > 0.0 ? (float)(qq / sn) : 0.f;
                p.mean_out[c] = mu_f;
                p.var_out[c] = var_f;
                if (p.fold.enabled) bn_fold_col(p.fold, c, mu_f, var_f);
            }
        } else {
            double a1 = 0.0, a2 = 0.0;
            for (int k = lane; k < P; k += 32) {
                const float* o = p.part + ((int64_t)k * p.N + c) * 2;
                a1 += (double)__ldcg(o);
                a2 += (double)__ldcg(o + 1);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                a1 += __shfl_xor_sync(0xffffffffu, a1, o);
                a2 += __shfl_xor_sync(0xffffffffu, a2, o);
            }
            if (lane == 0) {
                p.e_s12[c] = (float)a1;
                p.e_s12[p.N + c] = (float)a2;
            }
        }
    }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    });
    return fn;
}

// 2-D view of a weight image: [rows = (K/32)*2*N][32 floats]; one box = the NS rows of a CTA's slice
static int make_weight_map(CUtensorMap* map, const float* image, int N, int K, int NS) {
    EncodeTiledFn fn = encode_tiled();
    if (!fn) return SPG_E_UNSUPPORTED;
    const cuuint64_t dims[2] = {(cuuint64_t)T2_KC, (cuuint64_t)(K / T2_KC) * 2 * (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)T2_KC * 4};
    const cuuint32_t box[2] = {(cuuint32_t)T2_KC, (cuuint32_t)NS};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(image), dims, strides, box,
                          estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SPG_OK : SPG_E_BADARG;
}

static inline int fixed_smem(int NS, int K) {
    return (K / T2_KC) * 2 * NS * T2_KC * 4 + (4 * K + NS + 4 * NS + T2_EPI_WARPS * NS * 4) * 4;
}

static inline int stages_for(int NS, int K) {
    int nst = (232448 - 1024 - fixed_smem(NS, K)) / T2_STAGE_BYTES;  // 227 KB per CTA minus 1 KB static
    return nst > T2_MAX_STAGES ? T2_MAX_STAGES : nst;
}

template <int NS, int PRO>
static int launch_tc2(Tc2Args& a, const float* image, cudaStream_t s) {
    const int slices = a.N / NS;
    const int64_t tiles = ceil_div64(a.M, T2_BM);
    int64_t gx = kNumSMs / slices;
    if (gx > tiles) gx = tiles;
    if (gx < 1) gx = 1;
    const int nst = stages_for(NS, a.K);
    if (nst < 2) return SPG_E_UNSUPPORTED;
    a.nstages = nst;
    CUtensorMap map;
    int rc = make_weight_map(&map, image, a.N, a.K, NS);
    if (rc) return rc;
    const int smem = nst * T2_STAGE_BYTES + fixed_smem(NS, a.K);
    cudaError_t e = cudaFuncSetAttribute(tc_gemm2_kernel<NS, PRO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    dim3 grid((unsigned)gx, (unsigned)slices);
    SPG_LAUNCH(K_TC_GEMM, s, (tc_gemm2_kernel<NS, PRO>), grid, T2_THREADS, smem, a, map);
    rc = launch_status();
    if (rc || a.epi == EPI_NONE) return rc;
    SPG_LAUNCH(K_TC_MERGE, s, tc_merge_kernel, (unsigned)ceil_div64(a.N, 8), 256, 0, a, (int)gx);
    return launch_status();
}

// slice width: the resident image (2*NS*K*4 bytes) must fit next to a >= 2-stage A ring in 227 KB
static inline int pick_ns(int N, int K) {
    if (N % 128 == 0 && stages_for(128, K) >= 2) return 128;
    if (N % 64 == 0 && stages_for(64, K) >= 2) return 64;
    if (N % 32 == 0 && N <= 64 && stages_for(32, K) >= 2) return 32;
    return 0;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_tc_gemm_supported(int64_t M, int N, int K) {
    return (M > 0 && N > 0 && N <= 256 && K >= T2_KC && K % T2_KC == 0 && pick_ns(N, K) != 0) ? 1 : 0;
}

/* CTAs along the row dimension = number of per-column partials a fused reduction writes */
int spg_tc_gemm_max_partials(void) { return kNumSMs; }

int spg_tc_gemm_ex(const float* A, int64_t lda, const float* weight_image, const float* bias, float* C,
                   int64_t ldc, int64_t M, int N, int K,
                   const float* a_scale, const float* a_shift, int a_relu,
                   const float* a2, int64_t lda2, const float* a_mean, const float* a_var,
                   const float* a_s12, float a_eps, float* dy_out, int64_t lddy,
                   int epilogue, float* partials_ws,
                   float* mean_out, float* var_out, const float* gamma, const float* beta, float eps,
                   float* scale_out, float* shift_out, float* running_mean, float* running_var,
                   int64_t* num_batches_tracked, float momentum,
                   const float* e_y, int64_t e_ldy, const float* e_scale, const float* e_shift,
                   const float* e_mean, const float* e_var, float e_eps, int e_relu, float* e_s12,
                   spg_stream_t stream) {
    if (M < 0 || !A || !weight_image || !C) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!spg_tc_gemm_supported(M, N, K)) return SPG_E_UNSUPPORTED;
    if ((lda & 3) || (ldc & 3) || lda < K || ldc < N) return SPG_E_ALIGN;
    if (((uintptr_t)A | (uintptr_t)C | (uintptr_t)weight_image | (uintptr_t)a2 | (uintptr_t)dy_out |
         (uintptr_t)e_y) & 15)
        return SPG_E_ALIGN;
    if (ceil_div64(M, T2_BM) > 2147483647ll) return SPG_E_UNSUPPORTED;
    Tc2Args a;
    a.A = A; a.lda = lda; a.A2 = a2; a.lda2 = lda2; a.bias = bias; a.C = C; a.ldc = ldc; a.M = M;
    a.N = N; a.K = K; a.a_scale = a_scale; a.a_shift = a_shift; a.a_relu = a_relu;
    a.a_mean = a_mean; a.a_var = a_var; a.a_s12 = a_s12; a.a_eps = a_eps;
    a.dy_out = dy_out; a.lddy = lddy;
    a.epi = epilogue; a.part = partials_ws;
    a.mean_out = mean_out; a.var_out = var_out;
    a.fold = fold_args(gamma, beta, eps, scale_out, shift_out, running_mean, running_var, num_batches_tracked,
                       momentum, M);
    a.e_y = e_y; a.e_ldy = e_ldy; a.e_scale = e_scale; a.e_shift = e_shift; a.e_mean = e_mean;
    a.e_var = e_var; a.e_eps = e_eps; a.e_relu = e_relu; a.e_s12 = e_s12; a.nstages = 0;
    const bool bnbwd = a2 != nullptr;
    if (bnbwd && (!a_scale || !a_shift || !a_mean || !a_var || !a_s12 || (lda2 & 3) || lda2 < K))
        return SPG_E_BADARG;
    if (dy_out && (!bnbwd || (lddy & 3) || lddy < K)) return SPG_E_BADARG;
    if (epilogue == EPI_STATS) {
        if (!partials_ws || !mean_out || !var_out) return SPG_E_BADARG;
        if (a.fold.enabled && !shift_out) return SPG_E_BADARG;
    } else if (epilogue == EPI_BNRED) {
        if (!partials_ws || !e_y || !e_mean || !e_var || !e_s12 || (e_ldy & 3) || e_ldy < N) return SPG_E_BADARG;
    } else if (epilogue != EPI_NONE) {
        return SPG_E_BADARG;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int ns = pick_ns(N, K);
#define SPG_TC2_CASE(NS_)                                                                  \
    if (ns == NS_) return bnbwd ? launch_tc2<NS_, PRO_BNBWD>(a, weight_image, s)          \
                                : launch_tc2<NS_, PRO_AFFINE>(a, weight_image, s);
    SPG_TC2_CASE(128)
    SPG_TC2_CASE(64)
    SPG_TC2_CASE(32)
#undef SPG_TC2_CASE
    return SPG_E_UNSUPPORTED;
}

/* plain form: prologue affine+ReLU, no fused reduction */
int spg_tc_gemm(const float* A, int64_t lda, const float* weight_image, const float* bias, float* C,
                int64_t ldc, int64_t M, int N, int K, const float* a_scale, const float* a_shift,
                int a_relu, spg_stream_t stream) {
    return spg_tc_gemm_ex(A, lda, weight_image, bias, C, ldc, M, N, K, a_scale, a_shift, a_relu, nullptr, 0,
                          nullptr, nullptr, nullptr, 0.f, nullptr, 0, EPI_NONE, nullptr, nullptr, nullptr,
                          nullptr, nullptr, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f, nullptr, 0,
                          nullptr, nullptr, nullptr, nullptr, 0.f, 0, nullptr, stream);
}

}  // extern "C"
