// Eval-mode PointNet trunk as ONE kernel per chain: cloud tile -> (xy transform) -> up to six point-wise
// layers (Conv1d k=1 with BatchNorm folded into weights and bias, ReLU) -> max over the cloud's points.
// No [rows, C] activation ever reaches HBM: a CTA keeps one superpoint (128 points) on chip from the input
// tile to the pooled row.
//
//   reference: learning/pointnet.py:120-133 (PointNet.forward) and :55-61 (STNkD.forward) under
//   model.eval() (learning/main.py:229-311): conv -> BatchNorm1d(running statistics) -> ReLU chains, then
//   F.max_pool1d over the points.
//
// Per CTA (persistent over superpoints b = blockIdx.x, blockIdx.x + gridDim.x, ...):
//   warp 8 (one thread)  TMA producer: the superpoint's [F, 128] input tile (cp.async.bulk.tensor over the
//                        NCL clouds tensor) and the weight stream — for every layer, N-tile and K-chunk one
//                        [N_tile x 128 B] block (fp32 path: a hi and a lo block) of the pre-split,
//                        pre-swizzled weight image (the weights live in L2)
//   warps 0-7            two consumer warpgroups, one per 64 points: input tile -> transform -> A chunk 0;
//                        per layer wgmma.mma_async with A = the layer's input activations in shared memory
//                        (K-major SWIZZLE_128B, the warpgroup's own 64 rows) and B = the weight stage, fp32
//                        accumulator in registers; then + folded bias, ReLU, written IN PLACE as the next
//                        layer's A (every MMA of the layer has completed first: a non-last layer is one
//                        N-tile); after the last layer the max over the points -> pooled[b, :]
// fp32 path: 3xTF32 (hi/lo split of both operands, three MMAs per product: fp32-equivalent).
// bf16 path (configs[3] arithmetic): bf16 operands, fp32 accumulation, ONE MMA per product; inputs and every
// layer output are rounded to bf16 (8-bit mantissa): results agree with the fp32 path to ~1e-2 (tests state
// the bound), not to 1e-4.
// mbarriers: w_full/w_empty (weight ring), x_full/x_empty (input double buffer).
#include <cuda.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "tc_common.cuh"

namespace spg {

constexpr int PF_ROWS = 128;          // points per superpoint
constexpr int PF_KC = 32;             // floats per K chunk (one 128-byte swizzle row)
constexpr int PF_MAXK = 128;          // widest layer input kept in shared memory
constexpr int PF_NT = 128;            // accumulator tile width
constexpr int PF_STAGE_BYTES = 2 * PF_NT * PF_KC * 4;        // hi + lo of one (N-tile, K-chunk) = 32 KB
constexpr int PF_STAGES = 2;          // fp32 weight ring depth (the 128 KB hi|lo A operand takes the rest)
constexpr int PF_A_CHUNK_BYTES = PF_ROWS * 128;              // one 128-byte-row K chunk of A: 16 KB
constexpr int PF_A_BYTES = (PF_MAXK / PF_KC) * PF_A_CHUNK_BYTES;  // 64 KB (hi or lo)
constexpr int PF_MAXF = 16;            // input features (S3DIS 14, Semantic3D 11, vKITTI 9)
constexpr int PF_X_BYTES = PF_MAXF * PF_ROWS * 4;            // one input tile buffer (8 KB)
constexpr int PF_MAX_LAYERS = 6;
constexpr int PF_ACT_WARPS = 8;        // consumer warps: two warpgroups
constexpr int PF_THREADS = (PF_ACT_WARPS + 1) * 32;
constexpr int PF_MAX_BIAS = 1024;
constexpr int PF_POOL_FLOATS = PF_ACT_WARPS * 256;

constexpr int PB_KC = 64;                                   // bf16 elements per K chunk (128-byte row)
constexpr int PB_STAGES = 8;
constexpr int PB_STAGE_BYTES = PF_NT * 128;                 // one (N-tile, K-chunk) weight block = 16 KB
constexpr int PB_A_BYTES = (PF_MAXK / PB_KC) * PF_A_CHUNK_BYTES;  // 32 KB

struct PfLayer {
    int K, N;      // K padded to a multiple of the chunk, N in {32, 64, 128, 256}
    int w_row;     // first row of this layer's blocks in the weight image ([rows][128 B])
    int b_off;     // offset of the folded bias in the bias vector
};

struct PfArgs {
    int n_layers;
    PfLayer L[PF_MAX_LAYERS];
    int F;                 // input features (<= 16)
    int64_t B;             // superpoints
    const float* T;        // [B, 4] spatial transformer output (xy' = xy (T + I)), or null
    int add_eye;
    const float* bias;     // folded biases of all layers
    int n_bias;
    float* pooled;         // [B, ldp]
    int64_t ldp;
};

__device__ __forceinline__ void pf_tma_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(map), "r"(x), "r"(y), "r"(bar)
        : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16x2(float e0, float e1) {  // e0 -> low half (lower address)
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(e1), "f"(e0));
    return r;
}

__device__ __forceinline__ void bar_named(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

template <bool BF16>
struct PfCfg {
    static constexpr int KC = BF16 ? PB_KC : PF_KC;
    static constexpr int STAGES = BF16 ? PB_STAGES : PF_STAGES;
    static constexpr int STAGE_BYTES = BF16 ? PB_STAGE_BYTES : PF_STAGE_BYTES;
    static constexpr int A_BYTES = BF16 ? PB_A_BYTES : 2 * PF_A_BYTES;  // fp32: [hi][lo]
    static constexpr int SMEM = A_BYTES + STAGES * STAGE_BYTES + 2 * PF_X_BYTES + (PF_MAX_BIAS + PF_POOL_FLOATS) * 4;
};

// Shared-memory state one consumer warpgroup works with.
struct PfCtx {
    uint32_t a_u, w_u, bars_u;
    float* bias_s;
    float* pool_s;
    int g, warp, lane;
};

// One N-tile of one layer for the calling warpgroup: MMAs over the weight stream, then the epilogue.
template <bool BF16, int NT>
__device__ __forceinline__ void pf_tile(const PfCtx& c, const PfLayer& Ly, int nt, bool last, uint32_t& it) {
    using C = PfCfg<BF16>;
    float acc[NT / 2];
    const uint32_t a_rows = c.a_u + (uint32_t)c.g * (64 * 128);  // this warpgroup's 64 rows of every A chunk
    for (int kc = 0; kc < Ly.K / C::KC; ++kc, ++it) {
        const int s = it % C::STAGES;
        mbar_wait(c.bars_u + 8u * (uint32_t)s, (it / C::STAGES) & 1);  // w_full(s)
        const uint32_t a0 = a_rows + (uint32_t)kc * PF_A_CHUNK_BYTES;
        const uint32_t b0 = c.w_u + (uint32_t)s * C::STAGE_BYTES;
        wg_reg_fence(acc);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {  // 32 bytes of the 128-byte row per instruction
            const uint32_t ko = ks * 32;
            if constexpr (BF16) {
                wgmma_bf16<NT>(acc, wg_desc_k_sw128(a0 + ko), wg_desc_k_sw128(b0 + ko), (kc | ks) ? 1u : 0u);
            } else {
                const uint64_t dah = wg_desc_k_sw128(a0 + ko), dal = wg_desc_k_sw128(a0 + PF_A_BYTES + ko);
                const uint64_t dbh = wg_desc_k_sw128(b0 + ko), dbl = wg_desc_k_sw128(b0 + NT * 128 + ko);
                wgmma_tf32<NT>(acc, dah, dbh, (kc | ks) ? 1u : 0u);
                wgmma_tf32<NT>(acc, dal, dbh, 1u);
                wgmma_tf32<NT>(acc, dah, dbl, 1u);
            }
        }
        wg_commit();
        wg_wait<0>();
        wg_reg_fence(acc);
        __syncwarp();
        if (c.lane == 0) mbar_arrive(c.bars_u + 8u * (uint32_t)(C::STAGES + s));  // w_empty(s)
    }
    // this thread holds points prow and prow + 8, columns 8j + cq, 8j + cq + 1 of the tile
    const int r = c.lane >> 2, cq = 2 * (c.lane & 3);
    const int prow = c.g * 64 + (c.warp & 3) * 16 + r;
    const float* bs = c.bias_s + Ly.b_off + nt * NT;
    if (!last) {
        // in place: every warp of the warpgroup has finished reading this layer's A
        bar_named(1 + c.g, 128);
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int col = 8 * j + cq;  // a non-last layer is a single N-tile: col is the channel
            const float o0 = fmaxf(acc[4 * j] + bs[col], 0.f), o1 = fmaxf(acc[4 * j + 1] + bs[col + 1], 0.f);
            const float o2 = fmaxf(acc[4 * j + 2] + bs[col], 0.f), o3 = fmaxf(acc[4 * j + 3] + bs[col + 1], 0.f);
            if constexpr (BF16) {
                const uint32_t base = c.a_u + (uint32_t)(col / PB_KC) * PF_A_CHUNK_BYTES + (uint32_t)(col & 7) * 2u;
                const int c16 = (col % PB_KC) >> 3;
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + sw128_off(prow, c16)), "r"(pack_bf16x2(o0, o1)) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + sw128_off(prow + 8, c16)), "r"(pack_bf16x2(o2, o3)) : "memory");
                if (NT == 32) {  // a 32-wide layer fills only half of the next 64-element K chunk: zero the rest
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + sw128_off(prow, c16 + 4)), "r"(0u) : "memory");
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(base + sw128_off(prow + 8, c16 + 4)), "r"(0u) : "memory");
                }
            } else {
                const uint32_t base = c.a_u + (uint32_t)(col / PF_KC) * PF_A_CHUNK_BYTES + (uint32_t)(col & 3) * 4u;
                const int c16 = (col % PF_KC) >> 2;
                const float ov[4] = {o0, o1, o2, o3};
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t addr = base + sw128_off(prow + 8 * h, c16);
                    const uint32_t h0 = to_tf32(ov[2 * h]), h1 = to_tf32(ov[2 * h + 1]);
                    const uint32_t l0 = to_tf32(ov[2 * h] - __uint_as_float(h0));
                    const uint32_t l1 = to_tf32(ov[2 * h + 1] - __uint_as_float(h1));
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(h0), "r"(h1) : "memory");
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr + PF_A_BYTES), "r"(l0), "r"(l1) : "memory");
                }
            }
        }
    } else {
        // max over the points: the thread's two rows, then the 8 row pairs of the warp (lanes with the same
        // lane % 4 hold the same columns); the 8 warps are folded after the last N-tile
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int col = 8 * j + cq;
            float m0 = fmaxf(fmaxf(acc[4 * j] + bs[col], 0.f), fmaxf(acc[4 * j + 2] + bs[col], 0.f));
            float m1 = fmaxf(fmaxf(acc[4 * j + 1] + bs[col + 1], 0.f), fmaxf(acc[4 * j + 3] + bs[col + 1], 0.f));
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
                m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
            }
            if (r == 0) {
                c.pool_s[c.warp * 256 + nt * NT + col] = m0;
                c.pool_s[c.warp * 256 + nt * NT + col + 1] = m1;
            }
        }
    }
}

template <bool BF16>
__global__ void __launch_bounds__(PF_THREADS, 1)
pointnet_fused_kernel(const PfArgs p, const __grid_constant__ CUtensorMap wmap,
                      const __grid_constant__ CUtensorMap xmap) {
    using C = PfCfg<BF16>;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((smem_u32(smem) & 1023u) != 0u) __trap();
    // [A operand][weight ring][input tiles 2 x 8 KB][bias][pool scratch]
    uint8_t* a_s = smem;
    uint8_t* w_s = a_s + C::A_BYTES;
    uint8_t* x_s = w_s + C::STAGES * C::STAGE_BYTES;
    float* bias_s = reinterpret_cast<float*>(x_s + 2 * PF_X_BYTES);
    float* pool_s = bias_s + PF_MAX_BIAS;  // [8 warps][256]
    __shared__ __align__(8) uint64_t bars[2 * PB_STAGES + 4];

    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const uint32_t bars_u = smem_u32(&bars[0]);
    auto w_full = [&](int s) { return bars_u + 8u * (uint32_t)s; };
    auto w_empty = [&](int s) { return bars_u + 8u * (uint32_t)(C::STAGES + s); };
    auto x_full = [&](int s) { return bars_u + 8u * (uint32_t)(2 * C::STAGES + s); };
    auto x_empty = [&](int s) { return bars_u + 8u * (uint32_t)(2 * C::STAGES + 2 + s); };

    if (t == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            mbar_init(w_full(s), 1);
            mbar_init(w_empty(s), PF_ACT_WARPS);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(x_full(s), 1);
            mbar_init(x_empty(s), PF_ACT_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    SPG_PDL_ENTRY();  // set-up above overlaps the previous kernel of the stream; global memory only below
    for (int i = t; i < p.n_bias; i += PF_THREADS) bias_s[i] = p.bias[i];
    __syncthreads();
    const uint32_t a_u = smem_u32(a_s), w_u = smem_u32(w_s), x_u = smem_u32(x_s);

    if (warp == PF_ACT_WARPS) {
        // ================================ TMA producer ================================
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
            uint32_t it = 0, ci = 0;
            for (int64_t b = blockIdx.x; b < p.B; b += gridDim.x, ++ci) {
                const int xb = ci & 1;
                mbar_wait(x_empty(xb), ((ci >> 1) & 1) ^ 1);
                mbar_expect_tx(x_full(xb), (uint32_t)(p.F * PF_ROWS * 4));
                pf_tma_2d(x_u + xb * PF_X_BYTES, &xmap, 0, (int)(b * p.F), x_full(xb));
                for (int l = 0; l < p.n_layers; ++l) {
                    const PfLayer& Ly = p.L[l];
                    const int ntile = Ly.N < PF_NT ? Ly.N : PF_NT;
                    for (int nt = 0; nt < Ly.N / ntile; ++nt)
                        for (int kc = 0; kc < Ly.K / C::KC; ++kc, ++it) {
                            const int s = it % C::STAGES;
                            mbar_wait(w_empty(s), ((it / C::STAGES) & 1) ^ 1);
                            const uint32_t dst = w_u + s * C::STAGE_BYTES;
                            if constexpr (BF16) {
                                mbar_expect_tx(w_full(s), (uint32_t)(ntile * 128));
                                // image rows of this layer: [kc*N + n], 128 bytes each; boxes of 32 rows
                                for (int sub = 0; sub < ntile / 32; ++sub)
                                    pf_tma_2d(dst + (uint32_t)(sub * 32 * 128), &wmap, 0,
                                              Ly.w_row + kc * Ly.N + nt * ntile + sub * 32, w_full(s));
                            } else {
                                mbar_expect_tx(w_full(s), (uint32_t)(2 * ntile * 128));
                                // image rows of this layer: [(kc*2 + half)*N + n]
                                for (int half = 0; half < 2; ++half)
                                    for (int sub = 0; sub < ntile / 32; ++sub)
                                        pf_tma_2d(dst + (uint32_t)(half * ntile + sub * 32) * 128u, &wmap, 0,
                                                  Ly.w_row + (kc * 2 + half) * Ly.N + nt * ntile + sub * 32, w_full(s));
                            }
                        }
                }
            }
        }
    } else if (warp < PF_ACT_WARPS) {
        // ======================= consumer warpgroups: 64 points each =======================
        PfCtx c;
        c.a_u = a_u; c.w_u = w_u; c.bars_u = bars_u; c.bias_s = bias_s; c.pool_s = pool_s;
        c.g = warp >> 2; c.warp = warp; c.lane = lane;
        const int tw = t & 127;
        const int row = c.g * 64 + (tw & 63), fh = tw >> 6;  // input point; features 16*fh .. 16*fh+15
        uint32_t it = 0, ci = 0;
        for (int64_t b = blockIdx.x; b < p.B; b += gridDim.x, ++ci) {
            // ---- input tile -> (xy transform) -> A chunk 0 (features, zero-padded to the chunk)
            const int xb = ci & 1;
            mbar_wait(x_full(xb), (ci >> 1) & 1);
            const float* xin = reinterpret_cast<const float*>(x_s + xb * PF_X_BYTES);
            float v[16];
#pragma unroll
            for (int f = 0; f < 16; ++f) v[f] = (fh == 0 && f < p.F) ? xin[f * PF_ROWS + row] : 0.f;
            __syncwarp();
            if (lane == 0) mbar_arrive(x_empty(xb));
            if (fh == 0 && p.T) {
                const float eye = p.add_eye ? 1.f : 0.f;
                const float t00 = p.T[b * 4 + 0] + eye, t01 = p.T[b * 4 + 1], t10 = p.T[b * 4 + 2],
                            t11 = p.T[b * 4 + 3] + eye;
                const float x0 = v[0], x1 = v[1];
                v[0] = fmaf(x0, t00, x1 * t10);  // row vector times T (pointnet.py:123)
                v[1] = fmaf(x0, t01, x1 * t11);
            }
            if constexpr (BF16) {
                // 64-element chunk: fh 0 writes 16-byte chunks 0-1 (features), fh 1 chunks 2-7 (zeros)
                if (fh == 0) {
#pragma unroll
                    for (int q = 0; q < 2; ++q)
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a_u + sw128_off(row, q)),
                                     "r"(pack_bf16x2(v[8 * q], v[8 * q + 1])), "r"(pack_bf16x2(v[8 * q + 2], v[8 * q + 3])),
                                     "r"(pack_bf16x2(v[8 * q + 4], v[8 * q + 5])), "r"(pack_bf16x2(v[8 * q + 6], v[8 * q + 7]))
                                     : "memory");
                } else {
#pragma unroll
                    for (int q = 2; q < 8; ++q)
                        asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(a_u + sw128_off(row, q)), "r"(0u)
                                     : "memory");
                }
            } else {
                // 32-float chunk: fh writes 16-byte chunks 4*fh .. 4*fh+3, hi and lo
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    uint32_t hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        hi[e] = to_tf32(v[4 * q + e]);
                        lo[e] = to_tf32(v[4 * q + e] - __uint_as_float(hi[e]));
                    }
                    const uint32_t addr = a_u + sw128_off(row, 4 * fh + q);
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(hi[0]), "r"(hi[1]),
                                 "r"(hi[2]), "r"(hi[3]) : "memory");
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr + PF_A_BYTES), "r"(lo[0]),
                                 "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            bar_named(1 + c.g, 128);
            // ---- layers
            for (int l = 0; l < p.n_layers; ++l) {
                const PfLayer& Ly = p.L[l];
                const int ntile = Ly.N < PF_NT ? Ly.N : PF_NT;
                const bool last = l + 1 == p.n_layers;
                for (int nt = 0; nt < Ly.N / ntile; ++nt) {
                    if (ntile == 128) pf_tile<BF16, 128>(c, Ly, nt, last, it);
                    else if (ntile == 64) pf_tile<BF16, 64>(c, Ly, nt, last, it);
                    else pf_tile<BF16, 32>(c, Ly, nt, last, it);
                }
                if (!last) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    bar_named(1 + c.g, 128);
                } else {
                    bar_named(3, PF_ACT_WARPS * 32);
                    for (int col = t; col < Ly.N; col += PF_ACT_WARPS * 32) {
                        float m = pool_s[col];
#pragma unroll
                        for (int w = 1; w < PF_ACT_WARPS; ++w) m = fmaxf(m, pool_s[w * 256 + col]);
                        p.pooled[b * p.ldp + col] = m;
                    }
                    bar_named(3, PF_ACT_WARPS * 32);
                }
            }
        }
    }
}

// bf16 weight image of diag(row_scale) * W: for every 64-element K chunk [N rows][128 B], SWIZZLE_128B
__global__ void pack_weights_bf16_kernel(const float* __restrict__ W, int64_t ldw,
                                         const float* __restrict__ row_scale, int N, int K, int k_valid,
                                         uint16_t* __restrict__ img) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * K) return;
    const int n = (int)(i / K), k = (int)(i % K);
    float v = 0.f;
    if (k < k_valid) v = W[(int64_t)n * ldw + k] * (row_scale ? row_scale[n] : 1.f);
    const uint32_t pk = pack_bf16x2(v, 0.f);
    const int kc = k / PB_KC, kk = k % PB_KC;
    img[(int64_t)kc * N * PB_KC + (sw128_off(n, kk >> 3) >> 1) + (kk & 7)] = (uint16_t)(pk & 0xffffu);
}

typedef CUresult (*PfEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                               const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PfEncodeFn pf_encode() {
    static PfEncodeFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PfEncodeFn>(ptr);
    });
    return fn;
}

static int pf_map_2d(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint32_t box_cols,
                     uint32_t box_rows, bool bf16 = false) {
    PfEncodeFn fn = pf_encode();
    if (!fn) return SPG_E_UNSUPPORTED;
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {cols * (bf16 ? 2 : 4)};
    const cuuint32_t box[2] = {box_cols, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                          const_cast<void*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SPG_OK : SPG_E_BADARG;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_pointnet_fused_supported(int n_features, int n_points, int n_layers, const int32_t* widths) {
    if (n_points != PF_ROWS || n_features < 1 || n_features > PF_MAXF) return 0;
    if (n_layers < 1 || n_layers > PF_MAX_LAYERS || !widths) return 0;
    int total = 0;
    for (int l = 0; l < n_layers; ++l) {
        const int n = widths[l];
        if (n != 32 && n != 64 && n != 128 && n != 256) return 0;
        if (l + 1 < n_layers && n > PF_MAXK) return 0;  // a layer's output is the next layer's K
        total += n;
    }
    return total <= PF_MAX_BIAS ? 1 : 0;
}

int64_t spg_pointnet_fused_image_rows(int n_features, int n_layers, const int32_t* widths) {
    (void)n_features;
    int64_t rows = 0;
    int k = PF_KC;  // first layer: features padded to one chunk
    for (int l = 0; l < n_layers; ++l) {
        rows += (int64_t)(k / PF_KC) * 2 * widths[l];
        k = widths[l];
    }
    return rows;
}

int spg_pointnet_fused_eval(const float* clouds, int64_t n_clouds, int n_features, int n_points, const float* T,
                            int add_eye, const float* weight_image, const float* bias, int n_layers,
                            const int32_t* widths, float* pooled, int64_t ldp, spg_stream_t stream) {
    if (n_clouds < 0 || !widths) return SPG_E_BADARG;
    if (!spg_pointnet_fused_supported(n_features, n_points, n_layers, widths)) return SPG_E_UNSUPPORTED;
    if (n_clouds == 0) return SPG_OK;
    if (!clouds || !weight_image || !bias || !pooled || ldp < widths[n_layers - 1]) return SPG_E_BADARG;
    if (T && n_features < 2) return SPG_E_BADARG;  // the transform acts on the (x, y) features
    if (((uintptr_t)clouds | (uintptr_t)weight_image) & 15) return SPG_E_ALIGN;
    if (n_clouds * n_features >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    PfArgs a;
    a.n_layers = n_layers;
    int k = PF_KC, row = 0, boff = 0;
    for (int l = 0; l < n_layers; ++l) {
        a.L[l].K = k;
        a.L[l].N = widths[l];
        a.L[l].w_row = row;
        a.L[l].b_off = boff;
        row += (k / PF_KC) * 2 * widths[l];
        boff += widths[l];
        k = widths[l];
    }
    a.F = n_features; a.B = n_clouds; a.T = T; a.add_eye = add_eye; a.bias = bias; a.n_bias = boff;
    a.pooled = pooled; a.ldp = ldp;
    CUtensorMap wmap, xmap;
    int rc = pf_map_2d(&wmap, weight_image, PF_KC, (uint64_t)row, PF_KC, 32);
    if (rc) return rc;
    rc = pf_map_2d(&xmap, clouds, PF_ROWS, (uint64_t)(n_clouds * n_features), PF_ROWS, (uint32_t)n_features);
    if (rc) return rc;
    const int64_t grid = n_clouds < kNumSMs ? n_clouds : kNumSMs;
    const int smem = PfCfg<false>::SMEM;
    cudaError_t e = cudaFuncSetAttribute(pointnet_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_POINTNET_FUSED, (cudaStream_t)stream, pointnet_fused_kernel<false>, (unsigned)grid, PF_THREADS, smem,
               a, wmap, xmap);
    return launch_status();
}

/* bf16 twins (spg_b200.h): K chunks of 64 elements; a 32-wide layer is followed by a zero-padded chunk */
int64_t spg_pointnet_fused_bf16_image_rows(int n_features, int n_layers, const int32_t* widths) {
    (void)n_features;
    int64_t rows = 0;
    int k = PB_KC;
    for (int l = 0; l < n_layers; ++l) {
        rows += (int64_t)(k / PB_KC) * widths[l];
        k = widths[l] < PB_KC ? PB_KC : widths[l];
    }
    return rows;
}

int spg_tc_pack_weights_bf16(const float* W, int64_t ldw, const float* row_scale, int N, int K, int k_valid,
                             void* image, spg_stream_t stream) {
    if (!W || !image || N <= 0 || K <= 0 || k_valid <= 0 || k_valid > K) return SPG_E_BADARG;
    if (K % PB_KC != 0 || N % 8 != 0) return SPG_E_UNSUPPORTED;
    const int64_t total = (int64_t)N * K;
    SPG_LAUNCH(K_TC_PACK, (cudaStream_t)stream, pack_weights_bf16_kernel, (unsigned)ceil_div64(total, 256), 256, 0, W,
               ldw, row_scale, N, K, k_valid, (uint16_t*)image);
    return launch_status();
}

int spg_pointnet_fused_eval_bf16(const float* clouds, int64_t n_clouds, int n_features, int n_points, const float* T,
                                 int add_eye, const void* weight_image, const float* bias, int n_layers,
                                 const int32_t* widths, float* pooled, int64_t ldp, spg_stream_t stream) {
    if (n_clouds < 0 || !widths) return SPG_E_BADARG;
    if (!spg_pointnet_fused_supported(n_features, n_points, n_layers, widths)) return SPG_E_UNSUPPORTED;
    if (n_clouds == 0) return SPG_OK;
    if (!clouds || !weight_image || !bias || !pooled || ldp < widths[n_layers - 1]) return SPG_E_BADARG;
    if (T && n_features < 2) return SPG_E_BADARG;  // the transform acts on the (x, y) features
    if (((uintptr_t)clouds | (uintptr_t)weight_image) & 15) return SPG_E_ALIGN;
    if (n_clouds * n_features >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    PfArgs a;
    a.n_layers = n_layers;
    int k = PB_KC, row = 0, boff = 0;
    for (int l = 0; l < n_layers; ++l) {
        a.L[l].K = k;
        a.L[l].N = widths[l];
        a.L[l].w_row = row;
        a.L[l].b_off = boff;
        row += (k / PB_KC) * widths[l];
        boff += widths[l];
        k = widths[l] < PB_KC ? PB_KC : widths[l];
    }
    a.F = n_features; a.B = n_clouds; a.T = T; a.add_eye = add_eye; a.bias = bias; a.n_bias = boff;
    a.pooled = pooled; a.ldp = ldp;
    CUtensorMap wmap, xmap;
    int rc = pf_map_2d(&wmap, weight_image, PB_KC, (uint64_t)row, PB_KC, 32, true);
    if (rc) return rc;
    rc = pf_map_2d(&xmap, clouds, PF_ROWS, (uint64_t)(n_clouds * n_features), PF_ROWS, (uint32_t)n_features);
    if (rc) return rc;
    const int64_t grid = n_clouds < kNumSMs ? n_clouds : kNumSMs;
    const int smem = PfCfg<true>::SMEM;
    cudaError_t e = cudaFuncSetAttribute(pointnet_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_POINTNET_FUSED, (cudaStream_t)stream, pointnet_fused_kernel<true>, (unsigned)grid, PF_THREADS, smem, a,
               wmap, xmap);
    return launch_status();
}

}  // extern "C"
