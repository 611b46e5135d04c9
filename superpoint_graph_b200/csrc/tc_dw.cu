// Hopper (wgmma) weight-gradient GEMM of the point-wise layers:
//
//     dW[Co, Ci] = sum_m dY[m, Co] * f(P)[m, Ci]        (m runs over all Nv*L points)
//
// Both operands lie in HBM point-major (channels contiguous), i.e. the reduction dimension is the OUTER
// one.  wgmma reads tf32 operands K-major only, so the CTA transposes while it stages: it owns a
// contiguous slab of points and streams it in chunks of 32 points (one 128-byte SWIZZLE_128B row per
// channel) through a shared-memory ring, splitting every value into tf32 hi/lo on the fly (3xTF32,
// fp32-equivalent).  The CTA is warp-specialised, one CTA per SM:
//
//   warps 0-7   consumers: two warpgroups keep the [Co, Ci] accumulator in registers for the CTA's whole
//               lifetime (Co >= 128: half of the rows each; Co = 64: half of the columns each).  Per chunk
//               they wait on the stage's `full` mbarrier, issue its wgmmas, and hand the previous stage
//               back on its `empty` mbarrier once that chunk's wgmma group has completed.  Finally they
//               write one partial per CTA; gemm_splitk_reduce adds the partials in a fixed order
//               (deterministic).
//   warps 8-11  producers: coalesced 128-bit loads into a register ring of PF chunks per thread, f = affine
//               + ReLU of the layer that produced P (fused), hi/lo split, transposed stores into the ring.
//
// 384 threads leave every thread 168 registers, which the (256,128) consumers need for their 128-float
// accumulator; one producer warpgroup transposes a chunk in less time than the tensor cores or HBM take
// for it at every shape.
//
// Loads in flight.  A chunk is 128*(Co+Ci) bytes (12..48 KB).  A producer thread keeps up to 96 operand
// floats in its register ring: PF = 4 chunks at (64,32) down to ONE chunk from (128,128) on; there the
// next chunk's loads are issued as soon as the chunk's registers have been transposed, and fly while
// the thread waits for its stage to be released.  Two K-major stages of (256,128) (2 x 96 KB) leave no
// shared memory to stage raw chunks in instead.  Asking for the chunks behind the ring with
// cp.async.bulk.prefetch.L2 (one row per lane) was measured and made every shape 10-30 % slower.
//
// The chunk order, the order of the wgmmas into the accumulator, the split and the partial format are
// what determines the result; who moves the bytes and when does not.
//
// Reference semantics: the weight gradient of nn.Conv1d(k=1) (learning/pointnet.py:29,85) as
// autograd computes it; the reference materialises ReLU(BN(P)) and runs cuDNN/cuBLAS on it.
#include "common.cuh"
#include "tc_common.cuh"

namespace spg {

constexpr int DW_CONS_WARPS = 8, DW_PROD_WARPS = 4;
constexpr int DW_PROD_THREADS = DW_PROD_WARPS * 32;
constexpr int DW_THREADS = (DW_CONS_WARPS + DW_PROD_WARPS) * 32;  // 384
constexpr int DW_PTS = 32;  // points per chunk (4 wgmma K-steps of 8)
constexpr int DW_MAX_STAGES = 4;
constexpr int DW_SMEM_LIMIT = 232448;                  // 227 KB per CTA
constexpr int DW_STATIC_SMEM = 2048;  // prologue vectors + mbarriers, padded to the dynamic segment's alignment

template <int CO, int CI>
struct DwCfg {
    static constexpr int A_BYTES = CO * DW_PTS * 4;  // one of hi|lo: [CO rows][128 B]
    static constexpr int B_BYTES = CI * DW_PTS * 4;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
    static constexpr int FIT = (DW_SMEM_LIMIT - 1024 - DW_STATIC_SMEM) / STAGE_BYTES;
    static constexpr int STAGES = FIT < DW_MAX_STAGES ? FIT : DW_MAX_STAGES;
    static constexpr int SMEM = STAGES * STAGE_BYTES + 1024;  // + round-up to the 1024-byte swizzle atom
    static constexpr int A_F4 = CO * DW_PTS / 4 / DW_PROD_THREADS;  // float4 per producer thread per chunk
    static constexpr int B_F4 = CI * DW_PTS / 4 / DW_PROD_THREADS;
    // register ring: at most 24 float4 (96 registers) of operands per producer thread
    static constexpr int PF_FIT = 24 / (A_F4 + B_F4);
    static constexpr int PF = PF_FIT < 1 ? 1 : (PF_FIT > 4 ? 4 : PF_FIT);
    static_assert(STAGES >= 2, "ring");
};

struct DwArgs {
    const float* dY;
    int64_t lddy;
    const float* P;
    int64_t ldp;
    const float *p_scale, *p_shift;
    int p_relu;
    float* partial;  // [gridDim.x, CO, CI]
    int64_t M;
    int64_t pts_per_cta;  // multiple of DW_PTS
};

template <int CO, int CI>
__global__ void __launch_bounds__(DW_THREADS, 1) tc_dw_kernel(const DwArgs p) {
    using Cfg = DwCfg<CO, CI>;
    constexpr int WM = CO >= 128 ? CO / 2 : 64;  // accumulator rows of one warpgroup
    constexpr int WN = CO >= 128 ? CI : CI / 2;  // accumulator columns of one warpgroup
    constexpr int MSUB = WM / 64;                 // m64 sub-tiles
    constexpr int A_BYTES = Cfg::A_BYTES, B_BYTES = Cfg::B_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
    constexpr int STAGES = Cfg::STAGES, PF = Cfg::PF, A_F4 = Cfg::A_F4, B_F4 = Cfg::B_F4;
    static_assert(CO % 64 == 0 && CI % 32 == 0 && CI <= 128 && CO <= 256, "shape");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    __shared__ __align__(8) uint64_t bars[2 * DW_MAX_STAGES];
    __shared__ __align__(16) float sc_s[128], sh_s[128];
    static_assert(sizeof(bars) + sizeof(sc_s) + sizeof(sh_s) <= DW_STATIC_SMEM, "static shared memory");

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const uint32_t bars_u32 = smem_u32(&bars[0]);
    auto bar_full = [&](int s) { return bars_u32 + 8u * (uint32_t)s; };
    auto bar_empty = [&](int s) { return bars_u32 + 8u * (uint32_t)(DW_MAX_STAGES + s); };
    if (t == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full(s), DW_PROD_WARPS);   // one elected arrival per producer warp
            mbar_init(bar_empty(s), DW_CONS_WARPS);  // one elected arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // The barrier init above overlaps the previous kernel of the stream; nothing below this line runs
    // before that kernel's results are visible.
    SPG_PDL_ENTRY();

    const int64_t m_beg = (int64_t)blockIdx.x * p.pts_per_cta;
    const int64_t m_end = min(p.M, m_beg + p.pts_per_cta);
    const int nchunks = m_beg < m_end ? (int)((m_end - m_beg + DW_PTS - 1) / DW_PTS) : 0;

    // Producer thread i handles the float4s (point pt, channels 4*c4..4*c4+3) with c4 = c40 + 4*j: a warp
    // covers 8 points x 4 channel groups, so that its 64-byte row segments are whole sectors and its
    // transposed 4-byte shared-memory stores spread over 16 banks (2-way conflict).
    const int ptid = t - DW_CONS_WARPS * 32;  // producer thread id 0..127 (negative: consumers)
    const int pt = (ptid >> 5) * 8 + (lane & 7), c40 = lane >> 3;
    float4 q[PF][A_F4 + B_F4];
    // rows >= m_end (the ragged last chunk, and every chunk past the slab) read as zeros
    auto load_chunk = [&](int ch, float4 (&dst)[A_F4 + B_F4]) {
        const int64_t row = m_beg + (int64_t)ch * DW_PTS + pt;
        const bool ok = row < m_end;
        const float4* ga = reinterpret_cast<const float4*>(p.dY + row * p.lddy) + c40;
        const float4* gb = reinterpret_cast<const float4*>(p.P + row * p.ldp) + c40;
#pragma unroll
        for (int j = 0; j < A_F4; ++j) dst[j] = ok ? __ldg(ga + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < B_F4; ++j) dst[A_F4 + j] = ok ? __ldg(gb + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    // Producers put their first chunks in flight before anything else.
    if (ptid >= 0) {
#pragma unroll
        for (int d = 0; d < PF; ++d) load_chunk(d, q[d]);
    }
    if (t < CI) {
        sc_s[t] = p.p_scale ? p.p_scale[t] : 1.f;
        sh_s[t] = p.p_shift ? p.p_shift[t] : 0.f;
    }
    __syncthreads();

    if (warp >= DW_CONS_WARPS) {
        // ================================ producers ================================
        const bool pro = p.p_scale || p.p_shift || p.p_relu;
        // (point pt, channel 4*c40 + e) -> K-major row 4*c40 + e, element pt of its 128-byte row; the
        // channels 16*j further on lie two 8-row swizzle atoms (2048 bytes) further on
        uint32_t soff[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) soff[e] = sw128_off(4 * c40 + e, pt >> 2) + (uint32_t)(pt & 3) * 4u;
        auto st_shared = [](uint32_t addr, uint32_t v) {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
        };
        // hi image at stage + hi_off, lo image `lo` bytes behind it
        auto split_store = [&](const uint32_t (&base)[4], uint32_t hi_off, uint32_t lo, int j, float4 v) {
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const uint32_t addr = base[e] + hi_off + 2048u * (uint32_t)j;
                const uint32_t hi = to_tf32(vv[e]);
                st_shared(addr, hi);
                st_shared(addr + lo, to_tf32(vv[e] - __uint_as_float(hi)));
            }
        };
        const uint32_t smem_u = smem_u32(smem);
        int ch = 0, s = 0;
        uint32_t use = 0;  // how many times the ring has wrapped
        auto produce = [&](float4 (&cur)[A_F4 + B_F4]) {
            if (use > 0) mbar_wait(bar_empty(s), (use - 1) & 1);
            uint32_t base[4];  // stage layout: A hi | A lo | B hi | B lo
#pragma unroll
            for (int e = 0; e < 4; ++e) base[e] = smem_u + (uint32_t)s * STAGE_BYTES + soff[e];
            const bool affine = pro && m_beg + (int64_t)ch * DW_PTS + pt < m_end;
#pragma unroll
            for (int j = 0; j < A_F4; ++j) split_store(base, 0u, A_BYTES, j, cur[j]);
#pragma unroll
            for (int j = 0; j < B_F4; ++j) {
                float4 v = cur[A_F4 + j];
                if (affine) {
                    const float4 sc = *reinterpret_cast<const float4*>(sc_s + (c40 + 4 * j) * 4);
                    const float4 sh = *reinterpret_cast<const float4*>(sh_s + (c40 + 4 * j) * 4);
                    v.x = fmaf(v.x, sc.x, sh.x);
                    v.y = fmaf(v.y, sc.y, sh.y);
                    v.z = fmaf(v.z, sc.z, sh.z);
                    v.w = fmaf(v.w, sc.w, sh.w);
                    if (p.p_relu) {
                        v.x = fmaxf(v.x, 0.f);
                        v.y = fmaxf(v.y, 0.f);
                        v.z = fmaxf(v.z, 0.f);
                        v.w = fmaxf(v.w, 0.f);
                    }
                }
                split_store(base, 2 * A_BYTES, B_BYTES, j, v);
            }
            load_chunk(ch + PF, cur);  // the registers are free again: PF chunks stay in flight
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_full(s));
            ++ch;
            if (++s == STAGES) {
                s = 0;
                ++use;
            }
        };
        while (ch < nchunks) {
#pragma unroll
            for (int u = 0; u < PF; ++u) {
                produce(q[u]);
                if (ch >= nchunks) break;
            }
        }
    } else {
        // ================================ consumers ================================
        const int g = warp >> 2, wl = warp & 3;
        float acc[MSUB][WN / 2];
#pragma unroll
        for (int m = 0; m < MSUB; ++m)
#pragma unroll
            for (int i = 0; i < WN / 2; ++i) acc[m][i] = 0.f;
        const int row_g = CO >= 128 ? g * WM : 0;  // first accumulator row / column of this warpgroup
        const int col_g = CO >= 128 ? 0 : g * WN;
        const uint32_t smem_u = smem_u32(smem);

        int s = 0, s_prev = 0;
        uint32_t phase = 0;
        for (int ch = 0; ch < nchunks; ++ch) {
            mbar_wait(bar_full(s), phase);
            const uint32_t a_hi = smem_u + (uint32_t)s * STAGE_BYTES;
            const uint32_t ah = a_hi + (uint32_t)row_g * 128u, al = ah + A_BYTES;
            const uint32_t bh = a_hi + 2 * A_BYTES + (uint32_t)col_g * 128u, bl = bh + B_BYTES;
#pragma unroll
            for (int m = 0; m < MSUB; ++m) wg_reg_fence(acc[m]);
            wg_fence();
#pragma unroll
            for (int kb = 0; kb < DW_PTS / 8; ++kb) {
                const uint64_t dbh = wg_desc_k_sw128(bh + kb * 32), dbl = wg_desc_k_sw128(bl + kb * 32);
#pragma unroll
                for (int m = 0; m < MSUB; ++m) {
                    const uint64_t dah = wg_desc_k_sw128(ah + m * 64 * 128 + kb * 32);
                    const uint64_t dal = wg_desc_k_sw128(al + m * 64 * 128 + kb * 32);
                    wgmma_tf32<WN>(acc[m], dah, dbh, 1u);
                    wgmma_tf32<WN>(acc[m], dal, dbh, 1u);
                    wgmma_tf32<WN>(acc[m], dah, dbl, 1u);
                }
            }
            wg_commit();
            if (ch > 0) {
                // the products of chunk ch-1 have completed in this warpgroup: its stage may be refilled
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty(s_prev));
            }
            s_prev = s;
            if (++s == STAGES) {
                s = 0;
                phase ^= 1u;
            }
        }
        wg_wait<0>();
#pragma unroll
        for (int m = 0; m < MSUB; ++m) wg_reg_fence(acc[m]);

        // ---- epilogue: accumulator -> this CTA's partial [CO, CI] (zeros when the CTA got no points)
        float* out = p.partial + (int64_t)blockIdx.x * CO * CI;
        const int r = lane >> 2, cq = 2 * (lane & 3);
#pragma unroll
        for (int m = 0; m < MSUB; ++m) {
            const int row = row_g + m * 64 + wl * 16 + r;
#pragma unroll
            for (int j = 0; j < WN / 8; ++j) {
                const int col = col_g + 8 * j + cq;
                *reinterpret_cast<float2*>(out + (int64_t)row * CI + col) =
                    make_float2(acc[m][4 * j], acc[m][4 * j + 1]);
                *reinterpret_cast<float2*>(out + (int64_t)(row + 8) * CI + col) =
                    make_float2(acc[m][4 * j + 2], acc[m][4 * j + 3]);
            }
        }
    }
}

template <int CO, int CI>
static int launch_dw(const DwArgs& a, int ctas, cudaStream_t s) {
    constexpr int smem = DwCfg<CO, CI>::SMEM;
    cudaError_t e = cudaFuncSetAttribute(tc_dw_kernel<CO, CI>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_TC_DW, s, (tc_dw_kernel<CO, CI>), (unsigned)ctas, DW_THREADS, smem, a);
    return launch_status();
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_tc_dw_supported(int64_t M, int co, int ci) {
    const bool co_ok = (co == 64 || co == 128 || co == 256);
    const bool ci_ok = (ci == 32 || ci == 64 || ci == 128);
    return (M >= DW_PTS && co_ok && ci_ok) ? 1 : 0;
}

int spg_tc_dw_ctas(int64_t M) {
    int64_t chunks = ceil_div64(M, DW_PTS);
    int64_t ctas = chunks < kNumSMs ? chunks : kNumSMs;
    return (int)(ctas < 1 ? 1 : ctas);
}

int spg_tc_dw(const float* dY, int64_t lddy, const float* P, int64_t ldp, const float* p_scale,
              const float* p_shift, int p_relu, float* dW, float* workspace, int64_t M, int co, int ci,
              spg_stream_t stream) {
    if (!dY || !P || !dW || !workspace || M <= 0) return SPG_E_BADARG;
    if (!spg_tc_dw_supported(M, co, ci)) return SPG_E_UNSUPPORTED;
    if ((lddy & 3) || (ldp & 3) || lddy < co || ldp < ci) return SPG_E_ALIGN;
    if (((uintptr_t)dY | (uintptr_t)P | (uintptr_t)workspace | (uintptr_t)p_scale | (uintptr_t)p_shift) & 15)
        return SPG_E_ALIGN;
    const int ctas = spg_tc_dw_ctas(M);
    DwArgs a;
    a.dY = dY; a.lddy = lddy; a.P = P; a.ldp = ldp; a.p_scale = p_scale; a.p_shift = p_shift;
    a.p_relu = p_relu; a.partial = workspace; a.M = M;
    cudaStream_t s = (cudaStream_t)stream;
    a.pts_per_cta = ceil_div64(ceil_div64(M, ctas), DW_PTS) * DW_PTS;
    int rc;
#define SPG_DW_CASE(CO_, CI_) \
    if (co == CO_ && ci == CI_) rc = launch_dw<CO_, CI_>(a, ctas, s); else
    SPG_DW_CASE(64, 32) SPG_DW_CASE(64, 64) SPG_DW_CASE(64, 128) SPG_DW_CASE(128, 32)
    SPG_DW_CASE(128, 64) SPG_DW_CASE(128, 128) SPG_DW_CASE(256, 32) SPG_DW_CASE(256, 64)
    SPG_DW_CASE(256, 128) rc = SPG_E_UNSUPPORTED;
#undef SPG_DW_CASE
    if (rc) return rc;
    return spg_splitk_reduce(workspace, ctas, co, ci, nullptr, dW, ci, stream);
}

}  // extern "C"
