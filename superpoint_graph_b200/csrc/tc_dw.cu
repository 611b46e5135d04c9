// Hopper (wgmma) weight-gradient GEMM of the point-wise layers:
//
//     dW[Co, Ci] = sum_m dY[m, Co] * f(P)[m, Ci]        (m runs over all Nv*L points)
//
// Both operands lie in HBM point-major (channels contiguous), i.e. the reduction dimension is the OUTER
// one.  The CTA owns a contiguous slab of points and streams it in chunks of 32 points (four wgmma K-steps
// of 8), splitting every value into tf32 hi/lo (3xTF32, fp32-equivalent).  The A operand, dY^T, goes to
// the tensor cores from registers: a register fragment can be gathered in any order, so dY needs no
// transpose and never touches shared memory.  wgmma reads a shared-memory tf32 operand K-major only, so
// B, f(P)^T, is transposed into a SWIZZLE_128B ring (one 128-byte row per channel and chunk).  The CTA is
// warp-specialised, one CTA per SM:
//
//   warps 0-7   consumers: two warpgroups keep the [Co, Ci] accumulator in registers for the CTA's whole
//               lifetime (Co >= 128: half of the rows each; Co = 64: half of the columns each, both reading
//               the same 64 rows of dY).  Each thread loads its own A fragments straight from dY (one 8- or
//               16-byte load per point and K-step), RAW K-steps ahead of their use, and splits
//               them into one of HL hi/lo register buffers, after the wgmma group that last read that buffer
//               has completed.  Per chunk they wait on the stage's `full` mbarrier, issue one wgmma group
//               per K-step, and hand the previous chunk's stage back on its `empty` mbarrier once its last
//               group has completed.  Finally they write one partial per CTA; gemm_splitk_reduce adds the
//               partials in a fixed order (deterministic).
//   warps 8-11  producers: coalesced 128-bit loads of P into a register ring of PF chunks per thread,
//               f = affine + ReLU of the layer that produced P (fused), hi/lo split, transposed stores into
//               the ring.
//
// 384 threads leave every thread 168 registers; the (256,128) consumers hold a 128-float accumulator plus
// their A fragments and take more with setmaxnreg from the producers, which then keep one chunk in flight.
//
// The chunk order, the order of the wgmmas into the accumulator (per K-step and m64 sub-tile: hi*hi,
// lo*hi, hi*lo), the split and the partial format are what determines the result; who moves the bytes,
// from where and when does not.
//
// Reference semantics: the weight gradient of nn.Conv1d(k=1) (learning/pointnet.py:29,85) as
// autograd computes it; the reference materialises ReLU(BN(P)) and runs cuDNN/cuBLAS on it.
#include "common.cuh"
#include "tc_common.cuh"

#include <type_traits>

namespace spg {

constexpr int DW_CONS_WARPS = 8, DW_PROD_WARPS = 4;
constexpr int DW_PROD_THREADS = DW_PROD_WARPS * 32;
constexpr int DW_THREADS = (DW_CONS_WARPS + DW_PROD_WARPS) * 32;  // 384
constexpr int DW_PTS = 32;  // points per chunk
constexpr int DW_KSTEPS = DW_PTS / 8;  // wgmma K-steps per chunk
constexpr int DW_STAGES = 4;
constexpr int DW_SMEM_LIMIT = 232448;                  // 227 KB per CTA
constexpr int DW_STATIC_SMEM = 2048;  // prologue vectors + mbarriers, padded to the dynamic segment's alignment

template <int CO, int CI>
struct DwCfg {
    static constexpr int WM = CO >= 128 ? CO / 2 : 64;  // accumulator rows of one warpgroup
    static constexpr int WN = CO >= 128 ? CI : CI / 2;  // accumulator columns of one warpgroup
    static constexpr int MSUB = WM / 64;                 // m64 sub-tiles
    static constexpr int B_BYTES = CI * DW_PTS * 4;  // one of hi|lo: [CI rows][128 B]
    static constexpr int STAGE_BYTES = 2 * B_BYTES;
    static constexpr int SMEM = DW_STAGES * STAGE_BYTES + 1024;  // + round-up to the 1024-byte swizzle atom
    static_assert(SMEM + DW_STATIC_SMEM <= DW_SMEM_LIMIT, "ring");
    static constexpr int B_F4 = CI * DW_PTS / 4 / DW_PROD_THREADS;  // float4 per producer thread per chunk
    // Only the (256,128) consumers outgrow 168 registers: 128 accumulator + 16 hi/lo + 8 raw A per K-step.
    // They take 224 each from the producers, which keep 56 and so one chunk (32 registers) in flight (with
    // fewer consumer registers ptxas serialises the wgmmas).
    static constexpr bool REG_SPLIT = WM * WN > 128 * 64;
    static constexpr int CONS_REGS = 224, PROD_REGS = 56;  // 2 * 224 + 56 = 3 * 168
    // producer register ring: at most 24 float4 (96 registers) per thread
    static constexpr int PF_FIT = REG_SPLIT ? 1 : 24 / B_F4;
    static constexpr int PF = PF_FIT < 1 ? 1 : (PF_FIT > 4 ? 4 : PF_FIT);
    // consumer A fragments: HL hi/lo buffers of one K-step (8 * MSUB registers each), RAW K-steps of raw
    // values (4 * MSUB registers each) in flight.  One m64 sub-tile loads two chunks ahead: at the small
    // shapes a chunk takes less time than a load's latency, so one chunk ahead leaves too few bytes in
    // flight.
    static constexpr int HL = WN * MSUB <= 64 ? 4 : 2;
    static constexpr int RAW = MSUB == 1 ? 2 * DW_KSTEPS : 2;
    static_assert(DW_KSTEPS % HL == 0 && (DW_KSTEPS % RAW == 0 || RAW == 2 * DW_KSTEPS), "A fragment rings");
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
    constexpr int WM = Cfg::WM, WN = Cfg::WN, MSUB = Cfg::MSUB;
    constexpr int B_BYTES = Cfg::B_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
    constexpr int PF = Cfg::PF, B_F4 = Cfg::B_F4, HL = Cfg::HL, RAW = Cfg::RAW;
    static_assert(CO % 64 == 0 && CI % 32 == 0 && CI <= 128 && CO <= 256, "shape");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    __shared__ __align__(8) uint64_t bars[2 * DW_STAGES];
    __shared__ __align__(16) float sc_s[128], sh_s[128];
    static_assert(sizeof(bars) + sizeof(sc_s) + sizeof(sh_s) <= DW_STATIC_SMEM, "static shared memory");

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const uint32_t bars_u32 = smem_u32(&bars[0]);
    auto bar_full = [&](int s) { return bars_u32 + 8u * (uint32_t)s; };
    auto bar_empty = [&](int s) { return bars_u32 + 8u * (uint32_t)(DW_STAGES + s); };
    if (t == 0) {
#pragma unroll
        for (int s = 0; s < DW_STAGES; ++s) {
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
    float4 q[PF][B_F4];
    // rows >= m_end (the ragged last chunk, and every chunk past the slab) read as zeros
    auto load_chunk = [&](int ch, float4 (&dst)[B_F4]) {
        const int64_t row = m_beg + (int64_t)ch * DW_PTS + pt;
        const bool ok = row < m_end;
        const float4* gb = reinterpret_cast<const float4*>(p.P + row * p.ldp) + c40;
#pragma unroll
        for (int j = 0; j < B_F4; ++j) dst[j] = ok ? __ldg(gb + 4 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    // Which Co an accumulator row stands for is free, as long as the epilogue writes it there.  Consumer
    // thread (warpgroup g, warp wl, lane l) holds fragment rows 64m + 16wl + l/4 (+8); they stand for the
    // 2*MSUB consecutive Co a_co + 2m (+1), so that per K-step point (l%4, l%4 + 4) the thread reads them
    // with one 8- or 16-byte load (per warp instruction 4 points x 64 or 128 bytes, whole sectors).
    const int g = warp >> 2, wl = warp & 3;
    const int a_co = (CO >= 128 ? g * WM : 0) + (wl * 8 + (lane >> 2)) * 2 * MSUB;
    float a_raw[RAW][MSUB][4];
    auto load_a = [&](int kstep, float (&dst)[MSUB][4]) {
        const int64_t i0 = m_beg + (int64_t)kstep * 8 + (lane & 3);
        const bool ok0 = i0 < m_end, ok1 = i0 + 4 < m_end;
        const float* y0 = p.dY + i0 * p.lddy + a_co;
        const float* y1 = y0 + 4 * p.lddy;
        if constexpr (MSUB == 1) {
            const float2 v0 = ok0 ? __ldg(reinterpret_cast<const float2*>(y0)) : make_float2(0.f, 0.f);
            const float2 v1 = ok1 ? __ldg(reinterpret_cast<const float2*>(y1)) : make_float2(0.f, 0.f);
            dst[0][0] = v0.x; dst[0][1] = v0.y; dst[0][2] = v1.x; dst[0][3] = v1.y;
        } else {
            static_assert(MSUB == 2, "A fragment loads");
            const float4 v0 = ok0 ? __ldg(reinterpret_cast<const float4*>(y0)) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 v1 = ok1 ? __ldg(reinterpret_cast<const float4*>(y1)) : make_float4(0.f, 0.f, 0.f, 0.f);
            dst[0][0] = v0.x; dst[0][1] = v0.y; dst[1][0] = v0.z; dst[1][1] = v0.w;
            dst[0][2] = v1.x; dst[0][3] = v1.y; dst[1][2] = v1.z; dst[1][3] = v1.w;
        }
    };
    // Everyone puts its first loads in flight before anything else.
    if (ptid >= 0) {
#pragma unroll
        for (int d = 0; d < PF; ++d) load_chunk(d, q[d]);
    } else {
#pragma unroll
        for (int j = 0; j < RAW; ++j) load_a(j, a_raw[j]);
    }
    if (t < CI) {
        sc_s[t] = p.p_scale ? p.p_scale[t] : 1.f;
        sh_s[t] = p.p_shift ? p.p_shift[t] : 0.f;
    }
    __syncthreads();

    if (warp >= DW_CONS_WARPS) {
        // ================================ producers ================================
        if constexpr (Cfg::REG_SPLIT) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PROD_REGS));
        const bool pro = p.p_scale || p.p_shift || p.p_relu;
        // (point pt, channel 4*c40 + e) -> K-major row 4*c40 + e, element pt of its 128-byte row; the
        // channels 16*j further on lie two 8-row swizzle atoms (2048 bytes) further on
        uint32_t soff[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) soff[e] = sw128_off(4 * c40 + e, pt >> 2) + (uint32_t)(pt & 3) * 4u;
        auto st_shared = [](uint32_t addr, uint32_t v) {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
        };
        const uint32_t smem_u = smem_u32(smem);
        int ch = 0, s = 0;
        uint32_t use = 0;  // how many times the ring has wrapped
        auto produce = [&](float4 (&cur)[B_F4]) {
            if (use > 0) mbar_wait(bar_empty(s), (use - 1) & 1);
            const uint32_t stage = smem_u + (uint32_t)s * STAGE_BYTES;  // stage layout: B hi | B lo
            const bool affine = pro && m_beg + (int64_t)ch * DW_PTS + pt < m_end;
#pragma unroll
            for (int j = 0; j < B_F4; ++j) {
                float4 v = cur[j];
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
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const uint32_t addr = stage + soff[e] + 2048u * (uint32_t)j;
                    const uint32_t hi = to_tf32(vv[e]);
                    st_shared(addr, hi);
                    st_shared(addr + B_BYTES, to_tf32(vv[e] - __uint_as_float(hi)));
                }
            }
            load_chunk(ch + PF, cur);  // the registers are free again: PF chunks stay in flight
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_full(s));
            ++ch;
            if (++s == DW_STAGES) {
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
        if constexpr (Cfg::REG_SPLIT) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONS_REGS));
        float acc[MSUB][WN / 2];
#pragma unroll
        for (int m = 0; m < MSUB; ++m)
#pragma unroll
            for (int i = 0; i < WN / 2; ++i) acc[m][i] = 0.f;
        uint32_t a_hi[HL][MSUB][4], a_lo[HL][MSUB][4];
#pragma unroll
        for (int m = 0; m < MSUB; ++m) wg_reg_fence(acc[m]);
        const int col_g = CO >= 128 ? 0 : g * WN;  // first accumulator column of this warpgroup
        const uint32_t smem_u = smem_u32(smem);

        int s = 0, s_prev = 0;
        uint32_t phase = 0;
        // one chunk; PAR = ch % 2 keeps the raw A buffer index static when RAW spans two chunks
        auto consume = [&](int ch, auto par) {
            constexpr int PAR = decltype(par)::value;
            mbar_wait(bar_full(s), phase);
            const uint32_t bh = smem_u + (uint32_t)s * STAGE_BYTES + (uint32_t)col_g * 128u, bl = bh + B_BYTES;
#pragma unroll
            for (int kb = 0; kb < DW_KSTEPS; ++kb) {
                const int h = kb % HL, r = (PAR * DW_KSTEPS + kb) % RAW;
                // the group of the K-step HL steps back, the last reader of hi/lo buffer h, has completed
                wg_wait<HL - 1>();
#pragma unroll
                for (int m = 0; m < MSUB; ++m) {
                    wg_reg_fence(a_hi[h][m]);
                    wg_reg_fence(a_lo[h][m]);
                }
                if (kb == HL - 1 && ch > 0) {
                    // that was chunk ch-1's last group in this warpgroup: its stage may be refilled
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty(s_prev));
                }
#pragma unroll
                for (int m = 0; m < MSUB; ++m)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float v = a_raw[r][m][e];
                        const uint32_t hi = to_tf32(v);
                        a_hi[h][m][e] = hi;
                        a_lo[h][m][e] = to_tf32(v - __uint_as_float(hi));
                    }
                load_a(ch * DW_KSTEPS + kb + RAW, a_raw[r]);
                wg_fence();
                const uint64_t dbh = wg_desc_k_sw128(bh + kb * 32), dbl = wg_desc_k_sw128(bl + kb * 32);
#pragma unroll
                for (int m = 0; m < MSUB; ++m) {
                    wgmma_tf32<WN>(acc[m], a_hi[h][m], dbh, 1u);
                    wgmma_tf32<WN>(acc[m], a_lo[h][m], dbh, 1u);
                    wgmma_tf32<WN>(acc[m], a_hi[h][m], dbl, 1u);
                }
                wg_commit();
            }
            s_prev = s;
            if (++s == DW_STAGES) {
                s = 0;
                phase ^= 1u;
            }
        };
        if constexpr (RAW > DW_KSTEPS) {
            for (int ch = 0; ch < nchunks; ch += 2) {
                consume(ch, std::integral_constant<int, 0>());
                if (ch + 1 < nchunks) consume(ch + 1, std::integral_constant<int, 1>());
            }
        } else {
            for (int ch = 0; ch < nchunks; ++ch) consume(ch, std::integral_constant<int, 0>());
        }
        wg_wait<0>();
#pragma unroll
        for (int m = 0; m < MSUB; ++m) wg_reg_fence(acc[m]);
#pragma unroll
        for (int h = 0; h < HL; ++h)
#pragma unroll
            for (int m = 0; m < MSUB; ++m) {
                wg_reg_fence(a_hi[h][m]);
                wg_reg_fence(a_lo[h][m]);
            }

        // ---- epilogue: accumulator -> this CTA's partial [CO, CI] (zeros when the CTA got no points)
        float* out = p.partial + (int64_t)blockIdx.x * CO * CI;
        const int cq = 2 * (lane & 3);
#pragma unroll
        for (int m = 0; m < MSUB; ++m) {
            const int row = a_co + 2 * m;  // fragment row 64m + 16wl + l/4; row + 1: that row + 8
#pragma unroll
            for (int j = 0; j < WN / 8; ++j) {
                const int col = col_g + 8 * j + cq;
                *reinterpret_cast<float2*>(out + (int64_t)row * CI + col) =
                    make_float2(acc[m][4 * j], acc[m][4 * j + 1]);
                *reinterpret_cast<float2*>(out + (int64_t)(row + 1) * CI + col) =
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
