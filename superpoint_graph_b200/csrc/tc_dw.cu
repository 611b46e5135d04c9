// Hopper (wgmma) weight-gradient GEMM of the point-wise layers:
//
//     dW[Co, Ci] = sum_m dY[m, Co] * f(P)[m, Ci]        (m runs over all Nv*L points)
//
// Both operands lie in HBM point-major (channels contiguous), i.e. the reduction dimension is the OUTER
// one.  wgmma reads tf32 operands K-major only, so the CTA transposes while it stages: it owns a
// contiguous slab of points, streams it in chunks of 32 points (one 128-byte SWIZZLE_128B row per
// channel) through a 2-stage shared-memory ring, splitting every value into tf32 hi/lo on the fly (3xTF32,
// fp32-equivalent).  Two warpgroups keep the [Co, Ci] accumulator in registers for the CTA's whole
// lifetime (Co >= 128: half of the rows each; Co = 64: half of the columns each) and finally write one
// partial per CTA; gemm_splitk_reduce adds the partials in a fixed order (deterministic).
// f = affine + ReLU of the layer that produced P (fused).
//
// Reference semantics: the weight gradient of nn.Conv1d(k=1) (learning/pointnet.py:29,85) as
// autograd computes it; the reference materialises ReLU(BN(P)) and runs cuDNN/cuBLAS on it.
#include "common.cuh"
#include "tc_common.cuh"

namespace spg {

constexpr int DW_THREADS = 256;
constexpr int DW_PTS = 32;  // points per chunk (4 wgmma K-steps of 8)

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
    constexpr int WM = CO >= 128 ? CO / 2 : 64;  // accumulator rows of one warpgroup
    constexpr int WN = CO >= 128 ? CI : CI / 2;  // accumulator columns of one warpgroup
    constexpr int MSUB = WM / 64;                 // m64 sub-tiles
    constexpr int A_BYTES = CO * DW_PTS * 4;      // one of hi|lo: [CO rows][128 B]
    constexpr int B_BYTES = CI * DW_PTS * 4;
    constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
    static_assert(CO % 64 == 0 && CI % 32 == 0 && CI <= 128 && CO <= 256, "shape");
    constexpr int A_F4 = CO * DW_PTS / 4 / DW_THREADS;  // float4 per thread per chunk
    constexpr int B_F4 = CI * DW_PTS / 4 / DW_THREADS;

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const int g = warp >> 2, wl = warp & 3;
    SPG_PDL_ENTRY();

    const int64_t m_beg = (int64_t)blockIdx.x * p.pts_per_cta;
    const int64_t m_end = min(p.M, m_beg + p.pts_per_cta);
    const int nchunks = m_beg < m_end ? (int)((m_end - m_beg + DW_PTS - 1) / DW_PTS) : 0;
    const bool pro = p.p_scale || p.p_shift || p.p_relu;

    // Thread i of a chunk handles the float4 (point pt, channels 4*c4..4*c4+3): a warp covers 8 points x
    // 4 channel groups, so that its 64-byte row segments are whole sectors and its transposed 4-byte
    // shared-memory stores spread over 16 banks.
    auto coord = [](int i, int c4s, int& pt, int& c4) {
        const int wi = i >> 5, l = i & 31;
        pt = (wi & 3) * 8 + (l & 7);
        c4 = (wi >> 2) * 4 + (l >> 3);
        (void)c4s;
    };
    float4 ra[A_F4], rb[B_F4];
    auto load_chunk = [&](int ch) {
        const int64_t mrow = m_beg + (int64_t)ch * DW_PTS;
#pragma unroll
        for (int j = 0; j < A_F4; ++j) {
            int pt, c4;
            coord(t + DW_THREADS * j, CO / 4, pt, c4);
            ra[j] = (mrow + pt < m_end)
                        ? __ldg(reinterpret_cast<const float4*>(p.dY + (mrow + pt) * p.lddy + c4 * 4))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < B_F4; ++j) {
            int pt, c4;
            coord(t + DW_THREADS * j, CI / 4, pt, c4);
            rb[j] = (mrow + pt < m_end)
                        ? __ldg(reinterpret_cast<const float4*>(p.P + (mrow + pt) * p.ldp + c4 * 4))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    // (point pt, channels 4*c4 + e) -> K-major row 4*c4 + e, element pt of its 128-byte row
    auto split_store = [&](uint8_t* hi_base, uint8_t* lo_base, int pt, int c4, float4 v) {
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const uint32_t off = sw128_off(4 * c4 + e, pt >> 2) + (uint32_t)(pt & 3) * 4u;
            const uint32_t hi = to_tf32(vv[e]);
            *reinterpret_cast<uint32_t*>(hi_base + off) = hi;
            *reinterpret_cast<uint32_t*>(lo_base + off) = to_tf32(vv[e] - __uint_as_float(hi));
        }
    };

    float acc[MSUB][WN / 2];
#pragma unroll
    for (int m = 0; m < MSUB; ++m)
#pragma unroll
        for (int i = 0; i < WN / 2; ++i) acc[m][i] = 0.f;
    const int row_g = CO >= 128 ? g * WM : 0;  // first accumulator row / column of this warpgroup
    const int col_g = CO >= 128 ? 0 : g * WN;

    if (nchunks > 0) load_chunk(0);
    for (int ch = 0; ch < nchunks; ++ch) {
        const int s = ch & 1;
        uint8_t* stage = smem + (size_t)s * STAGE_BYTES;
        uint8_t* a_hi = stage;
        uint8_t* a_lo = stage + A_BYTES;
        uint8_t* b_hi = stage + 2 * A_BYTES;
        uint8_t* b_lo = b_hi + B_BYTES;
        // the products of chunk ch-2 (the last reader of this stage) have completed in both warpgroups
        wg_wait<1>();
        wg_reg_fence(acc[0]);
        if (MSUB > 1) wg_reg_fence(acc[MSUB - 1]);
        __syncthreads();
        const int64_t mrow = m_beg + (int64_t)ch * DW_PTS;
#pragma unroll
        for (int j = 0; j < A_F4; ++j) {
            int pt, c4;
            coord(t + DW_THREADS * j, CO / 4, pt, c4);
            split_store(a_hi, a_lo, pt, c4, ra[j]);
        }
#pragma unroll
        for (int j = 0; j < B_F4; ++j) {
            int pt, c4;
            coord(t + DW_THREADS * j, CI / 4, pt, c4);
            float4 v = rb[j];
            if (pro && (mrow + pt < m_end)) {
                float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.p_scale) sc = __ldg(reinterpret_cast<const float4*>(p.p_scale + c4 * 4));
                if (p.p_shift) sh = __ldg(reinterpret_cast<const float4*>(p.p_shift + c4 * 4));
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
            split_store(b_hi, b_lo, pt, c4, v);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        {
            const uint32_t ah = smem_u32(a_hi) + (uint32_t)row_g * 128u, al = smem_u32(a_lo) + (uint32_t)row_g * 128u;
            const uint32_t bh = smem_u32(b_hi) + (uint32_t)col_g * 128u, bl = smem_u32(b_lo) + (uint32_t)col_g * 128u;
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
        }
        if (ch + 1 < nchunks) load_chunk(ch + 1);  // in flight while the tensor core works
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
            *reinterpret_cast<float2*>(out + (int64_t)row * CI + col) = make_float2(acc[m][4 * j], acc[m][4 * j + 1]);
            *reinterpret_cast<float2*>(out + (int64_t)(row + 8) * CI + col) =
                make_float2(acc[m][4 * j + 2], acc[m][4 * j + 3]);
        }
    }
}

template <int CO, int CI>
static int launch_dw(const DwArgs& a, int ctas, cudaStream_t s) {
    constexpr int STAGE_BYTES = 2 * CO * DW_PTS * 4 + 2 * CI * DW_PTS * 4;
    const int smem = 2 * STAGE_BYTES + 1024;
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
