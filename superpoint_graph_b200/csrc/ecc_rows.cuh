// Vector-filter edge-conditioned convolution at 32 channels, one node per warp: the rows that the
// per-launch ECC kernels (ecc.cu) and the fused R x {ECC, cell} recurrences (rnn_cell.cu) both
// compute.  Both call these functions, so the two paths sum in the same order and agree bit for
// bit.
//
// Lane map: lane = (slot = lane>>3, sub = lane&7).  The 4 slots walk the node's edges interleaved
// (4 independent gather chains per node), the 8 sub lanes cover the 32 channels with float4.  The
// slot partials are combined with two xor shuffles, so every lane ends with the row's sum for its
// sub; callers store it from the slot-0 lanes.
#pragma once
#include "common.cuh"

namespace spg {

constexpr int kC = 32;
constexpr int kG = kC / 4;  // lanes per row

__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {
    c.x = fmaf(a.x, b.x, c.x);
    c.y = fmaf(a.y, b.y, c.y);
    c.z = fmaf(a.z, b.z, c.z);
    c.w = fmaf(a.w, b.w, c.w);
    return c;
}

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

// Sum over the 4 edge slots (lanes that differ in bits 3 and 4).
__device__ __forceinline__ float4 slot_reduce(float4 acc) {
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    return acc;
}

// The channels 4*sub..4*sub+3 of row `node` of a [n, 32] float array.
__device__ __forceinline__ const float4* row4(const float* a, int node, int sub) {
    return reinterpret_cast<const float4*>(a + (int64_t)node * kC + sub * 4);
}

// How a row function loads a node-feature or filter operand.
struct LdNc {  // read-only for the whole kernel: the non-coherent path
    __device__ static __forceinline__ float4 ld(const float4* p) { return __ldg(p); }
};
struct LdCg {  // written by other CTAs of the same kernel before a grid barrier: L2 only
    __device__ static __forceinline__ float4 ld(const float4* p) { return __ldcg(p); }
};
struct LdCs {  // read once: streamed, evict first
    __device__ static __forceinline__ float4 ld(const float4* p) { return ld_stream4(p); }
};

// out[node] = sum_{e in [beg, end)} x[idxn[e]] * w[e] / deg, deg = end - beg (0 if deg = 0), over
// the target CSR.  Each slot takes two edges per iteration (e, e+4) and one tail edge.
template <class LdX, class LdW>
__device__ __forceinline__ float4 ecc_vv_row_fwd(const float* x, const float4* w,
                                                 const int* __restrict__ idxn, int beg, int end,
                                                 int lane) {
    const int slot = lane >> 3, sub = lane & 7;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int e = beg + slot;
    for (; e + 4 < end; e += 8) {
        const int s0 = __ldg(idxn + e), s1 = __ldg(idxn + e + 4);
        const float4 w0 = LdW::ld(w + (int64_t)e * kG + sub);
        const float4 w1 = LdW::ld(w + (int64_t)(e + 4) * kG + sub);
        const float4 x0 = LdX::ld(row4(x, s0, sub));
        const float4 x1 = LdX::ld(row4(x, s1, sub));
        acc = fma4(x0, w0, acc);
        acc = fma4(x1, w1, acc);
    }
    if (e < end) {
        const int s0 = __ldg(idxn + e);
        const float4 w0 = LdW::ld(w + (int64_t)e * kG + sub);
        const float4 x0 = LdX::ld(row4(x, s0, sub));
        acc = fma4(x0, w0, acc);
    }
    acc = slot_reduce(acc);
    const int deg = end - beg;
    if (deg > 0) {
        const float d = (float)deg;
        acc.x /= d;
        acc.y /= d;
        acc.z /= d;
        acc.w /= d;
    }
    return acc;
}

// grad_x[node] without its added terms: sum_{p in [beg, end)} w[e] * g[t_e] / deg_t with
// e = src_perm[p], t_e = edge_tgt[e], over the source CSR.
template <class LdG, class LdW>
__device__ __forceinline__ float4 ecc_vv_row_bwd_x(const float4* w, const float* g,
                                                   const int* __restrict__ tgt_rowptr,
                                                   const int* __restrict__ src_perm,
                                                   const int* __restrict__ edge_tgt, int beg,
                                                   int end, int lane) {
    const int slot = lane >> 3, sub = lane & 7;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = beg + slot; p < end; p += 4) {
        const int e = __ldg(src_perm + p);
        const int tg = __ldg(edge_tgt + e);
        const float4 wv = LdW::ld(w + (int64_t)e * kG + sub);
        const float inv = 1.f / (float)(__ldg(tgt_rowptr + tg + 1) - __ldg(tgt_rowptr + tg));
        const float4 gv = LdG::ld(row4(g, tg, sub));
        acc.x = fmaf(wv.x, gv.x * inv, acc.x);
        acc.y = fmaf(wv.y, gv.y * inv, acc.y);
        acc.z = fmaf(wv.z, gv.z * inv, acc.z);
        acc.w = fmaf(wv.w, gv.w * inv, acc.w);
    }
    return slot_reduce(acc);
}

}  // namespace spg
