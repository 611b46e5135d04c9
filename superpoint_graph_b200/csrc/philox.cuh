// Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11), the
// counter-based generator of the Random123 library: four 32-bit words per (counter, key) pair, no state.
#pragma once
#include <stdint.h>

namespace spg {

struct Philox4 {
    uint32_t v[4];
};

__host__ __device__ __forceinline__ uint32_t philox_mulhi(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                          uint32_t k0, uint32_t k1) {
    constexpr uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u;
    constexpr uint32_t kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k0 += kW0;
            k1 += kW1;
        }
        const uint32_t hi0 = philox_mulhi(kM0, c0), lo0 = kM0 * c0;
        const uint32_t hi1 = philox_mulhi(kM1, c2), lo1 = kM1 * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0;
        c1 = lo1;
        c2 = n2;
        c3 = lo0;
    }
    Philox4 o;
    o.v[0] = c0;
    o.v[1] = c1;
    o.v[2] = c2;
    o.v[3] = c3;
    return o;
}

// Dropout mask words of the element group q = i >> 2 (logical indices 4q .. 4q+3 of a row-major [M, C]
// activation): key (seed_lo, seed_hi), counter (q_lo, q_hi, ctr_lo, ctr_hi); element i uses word i & 3.
__host__ __device__ __forceinline__ Philox4 dropout_words(uint64_t seed, uint64_t ctr, uint64_t q) {
    return philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), (uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)seed,
                         (uint32_t)(seed >> 32));
}

// Keep threshold: an element is kept iff its word >= floor(p * 2^32); p >= 1 drops everything (DropParams::all).
__host__ __device__ __forceinline__ uint32_t dropout_threshold(float p) {
    if (!(p > 0.f)) return 0u;
    const double t = (double)p * 4294967296.0;
    return t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
}

// Per-launch dropout state, read from a slot (seed, ctr) in device memory.
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

// drop1 of the element with logical index i, one Philox call for this element alone
__device__ __forceinline__ float drop_at(const DropParams& d, int64_t i, float g) {
    return drop1(d, word_of(dropout_words(d.seed, d.ctr, (uint64_t)(i >> 2)), i), g);
}

}  // namespace spg
