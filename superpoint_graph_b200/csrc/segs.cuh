// Segment layouts of point rows: the max-pool (pointnet.cu) and GroupNorm (group_norm.cu) kernels are
// templated on them.
#pragma once
#include <stdint.h>

namespace spg {

// Fixed-length clouds (the reference's loader resamples every superpoint to L points,
// spg.py:209-214): segment b is rows [b*L, (b+1)*L).
struct FixedSegs {
    static constexpr bool kMayBeEmpty = false;  // L > 0
    int L;
    __device__ int64_t begin(int64_t b) const { return b * L; }
    __device__ int64_t end(int64_t b) const { return (b + 1) * L; }
    __device__ int64_t seg_of(int64_t r) const { return r / L; }
};

// Ragged CSR segments (north_star: "ragged segment boundaries carried as a CSR offset array"), the
// variant WITHOUT that resampling: segment b is rows [offsets[b], offsets[b+1]), row_seg[r] is the
// segment of row r.  An empty segment pools to 0 with argmax -1.
struct CsrSegs {
    static constexpr bool kMayBeEmpty = true;
    const int64_t* offsets;
    const int32_t* row_seg;
    __device__ int64_t begin(int64_t b) const { return offsets[b]; }
    __device__ int64_t end(int64_t b) const { return offsets[b + 1]; }
    __device__ int64_t seg_of(int64_t r) const { return row_seg[r]; }
};

// f(segs) with the layout a C-ABI call describes: fixed length L if offsets is NULL, else CSR.
template <class F>
static int with_segs(int L, const int64_t* offsets, const int32_t* row_seg, F&& f) {
    return offsets ? f(CsrSegs{offsets, row_seg}) : f(FixedSegs{L});
}

}  // namespace spg
