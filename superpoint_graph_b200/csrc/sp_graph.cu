// The superpoint graph of a partition (ref: partition/graphs.py:75-210 `compute_sp_graph`), the third phase of both
// partition pipelines (partition/partition.py:184, supervized_partition/supervized_partition.py:346,
// supervized_partition/generate_partition.py:109):
//
//   sp_scan       max(in_component) + 1 and a status word (1: a non-finite coordinate, 4: a negative id)
//   sp_sort_keys  the points sorted by (component, x, y, z): two stable CUB radix sorts of 64-bit keys, (y, z)
//                 then (component, x), over order-preserving float keys with -0 mapped to +0 (np.unique(axis=0)
//                 compares them equal); the first sorted position of every component
//   sp_points     one warp per component: its point count m, its unique rows (a row differing from the previous
//                 sorted row), numpy's np.mean of them (a sequential fp32 sum in sorted order from +0, the warp's
//                 rows folded one by one through shuffles, / u), the label histogram (integer atomics), and
//                 u == 2: numpy's fp32 sqrt(sum(var)); u >= 3: the fp64 covariance (ddof 1, two passes), the
//                 cyclic Jacobi of eig3.cuh, length = ev0, surface = sqrt(ev0 ev1 + 1e-10), volume =
//                 sqrt(ev0 ev1 ev2 + 1e-10) in fp64, rounded once
//   sp_tets       per tetrahedron the number of its 6 vertex pairs (both directions) whose endpoints lie in
//                 different components (status 2: an id outside [0, n)); after a scan, the (u, v) keys of those
//                 pairs at their offsets
//   sp_pairs      per deduplicated pair (radix sort + unique of the 64-bit keys): the exact 64-bit (source
//                 component, target component) key, or ~0 where the d_max cut drops it; a radix sort of
//                 (key, pair) and a run-length encode give the superedges in ascending key order
//   sp_edges      one thread per superedge: its pairs' offset statistics in fp64, rounded once, and the ratios
//
// No float atomics anywhere: two runs give identical bits.
#include <cub/cub.cuh>

#include "workspace.cuh"
#include "eig3.cuh"

namespace spg {

constexpr int SPG_THREADS = 256;
constexpr int SP_WARPS = 8;  // components per block of sp_points
constexpr uint64_t kNoKey = ~0ull;

// ------------------------------------------------------------------------------------------------ scan
// words[0] = max id + 1 (preset to 0), words[1] = status (preset to 0)
__global__ void __launch_bounds__(SPG_THREADS) sp_scan_kernel(const float* __restrict__ xyz,
                                                              const int64_t* __restrict__ comp, int64_t n,
                                                              unsigned long long* __restrict__ words) {
    SPG_PDL_ENTRY();
    long long hi = 0;
    unsigned bad = 0u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const long long c = __ldg(comp + i);
        if (c < 0) bad |= 4u;
        hi = max(hi, c + 1);
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (!isfinite(__ldg(xyz + 3 * i + k))) bad |= 1u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (hi > 0) atomicMax(reinterpret_cast<long long*>(words), hi);
        if (bad) atomicOr(words + 1, (unsigned long long)bad);
    }
}

// ------------------------------------------------------------------------------------------------ sort
__global__ void __launch_bounds__(SPG_THREADS) sp_keys_lo_kernel(const float* __restrict__ xyz, int64_t n,
                                                                 uint64_t* __restrict__ keys,
                                                                 int32_t* __restrict__ idx) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // + 0.f maps -0 to +0
    keys[i] = ((uint64_t)float_key(__fadd_rn(__ldg(xyz + 3 * i + 1), 0.f)) << 32) |
              float_key(__fadd_rn(__ldg(xyz + 3 * i + 2), 0.f));
    idx[i] = (int32_t)i;
}

__global__ void __launch_bounds__(SPG_THREADS) sp_keys_hi_kernel(const float* __restrict__ xyz,
                                                                 const int64_t* __restrict__ comp, int64_t n,
                                                                 const int32_t* __restrict__ idx,
                                                                 uint64_t* __restrict__ keys) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t i = __ldg(idx + p);
    keys[p] = ((uint64_t)__ldg(comp + i) << 32) | float_key(__fadd_rn(__ldg(xyz + 3 * i), 0.f));
}

// start[c] = first sorted position of component c; an empty component gets the empty range [p, p)
__global__ void __launch_bounds__(SPG_THREADS) sp_starts_kernel(const uint64_t* __restrict__ keys, int64_t n,
                                                                int64_t n_com, int32_t* __restrict__ start) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t c = (int64_t)(__ldg(keys + p) >> 32);
    const int64_t prev = p > 0 ? (int64_t)(__ldg(keys + p - 1) >> 32) : -1;
    for (int64_t k = prev + 1; k <= c; ++k) start[k] = (int32_t)p;
    if (p == n - 1)
        for (int64_t k = c + 1; k <= n_com; ++k) start[k] = (int32_t)n;
}

// ------------------------------------------------------------------------------------------------ superpoints
struct PointsArgs {
    const float* xyz;
    const int64_t* labels;   // label_mode 1: [n]; 2: [n, n_label_cols]
    int label_mode;          // 0: none, 1: histogram of the values 0..n_labels, 2: sum of the label rows
    int n_labels;
    int64_t n_label_cols;
    const int32_t* order;    // [n] original index of every sorted position
    const int32_t* start;    // [n_com + 1]
    int64_t n_com;
    float* centroids;        // [n_com, 3]
    float* length;           // [n_com]
    float* surface;
    float* volume;
    int64_t* point_count;    // [n_com]
    int64_t* sp_labels;      // [n_com, n_label_cols] (zeroed)
    unsigned* status;        // 8: an empty component
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the row at sorted position p of [s0, s1) and whether it is unique (differs from the previous sorted row)
__device__ __forceinline__ bool sp_row(const PointsArgs& a, int64_t s0, int64_t p, float& x, float& y, float& z,
                                       int64_t& i) {
    i = __ldg(a.order + p);
    x = __ldg(a.xyz + 3 * i);
    y = __ldg(a.xyz + 3 * i + 1);
    z = __ldg(a.xyz + 3 * i + 2);
    if (p == s0) return true;
    const int64_t j = __ldg(a.order + p - 1);
    return x != __ldg(a.xyz + 3 * j) || y != __ldg(a.xyz + 3 * j + 1) || z != __ldg(a.xyz + 3 * j + 2);
}

__global__ void __launch_bounds__(SP_WARPS * 32) sp_points_kernel(const PointsArgs a) {
    SPG_PDL_ENTRY();
    const int lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * SP_WARPS + (threadIdx.x >> 5);
    if (c >= a.n_com) return;
    const int64_t s0 = __ldg(a.start + c), s1 = __ldg(a.start + c + 1);
    if (s1 <= s0) {
        if (lane == 0) atomicOr(a.status, 8u);
        return;
    }
    // pass 1: the sequential fp32 sum, the fp64 sums and the count of the unique rows; the labels
    float ax = 0.f, ay = 0.f, az = 0.f;  // identical in every lane
    double sx = 0.0, sy = 0.0, sz = 0.0;
    int u_lane = 0;
    for (int64_t base = s0; base < s1; base += 32) {
        const int64_t p = base + lane;
        float x = 0.f, y = 0.f, z = 0.f;
        int64_t i = 0;
        const bool uq = p < s1 && sp_row(a, s0, p, x, y, z, i);
        unsigned m = __ballot_sync(0xffffffffu, uq);
        while (m) {  // the warp's unique rows in sorted order, one at a time
            const int j = __ffs(m) - 1;
            m &= m - 1;
            ax = __fadd_rn(ax, __shfl_sync(0xffffffffu, x, j));
            ay = __fadd_rn(ay, __shfl_sync(0xffffffffu, y, j));
            az = __fadd_rn(az, __shfl_sync(0xffffffffu, z, j));
        }
        if (uq) {
            sx += (double)x;
            sy += (double)y;
            sz += (double)z;
            ++u_lane;
        }
        if (p < s1 && a.label_mode == 1) {
            const int64_t v = __ldg(a.labels + i);
            if (v >= 0 && v <= a.n_labels)
                atomicAdd(reinterpret_cast<unsigned long long*>(a.sp_labels + c * a.n_label_cols + v), 1ull);
        } else if (p < s1 && a.label_mode == 2) {
            for (int64_t l = 0; l < a.n_label_cols; ++l)
                atomicAdd(reinterpret_cast<unsigned long long*>(a.sp_labels + c * a.n_label_cols + l),
                          (unsigned long long)__ldg(a.labels + i * a.n_label_cols + l));
        }
    }
    int u = u_lane;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) u += __shfl_xor_sync(0xffffffffu, u, o);
    sx = warp_sum_d(sx);
    sy = warp_sum_d(sy);
    sz = warp_sum_d(sz);
    // np.mean: the float32 sum divided by the integer count in float64, rounded to float32
    float cx = __double2float_rn(__ddiv_rn((double)ax, (double)u));
    float cy = __double2float_rn(__ddiv_rn((double)ay, (double)u));
    float cz = __double2float_rn(__ddiv_rn((double)az, (double)u));
    if (u == 1) {  // graphs.py:157 assigns the unique row itself
        const int64_t i = __ldg(a.order + s0);
        cx = __ldg(a.xyz + 3 * i);
        cy = __ldg(a.xyz + 3 * i + 1);
        cz = __ldg(a.xyz + 3 * i + 2);
    }
    // pass 2 (u >= 2): u == 2 the fp32 squares of np.var (two terms, so their sum is order-free); u >= 3 the fp64
    // centred products
    const double mx = sx / u, my = sy / u, mz = sz / u;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    double cxx = 0.0, cxy = 0.0, cxz = 0.0, cyy = 0.0, cyz = 0.0, czz = 0.0;
    if (u >= 2) {
        for (int64_t base = s0; base < s1; base += 32) {
            const int64_t p = base + lane;
            float x, y, z;
            int64_t i;
            if (p >= s1 || !sp_row(a, s0, p, x, y, z, i)) continue;
            if (u == 2) {
                const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy), dz = __fsub_rn(z, cz);
                qx = __fadd_rn(qx, __fmul_rn(dx, dx));
                qy = __fadd_rn(qy, __fmul_rn(dy, dy));
                qz = __fadd_rn(qz, __fmul_rn(dz, dz));
            } else {
                const double dx = (double)x - mx, dy = (double)y - my, dz = (double)z - mz;
                cxx += dx * dx;
                cxy += dx * dy;
                cxz += dx * dz;
                cyy += dy * dy;
                cyz += dy * dz;
                czz += dz * dz;
            }
        }
    }
    float len = 0.f, surf = 0.f, vol = 0.f;
    if (u == 2) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            qx = __fadd_rn(qx, __shfl_xor_sync(0xffffffffu, qx, o));
            qy = __fadd_rn(qy, __shfl_xor_sync(0xffffffffu, qy, o));
            qz = __fadd_rn(qz, __shfl_xor_sync(0xffffffffu, qz, o));
        }
        const float vx = __fdiv_rn(qx, 2.f), vy = __fdiv_rn(qy, 2.f), vz = __fdiv_rn(qz, 2.f);
        len = __fsqrt_rn(__fadd_rn(__fadd_rn(vx, vy), vz));
    } else if (u >= 3) {
        cxx = warp_sum_d(cxx);
        cxy = warp_sum_d(cxy);
        cxz = warp_sum_d(cxz);
        cyy = warp_sum_d(cyy);
        cyz = warp_sum_d(cyz);
        czz = warp_sum_d(czz);
        const double inv = 1.0 / (double)(u - 1);
        double A[3][3] = {{cxx * inv, cxy * inv, cxz * inv}, {cxy * inv, cyy * inv, cyz * inv},
                          {cxz * inv, cyz * inv, czz * inv}};
        double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
        geo_jacobi(A, V);
        double e[3] = {A[0][0], A[1][1], A[2][2]};
        geo_order(e, V, 0, 1);
        geo_order(e, V, 1, 2);
        geo_order(e, V, 0, 1);
        const double e01 = __dmul_rn(e[0], e[1]);
        len = __double2float_rn(e[0]);
        surf = __double2float_rn(__dsqrt_rn(__dadd_rn(e01, 1e-10)));
        vol = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(e01, e[2]), 1e-10)));
    }
    if (lane == 0) {
        a.centroids[3 * c] = cx;
        a.centroids[3 * c + 1] = cy;
        a.centroids[3 * c + 2] = cz;
        a.length[c] = len;
        a.surface[c] = surf;
        a.volume[c] = vol;
        a.point_count[c] = s1 - s0;
    }
}

// ------------------------------------------------------------------------------------------------ superedges
__device__ __forceinline__ int64_t sp_id(const void* s, int ids64, int64_t k) {
    return ids64 ? __ldg(static_cast<const int64_t*>(s) + k) : (int64_t)__ldg(static_cast<const int32_t*>(s) + k);
}


// emit == false: counts[t] = the directed pairs of tetrahedron t across components; true: their keys at offsets[t]
template <bool kEmit>
__global__ void __launch_bounds__(SPG_THREADS) sp_tets_kernel(const int64_t* __restrict__ comp, int64_t n,
                                                              const void* __restrict__ simplices, int ids64,
                                                              int64_t n_tets, int32_t* __restrict__ counts,
                                                              const int32_t* __restrict__ offsets,
                                                              uint64_t* __restrict__ keys,
                                                              unsigned* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tets) return;
    int64_t v[4], cv[4];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        v[k] = sp_id(simplices, ids64, 4 * t + k);
        bad |= v[k] < 0 || v[k] >= n;
    }
    if (bad) {
        if (!kEmit) {
            counts[t] = 0;
            atomicOr(status, 2u);
        }
        return;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) cv[k] = __ldg(comp + v[k]);
    int64_t o = kEmit ? __ldg(offsets + t) : 0;
    constexpr int kA[6] = {0, 0, 0, 1, 1, 2}, kB[6] = {1, 2, 3, 2, 3, 3};  // the tetrahedron's 6 vertex pairs
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        const int64_t p = v[kA[e]], q = v[kB[e]];
        if (cv[kA[e]] == cv[kB[e]]) continue;
        if (kEmit) {
            keys[o] = ((uint64_t)p << 32) | (uint64_t)q;
            keys[o + 1] = ((uint64_t)q << 32) | (uint64_t)p;
        }
        o += 2;
    }
    if (!kEmit) counts[t] = (int32_t)o;
}

// the component key of every deduplicated pair, ~0 beyond the pairs or where the d_max cut drops it
__global__ void __launch_bounds__(SPG_THREADS) sp_pairs_kernel(const float* __restrict__ xyz,
                                                               const int64_t* __restrict__ comp,
                                                               const uint64_t* __restrict__ pairs,
                                                               const int32_t* __restrict__ n_pairs, int64_t n_cand,
                                                               double d_max, uint64_t* __restrict__ ckeys) {
    SPG_PDL_ENTRY();
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_cand) return;
    uint64_t key = kNoKey;
    if (k < __ldg(n_pairs)) {
        const uint64_t pr = __ldg(pairs + k);
        const int64_t a = (int64_t)(pr >> 32), b = (int64_t)(pr & 0xffffffffu);
        bool keep = true;
        if (d_max > 0.0) {  // numpy's float32 sqrt(((dx dx + dy dy) + dz dz)) < float32(d_max)
            const float dx = __fsub_rn(__ldg(xyz + 3 * a), __ldg(xyz + 3 * b));
            const float dy = __fsub_rn(__ldg(xyz + 3 * a + 1), __ldg(xyz + 3 * b + 1));
            const float dz = __fsub_rn(__ldg(xyz + 3 * a + 2), __ldg(xyz + 3 * b + 2));
            keep = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))) <
                   __double2float_rn(d_max);
        }
        if (keep) key = ((uint64_t)__ldg(comp + a) << 32) | (uint64_t)__ldg(comp + b);
    }
    ckeys[k] = key;
}

// n_sedg = the runs of component keys, less the run of dropped pairs
__global__ void sp_count_kernel(const uint64_t* __restrict__ run_keys, const int32_t* __restrict__ n_runs,
                                int64_t* __restrict__ n_sedg) {
    SPG_PDL_ENTRY();
    const int r = __ldg(n_runs);
    n_sedg[0] = r - (r > 0 && __ldg(run_keys + r - 1) == kNoKey ? 1 : 0);
}

struct EdgesArgs {
    const float* xyz;
    const uint64_t* pairs;      // [n_cand] the kept pairs, sorted by component key
    const uint64_t* run_keys;   // [n_sedg] component keys, ascending
    const int32_t* run_start;   // [n_sedg] first pair
    const int32_t* run_count;   // [n_sedg] pairs
    int64_t n_sedg;
    const float *centroids, *length, *surface, *volume;
    const int64_t* point_count;
    int64_t *source, *target;
    float *delta_mean, *delta_std, *delta_norm, *delta_centroid, *length_ratio, *surface_ratio, *volume_ratio,
        *point_count_ratio;
};

__global__ void __launch_bounds__(SPG_THREADS) sp_edges_kernel(const EdgesArgs a) {
    SPG_PDL_ENTRY();
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_sedg) return;
    const uint64_t key = __ldg(a.run_keys + s);
    const int64_t cs = (int64_t)(key >> 32), ct = (int64_t)(key & 0xffffffffu);
    const int64_t k0 = __ldg(a.run_start + s), cnt = __ldg(a.run_count + s);
    auto delta = [&](int64_t k, double d[3]) {
        const uint64_t pr = __ldg(a.pairs + k);
        const int64_t u = (int64_t)(pr >> 32), v = (int64_t)(pr & 0xffffffffu);
#pragma unroll
        for (int c = 0; c < 3; ++c) d[c] = (double)__ldg(a.xyz + 3 * u + c) - (double)__ldg(a.xyz + 3 * v + c);
    };
    float mean[3], stdv[3], norm;
    if (cnt == 1) {  // graphs.py:207-209: the fp32 delta, std 0, its fp32 norm
        double d[3];
        delta(k0, d);
        float f[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            f[c] = __double2float_rn(d[c]);
            mean[c] = f[c];
            stdv[c] = 0.f;
        }
        norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(f[0], f[0]), __fmul_rn(f[1], f[1])), __fmul_rn(f[2], f[2])));
    } else {
        double sum[3] = {0.0, 0.0, 0.0}, nsum = 0.0;
        for (int64_t k = k0; k < k0 + cnt; ++k) {
            double d[3];
            delta(k, d);
#pragma unroll
            for (int c = 0; c < 3; ++c) sum[c] += d[c];
            nsum += sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        }
        double m[3], q[3] = {0.0, 0.0, 0.0};
#pragma unroll
        for (int c = 0; c < 3; ++c) m[c] = sum[c] / (double)cnt;
        for (int64_t k = k0; k < k0 + cnt; ++k) {
            double d[3];
            delta(k, d);
#pragma unroll
            for (int c = 0; c < 3; ++c) q[c] += (d[c] - m[c]) * (d[c] - m[c]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            mean[c] = __double2float_rn(m[c]);
            stdv[c] = __double2float_rn(sqrt(q[c] / (double)cnt));
        }
        norm = __double2float_rn(nsum / (double)cnt);
    }
    a.source[s] = cs;
    a.target[s] = ct;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        a.delta_mean[3 * s + c] = mean[c];
        a.delta_std[3 * s + c] = stdv[c];
        a.delta_centroid[3 * s + c] = __fsub_rn(__ldg(a.centroids + 3 * cs + c), __ldg(a.centroids + 3 * ct + c));
    }
    a.delta_norm[s] = norm;
    // graphs.py:196-199: float32 a / (b + 1e-6f); the point counts are uint64, so that ratio is in float64
    a.length_ratio[s] = __fdiv_rn(__ldg(a.length + cs), __fadd_rn(__ldg(a.length + ct), 1e-6f));
    a.surface_ratio[s] = __fdiv_rn(__ldg(a.surface + cs), __fadd_rn(__ldg(a.surface + ct), 1e-6f));
    a.volume_ratio[s] = __fdiv_rn(__ldg(a.volume + cs), __fadd_rn(__ldg(a.volume + ct), 1e-6f));
    a.point_count_ratio[s] = __double2float_rn(
        __ddiv_rn((double)__ldg(a.point_count + cs), __dadd_rn((double)__ldg(a.point_count + ct), 1e-6)));
}

// ------------------------------------------------------------------------------------------------ plans
struct PointsWs {
    uint64_t *keys_in, *keys;
    int32_t *idx_in, *idx, *start;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n, void* base, PointsWs* w) {
    const int m = (int)(n > 0 ? n : 1);
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int32_t*)nullptr, (int32_t*)nullptr, m);
    const size_t N = (size_t)m;
    Planner p(base);
    w->keys_in = p.take<uint64_t>(N);
    w->keys = p.take<uint64_t>(N);
    w->idx_in = p.take<int32_t>(N);
    w->idx = p.take<int32_t>(N);
    w->start = p.take<int32_t>(N + 1);  // n_com <= n for a partition with no empty component
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

struct EdgesWs {
    int32_t* counts;
    uint64_t* a;  // candidate keys, then the component keys
    uint64_t* b;  // sorted candidates, then the sorted component keys
    uint64_t* c;  // deduplicated pairs
    uint64_t* d;  // pairs in component-key order
    uint64_t* run_keys;
    int32_t *run_count, *run_start, *n_pairs, *n_runs;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n_tets, int64_t n_cand, void* base, EdgesWs* w) {
    const int t = (int)(n_tets + 1), m = (int)(n_cand > 0 ? n_cand : 1);
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, t);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortKeys, (const uint64_t*)nullptr, (uint64_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceSelect::Unique, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (int32_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const uint64_t*)nullptr, (uint64_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRunLengthEncode::Encode, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (int32_t*)nullptr, (int32_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, m + 1);
    const size_t T = (size_t)t, C = n_cand > 0 ? (size_t)n_cand : 0;
    Planner p(base);
    w->counts = p.take<int32_t>(T);
    w->a = p.take<uint64_t>(C);
    w->b = p.take<uint64_t>(C);
    w->c = p.take<uint64_t>(C);
    w->d = p.take<uint64_t>(C);
    w->run_keys = p.take<uint64_t>(C);
    w->run_count = p.take<int32_t>(C + 1);
    w->run_start = p.take<int32_t>(C + 1);
    w->n_pairs = p.take<int32_t>(1);
    w->n_runs = p.take<int32_t>(1);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

// 12 directed pairs per tetrahedron must be countable in int32
static bool too_many_tets(int64_t t) { return t < 0 || t > ((1ll << 31) - 2) / 12; }

static int id_bits(int64_t n) {
    int b = 1;
    while (b < 32 && (1ll << b) < n) ++b;
    return b;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_sp_scan(const float* xyz, const int64_t* in_component, int64_t n, int64_t* words, spg_stream_t stream) {
    if (n < 0 || !words || (n > 0 && (!xyz || !in_component))) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = cudaMemsetAsync(words, 0, 2 * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n == 0) return SPG_OK;
    const int64_t blocks = ceil_div64(n, SPG_THREADS);
    SPG_LAUNCH(K_SP_SCAN, s, sp_scan_kernel, (unsigned)(blocks < 4 * kNumSMs ? blocks : 4 * kNumSMs), SPG_THREADS, 0,
               xyz, in_component, n, (unsigned long long*)words);
    return launch_status();
}

int spg_sp_points_workspace(int64_t n, int64_t* bytes) {
    if (!bytes || n < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    PointsWs w;
    const int rc = layout(n, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_sp_points(const float* xyz, const int64_t* in_component, int64_t n, int64_t n_com, const int64_t* labels,
                  int label_mode, int64_t n_label_cols, int n_labels, void* workspace, int64_t workspace_bytes,
                  float* centroids, float* length, float* surface, float* volume, int64_t* point_count,
                  int64_t* sp_labels, uint32_t* status, spg_stream_t stream) {
    if (n <= 0 || n_com <= 0 || n_com > n || !xyz || !in_component || !centroids || !length ||
        !surface || !volume || !point_count || !status)
        return SPG_E_BADARG;
    if (label_mode < 0 || label_mode > 2 || (label_mode > 0 && (!labels || !sp_labels || n_label_cols < 1)) ||
        (label_mode == 1 && n_label_cols != (int64_t)n_labels + 1))
        return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    PointsWs w;
    int rc = layout(n, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e == cudaSuccess && label_mode > 0)
        e = cudaMemsetAsync(sp_labels, 0, (size_t)n_com * n_label_cols * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    const unsigned blocks = (unsigned)ceil_div64(n, SPG_THREADS);
    // (y, z) first, then a stable sort by (component, x): lexicographic (component, x, y, z)
    SPG_LAUNCH(K_SP_SORT_KEYS, s, sp_keys_lo_kernel, blocks, SPG_THREADS, 0, xyz, n, w.keys_in, w.idx_in);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.keys_in, w.keys, (const int32_t*)w.idx_in,
            w.idx, (int)n, 0, 64, s);
    SPG_LAUNCH(K_SP_SORT_KEYS, s, sp_keys_hi_kernel, blocks, SPG_THREADS, 0, xyz, in_component, n,
               (const int32_t*)w.idx, w.keys_in);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.keys_in, w.keys, (const int32_t*)w.idx,
            w.idx_in, (int)n, 0, 32 + id_bits(n_com), s);
    SPG_LAUNCH(K_SP_SORT_KEYS, s, sp_starts_kernel, blocks, SPG_THREADS, 0, (const uint64_t*)w.keys, n, n_com,
               w.start);
    PointsArgs a;
    a.xyz = xyz;
    a.labels = labels;
    a.label_mode = label_mode;
    a.n_labels = n_labels;
    a.n_label_cols = n_label_cols;
    a.order = w.idx_in;
    a.start = w.start;
    a.n_com = n_com;
    a.centroids = centroids;
    a.length = length;
    a.surface = surface;
    a.volume = volume;
    a.point_count = point_count;
    a.sp_labels = sp_labels;
    a.status = (unsigned*)status;
    SPG_LAUNCH(K_SP_POINTS, s, sp_points_kernel, (unsigned)ceil_div64(n_com, SP_WARPS), SP_WARPS * 32, 0, a);
    return launch_status();
}

int spg_sp_edges_workspace(int64_t n_tets, int64_t n_cand, int64_t* bytes) {
    if (!bytes || n_tets < 0 || n_cand < 0) return SPG_E_BADARG;
    if (too_many_tets(n_tets) || n_cand > 12 * n_tets) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    const int rc = layout(n_tets, n_cand, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_sp_edges_count(const int64_t* in_component, int64_t n, const void* simplices, int ids64, int64_t n_tets,
                       int32_t* tet_offsets, void* workspace, int64_t workspace_bytes, uint32_t* status,
                       spg_stream_t stream) {
    if (n <= 0 || n_tets < 0 || !in_component || !tet_offsets || !status || (n_tets > 0 && !simplices))
        return SPG_E_BADARG;
    if (too_big(n) || too_many_tets(n_tets)) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    int rc = layout(n_tets, 0, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.counts + n_tets, 0, sizeof(int32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n_tets > 0)
        SPG_LAUNCH(K_SP_TETS, s, sp_tets_kernel<false>, (unsigned)ceil_div64(n_tets, SPG_THREADS), SPG_THREADS, 0,
                   in_component, n, simplices, ids64, n_tets, w.counts, (const int32_t*)nullptr, (uint64_t*)nullptr,
                   (unsigned*)status);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.counts, tet_offsets, (int)n_tets + 1, s);
    return launch_status();
}

int spg_sp_edges_build(const float* xyz, const int64_t* in_component, int64_t n, const void* simplices, int ids64,
                       int64_t n_tets, const int32_t* tet_offsets, int64_t n_cand, double d_max, void* workspace,
                       int64_t workspace_bytes, int64_t* n_sedg, spg_stream_t stream) {
    if (n <= 0 || n_tets < 0 || n_cand < 0 || !xyz || !in_component || !tet_offsets || !n_sedg ||
        (n_tets > 0 && !simplices))
        return SPG_E_BADARG;
    if (too_big(n) || too_many_tets(n_tets) || n_cand > 12 * n_tets) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    int rc = layout(n_tets, n_cand, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (n_cand == 0) return (int)cudaMemsetAsync(n_sedg, 0, sizeof(int64_t), s);
    const int m = (int)n_cand;
    SPG_LAUNCH(K_SP_TETS, s, sp_tets_kernel<true>, (unsigned)ceil_div64(n_tets, SPG_THREADS), SPG_THREADS, 0,
               in_component, n, simplices, ids64, n_tets, (int32_t*)nullptr, tet_offsets, w.a, (unsigned*)nullptr);
    const int bits = id_bits(n);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortKeys, (const uint64_t*)w.a, w.b, m, 0, 32 + bits, s);
    SPG_CUB(w.cub, cub::DeviceSelect::Unique, (const uint64_t*)w.b, w.c, w.n_pairs, m, s);
    SPG_LAUNCH(K_SP_PAIRS, s, sp_pairs_kernel, (unsigned)ceil_div64(n_cand, SPG_THREADS), SPG_THREADS, 0, xyz,
               in_component, (const uint64_t*)w.c, (const int32_t*)w.n_pairs, n_cand, d_max, w.a);
    // the dropped pairs (key ~0) sort last; the component ids are below 2^31, so all 64 bits are sorted
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.a, w.b, (const uint64_t*)w.c, w.d, m, 0, 64,
            s);
    // counts beyond the last run stay 0, so the scan is valid for every run
    const cudaError_t e = cudaMemsetAsync(w.run_count, 0, ((size_t)m + 1) * 4, s);
    if (e != cudaSuccess) return (int)e;
    SPG_CUB(w.cub, cub::DeviceRunLengthEncode::Encode, (const uint64_t*)w.b, w.run_keys, w.run_count, w.n_runs, m, s);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.run_count, w.run_start, m + 1, s);
    SPG_LAUNCH(K_SP_PAIRS, s, sp_count_kernel, 1, 1, 0, (const uint64_t*)w.run_keys, (const int32_t*)w.n_runs,
               n_sedg);
    return launch_status();
}

int spg_sp_edges_features(const float* xyz, int64_t n_tets, int64_t n_cand, const void* workspace,
                          int64_t workspace_bytes, int64_t n_sedg, const float* centroids, const float* length,
                          const float* surface, const float* volume, const int64_t* point_count, int64_t* source,
                          int64_t* target, float* delta_mean, float* delta_std, float* delta_norm,
                          float* delta_centroid, float* length_ratio, float* surface_ratio, float* volume_ratio,
                          float* point_count_ratio, spg_stream_t stream) {
    if (n_sedg < 0 || n_sedg > n_cand || !workspace) return SPG_E_BADARG;
    if (n_sedg == 0) return SPG_OK;
    if (!xyz || !centroids || !length || !surface || !volume || !point_count || !source || !target || !delta_mean ||
        !delta_std || !delta_norm || !delta_centroid || !length_ratio || !surface_ratio || !volume_ratio ||
        !point_count_ratio)
        return SPG_E_BADARG;
    if (too_many_tets(n_tets) || n_cand > 12 * n_tets) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    int rc = layout(n_tets, n_cand, const_cast<void*>(workspace), &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    EdgesArgs a;
    a.xyz = xyz;
    a.pairs = w.d;
    a.run_keys = w.run_keys;
    a.run_start = w.run_start;
    a.run_count = w.run_count;
    a.n_sedg = n_sedg;
    a.centroids = centroids;
    a.length = length;
    a.surface = surface;
    a.volume = volume;
    a.point_count = point_count;
    a.source = source;
    a.target = target;
    a.delta_mean = delta_mean;
    a.delta_std = delta_std;
    a.delta_norm = delta_norm;
    a.delta_centroid = delta_centroid;
    a.length_ratio = length_ratio;
    a.surface_ratio = surface_ratio;
    a.volume_ratio = volume_ratio;
    a.point_count_ratio = point_count_ratio;
    SPG_LAUNCH(K_SP_EDGES, (cudaStream_t)stream, sp_edges_kernel, (unsigned)ceil_div64(n_sedg, SPG_THREADS),
               SPG_THREADS, 0, a);
    return launch_status();
}

}  // extern "C"
