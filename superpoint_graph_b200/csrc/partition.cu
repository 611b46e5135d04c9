// The learned partition's objective and its evaluation (ref: supervized_partition/losses.py, learning/metrics.py:87-92,
// partition/provider.py:689-695), everything of a training step after the embedding except cut pursuit:
//
//   lp_incidence   per-vertex CSR of the edge endpoints (CUB stable radix sort): the backward gathers through it
//   lp_dist_fwd    diff[e] of compute_dist (euclidian / intrinsic / scalar), and the per-edge factor of its backward
//   lp_dist_bwd    dL/dembeddings, a thread per (vertex, column) over the vertex's incidences in a fixed order
//   lp_loss_fwd    compute_loss: fp64 per-block partials over a fixed grid, merged in a fixed order
//   lp_loss_bwd    dL/ddiff
//   lp_cc          connected components of the edges with is_transition + pred_transition == 0 (the union-find
//                  of cc.cuh: libply_c's connected_comp with cutoff 0)
//   lp_xpart       crosspartition weights: a radix sort of the transition edges' unordered component pairs,
//                  run lengths by binary search in the sorted keys
//   lp_seal        SEAL weights: a radix sort of (component, object) pairs, run lengths, per-component maximum
//   lp_weights     'none' / 'proportional' weights, transition counts, cut pursuit's edge weights
//   lp_relax       relax_edge_binary
//   lp_metrics     boundary recall / precision counts and perfect_prediction
//
// No float atomics anywhere; the integer atomics (component sizes, run-length maxima, hooks of the union-find,
// counts) give the same result in any order.  Every float output is bit-reproducible.
#include <algorithm>
#include <climits>

#include <cub/cub.cuh>

#include "cc.cuh"
#include "workspace.cuh"

namespace spg {

constexpr int LP_THREADS = 256;
constexpr int LP_LOSS_BLOCKS = 2 * kNumSMs;

enum { LP_EUCLIDIAN = 0, LP_INTRINSIC = 1, LP_SCALAR = 2 };
enum { LP_TV = 0, LP_LAPLACIAN = 1, LP_TVH = 2 };
enum { LP_NONE = -1, LP_ZHANG = 0, LP_TVMINUS = 1 };

// losses.py:35-37: (acos(0.999*dot) - acos(0.999)) / (acos(-0.999) - acos(0.999)) * 3.141592
constexpr double kSmooth = 0.999;
constexpr double kPiRef = 3.141592;

static unsigned grid_of(int64_t n) { return (unsigned)ceil_div64(n > 0 ? n : 1, LP_THREADS); }

static int bits_for(uint64_t n) {  // smallest b with 2^b >= n (at least 1)
    int b = 1;
    while (b < 64 && (1ull << b) < n) ++b;
    return b;
}

// ------------------------------------------------------------------------------------------ incidence CSR
__global__ void __launch_bounds__(LP_THREADS)
lp_incidence_keys_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt, int64_t n_ver,
                         int64_t n_edges, int* __restrict__ keys, int* __restrict__ vals) {
    SPG_PDL_ENTRY();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= 2 * n_edges) return;
    const int64_t v = j < n_edges ? src[j] : tgt[j - n_edges];
    keys[j] = (v >= 0 && v < n_ver) ? (int)v : (int)n_ver;  // out-of-range endpoints sort past every row
    vals[j] = (int)j;
}

__global__ void __launch_bounds__(LP_THREADS)
lp_rowptr_kernel(const int* __restrict__ keys_sorted, int64_t n_rows, int64_t n, int* __restrict__ rowptr) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v > n_rows) return;
    int64_t lo = 0, hi = n;  // first position with key >= v
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys_sorted + mid) < (int)v) lo = mid + 1; else hi = mid;
    }
    rowptr[v] = (int)lo;
}

// ------------------------------------------------------------------------------------------ distance
__device__ __forceinline__ bool in_range(int64_t v, int64_t n) { return v >= 0 && v < n; }

__global__ void __launch_bounds__(LP_THREADS)
lp_dist_fwd_kernel(const float* __restrict__ emb, int64_t n_ver, int D, const int64_t* __restrict__ src,
                   const int64_t* __restrict__ tgt, int64_t n_edges, int dist_type, float* __restrict__ diff,
                   float* __restrict__ coef) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int64_t s = src[e], t = tgt[e];
    if (!in_range(s, n_ver) || !in_range(t, n_ver)) {
        diff[e] = __int_as_float(0x7fc00000);
        if (coef) coef[e] = 0.f;
        return;
    }
    const float* xs = emb + s * D;
    const float* xt = emb + t * D;
    double acc = 0.0;
    if (dist_type == LP_EUCLIDIAN) {
        for (int d = 0; d < D; ++d) {
            const double u = (double)__ldg(xs + d) - (double)__ldg(xt + d);
            acc = fma(u, u, acc);
        }
        diff[e] = (float)acc;
        return;
    }
    for (int d = 0; d < D; ++d) acc = fma((double)__ldg(xs + d), (double)__ldg(xt + d), acc);
    if (dist_type == LP_SCALAR) {
        diff[e] = (float)(acc - 1.0);
        coef[e] = 1.f;
        return;
    }
    const double a0 = acos(kSmooth), a1 = acos(-kSmooth);
    const double x = acc * kSmooth;
    diff[e] = (float)((acos(x) - a0) / (a1 - a0) * kPiRef);
    coef[e] = (float)(-kSmooth / sqrt(1.0 - x * x) * kPiRef / (a1 - a0));  // d diff / d dot
}

// gemb[v, d] = sum over the incidences of v (sorted by edge, source side first) of
//   euclidian:        2 g (x_v[d] - x_other[d])
//   intrinsic/scalar: g coef x_other[d]
__global__ void __launch_bounds__(LP_THREADS)
lp_dist_bwd_kernel(const float* __restrict__ emb, int64_t n_ver, int D, const int64_t* __restrict__ src,
                   const int64_t* __restrict__ tgt, int64_t n_edges, int dist_type, const float* __restrict__ coef,
                   const float* __restrict__ gdiff, const int* __restrict__ rowptr, const int* __restrict__ entry,
                   float* __restrict__ gemb) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_ver * D) return;
    const int64_t v = i / D;
    const int d = (int)(i - v * D);
    const double xv = (double)__ldg(emb + i);
    double acc = 0.0;
    const int k1 = __ldg(rowptr + v + 1);
    for (int k = __ldg(rowptr + v); k < k1; ++k) {
        const int j = __ldg(entry + k);
        const int64_t e = j < n_edges ? j : j - n_edges;
        const int64_t o = j < n_edges ? __ldg(tgt + e) : __ldg(src + e);
        if (!in_range(o, n_ver)) continue;
        const double g = (double)__ldg(gdiff + e);
        const double xo = (double)__ldg(emb + o * D + d);
        if (dist_type == LP_EUCLIDIAN) acc = fma(2.0 * g, xv - xo, acc);
        else acc = fma(g * (double)__ldg(coef + e), xo, acc);
    }
    gemb[i] = (float)acc;
}

// ------------------------------------------------------------------------------------------ loss
struct LossTerms {
    double l1, l2;   // this edge's contribution to loss1 / loss2
    double d1, d2;   // d l1 / d diff, d l2 / d diff
};

__device__ __forceinline__ LossTerms loss_terms(float diff, float w, uint8_t t, int intra, int inter, double beta) {
    LossTerms r = {0.0, 0.0, 0.0, 0.0};
    const double d = (double)diff, wd = (double)w;
    if (t == 0) {
        if (intra == LP_TV) {
            const double s = sqrt(d + 1e-10);
            r.l1 = wd * s;
            r.d1 = wd * 0.5 / s;
        } else if (intra == LP_LAPLACIAN) {
            r.l1 = wd * d;
            r.d1 = wd;
        } else {  // TVH, delta = 0.2 (losses.py:51-52)
            const double delta = 0.2, d2 = delta * delta;
            const double s = sqrt(1.0 + d / d2);
            r.l1 = delta * wd * (s - 1.0);
            r.d1 = delta * wd * 0.5 / (s * d2);
        }
    } else if (t == 1) {
        const double s = sqrt(d + 1e-10);
        if (inter == LP_ZHANG) {  // clamp(-w x + w beta, min = 0); torch passes the gradient where the input >= 0
            const double z = -wd * s + wd * beta;
            r.l2 = z < 0.0 ? 0.0 : z;  // NaN stays NaN, as torch.clamp
            r.d2 = (z >= 0.0 ? -wd : 0.0) * (0.5 / s);  // 0 * NaN stays NaN, as in torch's chain
        } else if (inter == LP_TVMINUS) {
            r.l2 = s * wd;
            r.d2 = wd * 0.5 / s;
        }
    }
    return r;
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(LP_THREADS)
lp_loss_fwd_kernel(const float* __restrict__ diff, const float* __restrict__ w, const uint8_t* __restrict__ is_trans,
                   int64_t n_edges, int intra, int inter, double beta, double* __restrict__ partials) {
    SPG_PDL_ENTRY();
    __shared__ double sh[2][LP_THREADS / 32];
    double a = 0.0, b = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += (int64_t)gridDim.x * blockDim.x) {
        const LossTerms r = loss_terms(__ldg(diff + e), __ldg(w + e), __ldg(is_trans + e), intra, inter, beta);
        a += r.l1;
        b += r.l2;
    }
    a = warp_sum_d(a);
    b = warp_sum_d(b);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        sh[0][warp] = a;
        sh[1][warp] = b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0.0, s1 = 0.0;
        for (int k = 0; k < LP_THREADS / 32; ++k) {
            s0 += sh[0][k];
            s1 += sh[1][k];
        }
        partials[2 * blockIdx.x] = s0;
        partials[2 * blockIdx.x + 1] = s1;
    }
}

__global__ void __launch_bounds__(32)
lp_loss_final_kernel(const double* __restrict__ partials, int n_partials, float* __restrict__ loss) {
    SPG_PDL_ENTRY();
    double a = 0.0, b = 0.0;
    for (int k = threadIdx.x; k < n_partials; k += 32) {
        a += partials[2 * k];
        b += partials[2 * k + 1];
    }
    a = warp_sum_d(a);
    b = warp_sum_d(b);
    if (threadIdx.x == 0) {
        loss[0] = (float)a;
        loss[1] = (float)b;
    }
}

__global__ void __launch_bounds__(LP_THREADS)
lp_loss_bwd_kernel(const float* __restrict__ diff, const float* __restrict__ w, const uint8_t* __restrict__ is_trans,
                   int64_t n_edges, int intra, int inter, double beta, const float* __restrict__ gloss,
                   float* __restrict__ gdiff) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const LossTerms r = loss_terms(__ldg(diff + e), __ldg(w + e), __ldg(is_trans + e), intra, inter, beta);
    gdiff[e] = (float)((double)__ldg(gloss) * r.d1 + (double)__ldg(gloss + 1) * r.d2);
}

// ------------------------------------------------------------------------------------------ connected components
__global__ void __launch_bounds__(LP_THREADS)
lp_cc_init_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt, const uint8_t* __restrict__ is_trans,
                  const int64_t* __restrict__ pic, int64_t n_ver, int64_t n_edges, int* __restrict__ parent,
                  int* __restrict__ comp_size, float* __restrict__ weights) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_ver) {
        parent[i] = (int)i;
        comp_size[i] = 0;
    }
    if (i < n_edges) weights[i] = 1.f;
}

// union of the endpoints of every active edge: is_transition + (pic[s] != pic[t]) == 0 (losses.py:133-136)
__global__ void __launch_bounds__(LP_THREADS)
lp_cc_hook_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt, const uint8_t* __restrict__ is_trans,
                  const int64_t* __restrict__ pic, int64_t n_ver, int64_t n_edges, int* __restrict__ parent) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges || is_trans[e] != 0) return;
    const int64_t s = src[e], t = tgt[e];
    if (!in_range(s, n_ver) || !in_range(t, n_ver) || pic[s] != pic[t]) return;
    cc_union(parent, (int)s, (int)t);
}

// ------------------------------------------------------------------------------------------ crosspartition
__global__ void __launch_bounds__(LP_THREADS)
lp_xpart_keys_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt,
                     const uint8_t* __restrict__ is_trans, const int* __restrict__ in_comp, int64_t n_ver,
                     int64_t n_edges, unsigned long long* __restrict__ keys, int* __restrict__ vals) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const unsigned long long sentinel = (unsigned long long)n_ver * (unsigned long long)n_ver;
    unsigned long long k = sentinel;
    const int64_t s = src[e], t = tgt[e];
    if (is_trans[e] != 0 && in_range(s, n_ver) && in_range(t, n_ver)) {
        const int a = in_comp[s], b = in_comp[t];
        const int lo = a < b ? a : b, hi = a < b ? b : a;
        k = (unsigned long long)lo * (unsigned long long)n_ver + (unsigned long long)hi;
    }
    keys[e] = k;
    vals[e] = (int)e;
}

__device__ __forceinline__ int64_t lower_bound_u64(const unsigned long long* a, int64_t n, unsigned long long k) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// weight of transition edge = 1 + min(|c1|, |c2|) / (#transition edges between c1 and c2) * factor (losses.py:150-158)
__global__ void __launch_bounds__(LP_THREADS)
lp_xpart_weights_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, int64_t n_ver,
                        int64_t n_edges, const int* __restrict__ comp_size, double factor, float* __restrict__ weights) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_edges) return;
    const unsigned long long sentinel = (unsigned long long)n_ver * (unsigned long long)n_ver;
    const unsigned long long k = keys[i];
    if (k >= sentinel) return;
    const int64_t count = lower_bound_u64(keys, n_edges, k + 1) - lower_bound_u64(keys, n_edges, k);
    const int lo = (int)(k / (unsigned long long)n_ver), hi = (int)(k % (unsigned long long)n_ver);
    const int m = min(comp_size[lo], comp_size[hi]);
    weights[vals[i]] = (float)(1.0 + (double)m / (double)count * factor);
}

// ------------------------------------------------------------------------------------------ SEAL
__global__ void __launch_bounds__(LP_THREADS)
lp_seal_keys_kernel(const int64_t* __restrict__ pic, const int64_t* __restrict__ objects, int64_t n_ver,
                    int64_t n_comp, unsigned long long* __restrict__ keys, unsigned* __restrict__ size,
                    unsigned* __restrict__ maxfreq) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v < n_comp) {
        size[v] = 0u;
        maxfreq[v] = 0u;
    }
    if (v >= n_ver) return;
    keys[v] = ((unsigned long long)pic[v] << 32) | (unsigned long long)(uint32_t)objects[v];
}

__global__ void __launch_bounds__(LP_THREADS)
lp_seal_runs_kernel(const unsigned long long* __restrict__ keys, int64_t n_ver, int64_t n_comp,
                    unsigned* __restrict__ size, unsigned* __restrict__ maxfreq) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_ver) return;
    const unsigned long long k = keys[i];
    const int64_t c = (int64_t)(k >> 32);
    if (c < 0 || c >= n_comp) return;
    atomicAdd(size + c, 1u);
    if (i > 0 && keys[i - 1] == k) return;  // run head only
    const int64_t len = lower_bound_u64(keys, n_ver, k + 1) - i;
    atomicMax(maxfreq + c, (unsigned)len);
}

// 1 + max(w[pic[s]], w[pic[t]]) * factor on transition edges, w = size - mode frequency (losses.py:121-127)
__global__ void __launch_bounds__(LP_THREADS)
lp_seal_weights_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ tgt,
                       const uint8_t* __restrict__ is_trans, const int64_t* __restrict__ pic, int64_t n_ver,
                       int64_t n_edges, int64_t n_comp, const unsigned* __restrict__ size,
                       const unsigned* __restrict__ maxfreq, double factor, float* __restrict__ weights,
                       int32_t* __restrict__ w_comp) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w_comp && i < n_comp) w_comp[i] = (int32_t)(size[i] - maxfreq[i]);
    if (i >= n_edges) return;
    float w = 1.f;
    const int64_t s = src[i], t = tgt[i];
    if (is_trans[i] != 0 && in_range(s, n_ver) && in_range(t, n_ver)) {
        const int64_t a = pic[s], b = pic[t];
        if (a >= 0 && a < n_comp && b >= 0 && b < n_comp) {
            const unsigned wa = size[a] - maxfreq[a], wb = size[b] - maxfreq[b];
            w = (float)(1.0 + (double)(wa > wb ? wa : wb) * factor);
        }
    }
    weights[i] = w;
}

// ------------------------------------------------------------------------------------------ simple weights, counts
__global__ void __launch_bounds__(LP_THREADS)
lp_fill_weights_kernel(const uint8_t* __restrict__ is_trans, int64_t n_edges, float w_other, float w_trans,
                       float* __restrict__ weights) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_edges) weights[e] = is_trans[e] != 0 ? w_trans : w_other;
}

// counts[0] += #(truth != 0 && pred != 0), counts[1] += #(truth != 0): the numerator and denominator of
// 100 * ((truth == pred) * truth).sum() / truth.sum() for 0/1 masks
__global__ void __launch_bounds__(LP_THREADS)
lp_count_kernel(const uint8_t* __restrict__ truth, const uint8_t* __restrict__ pred, int64_t n,
                unsigned long long* __restrict__ counts) {
    SPG_PDL_ENTRY();
    unsigned long long a = 0, b = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const bool t = truth[i] != 0;
        b += t;
        if (pred) a += t && pred[i] != 0;
    }
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (a) atomicAdd(counts, a);
        if (b) atomicAdd(counts + 1, b);
    }
}

// cut pursuit's edge weights (losses.py:68-72): threshold > 0: diff > 1 ? threshold : 1;
// threshold < 0: exp(diff * threshold) (float32, as torch) / exp(threshold) (float64, as numpy)
__global__ void __launch_bounds__(LP_THREADS)
lp_edge_weight_kernel(const float* __restrict__ diff, int64_t n_edges, double threshold, double* __restrict__ out) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const float d = diff[e];
    double w = 1.0;
    if (threshold > 0.0) w = d > 1.f ? (double)(float)threshold : 1.0;
    else if (threshold < 0.0) w = (double)expf(d * (float)threshold) / exp(threshold);
    out[e] = w;
}

// ------------------------------------------------------------------------------------------ relax_edge_binary
__global__ void __launch_bounds__(LP_THREADS)
lp_relax_mark_kernel(const uint8_t* __restrict__ relaxed, const int64_t* __restrict__ src,
                     const int64_t* __restrict__ tgt, int64_t n_ver, int64_t n_edges, uint8_t* __restrict__ mark) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges || relaxed[e] == 0) return;
    const int64_t s = src[e], t = tgt[e];
    if (in_range(s, n_ver)) mark[s] = 1;
    if (in_range(t, n_ver)) mark[t] = 1;
}

// losses.py:184 indexes with the uint8 mark values themselves (positions 0 and 1), :185 with a mask
__global__ void __launch_bounds__(LP_THREADS)
lp_relax_spread_kernel(uint8_t* __restrict__ relaxed, const int64_t* __restrict__ src, const int64_t* __restrict__ tgt,
                       const uint8_t* __restrict__ mark, int64_t n_ver, int64_t n_edges, int* __restrict__ hit) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int f = 0;
    if (e < n_edges) {
        const int64_t s = src[e], t = tgt[e];
        f = in_range(s, n_ver) && mark[s] ? 2 : 1;
        if (in_range(t, n_ver) && mark[t]) relaxed[e] = 1;
    }
    f = __reduce_or_sync(0xffffffffu, f);  // one atomic per warp
    if ((threadIdx.x & 31) == 0 && f) atomicOr(hit, f);
}

__global__ void __launch_bounds__(32)
lp_relax_index_kernel(uint8_t* __restrict__ relaxed, int64_t n_edges, int* __restrict__ hit,
                      int* __restrict__ status) {
    SPG_PDL_ENTRY();
    if (threadIdx.x != 0) return;
    const int h = *hit;
    if ((h & 1) && n_edges > 0) relaxed[0] = 1;
    if (h & 2) {
        if (n_edges > 1) relaxed[1] = 1;
        else *status = 1;  // numpy raises IndexError
    }
    *hit = 0;
}

// ------------------------------------------------------------------------------------------ perfect_prediction
// A warp per component: lane c sums labels[v, 1 + c] over the members in order (int64), the first maximum wins,
// then the warp writes it to every member.
__global__ void __launch_bounds__(LP_THREADS)
lp_perfect_kernel(const int64_t* __restrict__ comp_ptr, const int64_t* __restrict__ point_ids, int64_t n_comp,
                  const int64_t* __restrict__ labels, int64_t ld_labels, int n_classes, int64_t n_ver,
                  int64_t* __restrict__ pred) {
    SPG_PDL_ENTRY();
    const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (c >= n_comp) return;
    const int64_t p0 = comp_ptr[c], p1 = comp_ptr[c + 1];
    long long best = 0;
    int best_k = 0;
    for (int k0 = 0; k0 < n_classes; k0 += 32) {
        const int k = k0 + lane;
        long long s = 0;
        if (k < n_classes) {
            for (int64_t p = p0; p < p1; ++p) {
                const int64_t v = point_ids[p];
                if (in_range(v, n_ver)) s += labels[v * ld_labels + 1 + k];
            }
        }
        // first maximum over this chunk, then against the previous chunks (ties keep the earlier class)
        long long m = k < n_classes ? s : LLONG_MIN;
        int mk = k;
        for (int o = 16; o > 0; o >>= 1) {
            const long long om = __shfl_xor_sync(0xffffffffu, m, o);
            const int ok = __shfl_xor_sync(0xffffffffu, mk, o);
            if (om > m || (om == m && ok < mk)) {
                m = om;
                mk = ok;
            }
        }
        if (k0 == 0 || m > best) {
            best = m;
            best_k = mk;
        }
    }
    for (int64_t p = p0 + lane; p < p1; p += 32) {
        const int64_t v = point_ids[p];
        if (in_range(v, n_ver)) pred[v] = best_k;
    }
}

// 2E incidence entries must fit in int32: a lower limit than too_big (workspace.cuh)
static bool lp_too_big(int64_t n) { return n >= (1ll << 30); }

// The scratch of spg_lp_incidence, spg_lp_xpart and spg_lp_seal; each call uses its own regions
struct LpWs {
    int *inc_keys, *inc_keys_sorted, *inc_vals;             // incidence [2E]
    int *parent, *is_root, *root_rank;                      // xpart [V]
    unsigned long long *pair_keys, *pair_keys_sorted;       // xpart [E]
    int *pair_vals, *pair_vals_sorted;                      // xpart [E]
    unsigned long long *comp_keys, *comp_keys_sorted;       // seal [V]
    unsigned *size, *maxfreq;                               // seal [n_comp]
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n_ver, int64_t n_edges, int64_t n_comp, void* base, LpWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const unsigned long long*)nullptr,
                  (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr, (int)n_edges, 0,
                  bits_for((uint64_t)n_ver * (uint64_t)n_ver + 1));
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortKeys, (const unsigned long long*)nullptr,
                  (unsigned long long*)nullptr, (int)n_ver, 0, 32 + bits_for((uint64_t)n_comp + 1));
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const int*)nullptr, (int*)nullptr,
                  (const int*)nullptr, (int*)nullptr, (int)(2 * n_edges), 0, bits_for((uint64_t)n_ver + 1));
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int*)nullptr, (int*)nullptr, (int)n_ver);
    Planner p(base);
    w->inc_keys = p.take<int>(2 * n_edges);
    w->inc_keys_sorted = p.take<int>(2 * n_edges);
    w->inc_vals = p.take<int>(2 * n_edges);
    w->parent = p.take<int>(n_ver);
    w->is_root = p.take<int>(n_ver);
    w->root_rank = p.take<int>(n_ver);
    w->pair_keys = p.take<unsigned long long>(n_edges);
    w->pair_keys_sorted = p.take<unsigned long long>(n_edges);
    w->pair_vals = p.take<int>(n_edges);
    w->pair_vals_sorted = p.take<int>(n_edges);
    w->comp_keys = p.take<unsigned long long>(n_ver);
    w->comp_keys_sorted = p.take<unsigned long long>(n_ver);
    w->size = p.take<unsigned>(n_comp);
    w->maxfreq = p.take<unsigned>(n_comp);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_lp_workspace(int64_t n_ver, int64_t n_edges, int64_t n_comp, int64_t* bytes) {
    if (!bytes || n_ver < 0 || n_edges < 0 || n_comp < 0) return SPG_E_BADARG;
    if (lp_too_big(n_ver) || lp_too_big(2 * n_edges) || n_comp >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    LpWs w;
    const int rc = layout(n_ver, n_edges, n_comp, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_lp_incidence(const int64_t* src, const int64_t* tgt, int64_t n_ver, int64_t n_edges, int32_t* rowptr,
                     int32_t* entry, void* workspace, int64_t workspace_bytes, spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || !rowptr) return SPG_E_BADARG;
    if (lp_too_big(2 * n_edges) || lp_too_big(n_ver)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n = 2 * n_edges;
    LpWs w;
    int rc = layout(n_ver, n_edges, 0, workspace, &w);
    if (rc != SPG_OK) return rc;
    if (n > 0) {
        if (!src || !tgt || !entry) return SPG_E_BADARG;
        rc = ws_check(workspace, workspace_bytes, w.bytes);
        if (rc != SPG_OK) return rc;
        SPG_LAUNCH(K_LP_INCIDENCE, s, lp_incidence_keys_kernel, grid_of(n), LP_THREADS, 0, src, tgt, n_ver, n_edges,
                   w.inc_keys, w.inc_vals);
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const int*)w.inc_keys, w.inc_keys_sorted,
                (const int*)w.inc_vals, (int*)entry, (int)n, 0, bits_for((uint64_t)n_ver + 1), s);
    }
    SPG_LAUNCH(K_LP_INCIDENCE, s, lp_rowptr_kernel, grid_of(n_ver + 1), LP_THREADS, 0, (const int*)w.inc_keys_sorted,
               n_ver, n, (int*)rowptr);
    return launch_status();
}

int spg_lp_dist_fwd(const float* emb, int64_t n_ver, int D, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                    int dist_type, float* diff, float* coef, spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || D <= 0 || dist_type < 0 || dist_type > 2) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!emb || !src || !tgt || !diff || (dist_type != LP_EUCLIDIAN && !coef)) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_DIST_FWD, (cudaStream_t)stream, lp_dist_fwd_kernel, grid_of(n_edges), LP_THREADS, 0, emb, n_ver,
               D, src, tgt, n_edges, dist_type, diff, coef);
    return launch_status();
}

int spg_lp_dist_bwd(const float* emb, int64_t n_ver, int D, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                    int dist_type, const float* coef, const float* gdiff, const int32_t* rowptr, const int32_t* entry,
                    float* gemb, spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || D <= 0 || dist_type < 0 || dist_type > 2) return SPG_E_BADARG;
    if (n_ver == 0) return SPG_OK;
    if (!emb || !rowptr || !gemb || (n_edges > 0 && (!src || !tgt || !gdiff || !entry))) return SPG_E_BADARG;
    if (n_edges > 0 && dist_type != LP_EUCLIDIAN && !coef) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_DIST_BWD, (cudaStream_t)stream, lp_dist_bwd_kernel, grid_of(n_ver * D), LP_THREADS, 0, emb,
               n_ver, D, src, tgt, n_edges, dist_type, coef, gdiff, (const int*)rowptr, (const int*)entry, gemb);
    return launch_status();
}

int64_t spg_lp_loss_partials(void) { return LP_LOSS_BLOCKS; }

static double zhang_beta(int dist_type) { return dist_type == LP_INTRINSIC ? 1.0471975512 : 1.0; }

int spg_lp_loss_fwd(const float* diff, const float* weights, const uint8_t* is_transition, int64_t n_edges,
                    int intra, int inter, int dist_type, double* partials, float* loss, spg_stream_t stream) {
    if (n_edges < 0 || intra < 0 || intra > 2 || inter < -1 || inter > 1 || !partials || !loss) return SPG_E_BADARG;
    if (n_edges > 0 && (!diff || !weights || !is_transition)) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    SPG_LAUNCH(K_LP_LOSS_FWD, s, lp_loss_fwd_kernel, LP_LOSS_BLOCKS, LP_THREADS, 0, diff, weights, is_transition,
               n_edges, intra, inter, zhang_beta(dist_type), partials);
    SPG_LAUNCH(K_LP_LOSS_FWD, s, lp_loss_final_kernel, 1, 32, 0, (const double*)partials, LP_LOSS_BLOCKS, loss);
    return launch_status();
}

int spg_lp_loss_bwd(const float* diff, const float* weights, const uint8_t* is_transition, int64_t n_edges,
                    int intra, int inter, int dist_type, const float* gloss, float* gdiff, spg_stream_t stream) {
    if (n_edges < 0 || intra < 0 || intra > 2 || inter < -1 || inter > 1) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!diff || !weights || !is_transition || !gloss || !gdiff) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_LOSS_BWD, (cudaStream_t)stream, lp_loss_bwd_kernel, grid_of(n_edges), LP_THREADS, 0, diff,
               weights, is_transition, n_edges, intra, inter, zhang_beta(dist_type), gloss, gdiff);
    return launch_status();
}

int spg_lp_xpart(const int64_t* src, const int64_t* tgt, const uint8_t* is_transition,
                 const int64_t* pred_in_component, int64_t n_ver, int64_t n_edges, double transition_factor,
                 float* weights, int32_t* in_component_x, int32_t* comp_size, int32_t* n_comp, void* workspace,
                 int64_t workspace_bytes, spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || !n_comp) return SPG_E_BADARG;
    if (lp_too_big(n_ver) || lp_too_big(n_edges)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if (n_ver == 0) {
        e = cudaMemsetAsync(n_comp, 0, sizeof(int32_t), s);
        if (e != cudaSuccess) return (int)e;
    }
    if (n_ver > 0 && (!pred_in_component || !in_component_x || !comp_size)) return SPG_E_BADARG;
    if (n_edges > 0 && (!src || !tgt || !is_transition || !weights)) return SPG_E_BADARG;
    const int64_t nmax = n_ver > n_edges ? n_ver : n_edges;
    if (nmax == 0) return SPG_OK;
    LpWs w;
    int rc = layout(n_ver, n_edges, 0, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    SPG_LAUNCH(K_LP_CC, s, lp_cc_init_kernel, grid_of(nmax), LP_THREADS, 0, src, tgt, is_transition,
               pred_in_component, n_ver, n_edges, w.parent, (int*)comp_size, weights);
    if (n_ver == 0) return launch_status();
    if (n_edges > 0)
        SPG_LAUNCH(K_LP_CC, s, lp_cc_hook_kernel, grid_of(n_edges), LP_THREADS, 0, src, tgt, is_transition,
                   pred_in_component, n_ver, n_edges, w.parent);
    SPG_LAUNCH(K_LP_CC, s, cc_flatten_kernel, grid_of(n_ver), CC_THREADS, 0, w.parent, n_ver, w.is_root);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int*)w.is_root, w.root_rank, (int)n_ver, s);
    SPG_LAUNCH(K_LP_CC, s, cc_label_kernel<int>, grid_of(n_ver), CC_THREADS, 0, (const int*)w.parent,
               (const int*)w.root_rank, (const int*)w.is_root, n_ver, (int*)in_component_x, (int*)comp_size,
               (int*)n_comp);
    if (n_edges == 0) return launch_status();
    SPG_LAUNCH(K_LP_XPART, s, lp_xpart_keys_kernel, grid_of(n_edges), LP_THREADS, 0, src, tgt, is_transition,
               (const int*)in_component_x, n_ver, n_edges, w.pair_keys, w.pair_vals);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const unsigned long long*)w.pair_keys, w.pair_keys_sorted,
            (const int*)w.pair_vals, w.pair_vals_sorted, (int)n_edges, 0,
            bits_for((uint64_t)n_ver * (uint64_t)n_ver + 1), s);
    SPG_LAUNCH(K_LP_XPART, s, lp_xpart_weights_kernel, grid_of(n_edges), LP_THREADS, 0,
               (const unsigned long long*)w.pair_keys_sorted, (const int*)w.pair_vals_sorted, n_ver, n_edges,
               (const int*)comp_size, transition_factor, weights);
    return launch_status();
}

int spg_lp_seal(const int64_t* src, const int64_t* tgt, const uint8_t* is_transition, const int64_t* pred_in_component,
                const int64_t* objects, int64_t n_ver, int64_t n_edges, int64_t n_comp, double transition_factor,
                float* weights, int32_t* w_per_component, void* workspace, int64_t workspace_bytes,
                spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || n_comp < 0) return SPG_E_BADARG;
    if (lp_too_big(n_ver) || lp_too_big(n_edges) || n_comp >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t nmax = std::max(n_ver, n_comp);
    LpWs w;
    int rc = layout(n_ver, n_edges, n_comp, workspace, &w);
    if (rc != SPG_OK) return rc;
    if (nmax > 0) {
        if (n_ver > 0 && (!pred_in_component || !objects)) return SPG_E_BADARG;
        rc = ws_check(workspace, workspace_bytes, w.bytes);
        if (rc != SPG_OK) return rc;
        SPG_LAUNCH(K_LP_SEAL, s, lp_seal_keys_kernel, grid_of(nmax), LP_THREADS, 0, pred_in_component, objects, n_ver,
                   n_comp, w.comp_keys, w.size, w.maxfreq);
    }
    if (n_ver > 0) {
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortKeys, (const unsigned long long*)w.comp_keys, w.comp_keys_sorted,
                (int)n_ver, 0, 32 + bits_for((uint64_t)n_comp + 1), s);
        SPG_LAUNCH(K_LP_SEAL, s, lp_seal_runs_kernel, grid_of(n_ver), LP_THREADS, 0,
                   (const unsigned long long*)w.comp_keys_sorted, n_ver, n_comp, w.size, w.maxfreq);
    }
    const int64_t n2 = std::max(n_edges, w_per_component ? n_comp : 0);
    if (n2 == 0) return launch_status();
    if (n_edges > 0 && (!src || !tgt || !is_transition || !weights)) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_SEAL, s, lp_seal_weights_kernel, grid_of(n2), LP_THREADS, 0, src, tgt, is_transition,
               pred_in_component, n_ver, n_edges, n_comp, (const unsigned*)w.size, (const unsigned*)w.maxfreq,
               transition_factor, weights, w_per_component);
    return launch_status();
}

int spg_lp_fill_weights(const uint8_t* is_transition, int64_t n_edges, float w_other, float w_transition,
                        float* weights, spg_stream_t stream) {
    if (n_edges < 0) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!is_transition || !weights) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_WEIGHTS, (cudaStream_t)stream, lp_fill_weights_kernel, grid_of(n_edges), LP_THREADS, 0,
               is_transition, n_edges, w_other, w_transition, weights);
    return launch_status();
}

int spg_lp_count(const uint8_t* truth, const uint8_t* pred, int64_t n, int64_t* counts, spg_stream_t stream) {
    if (n < 0 || !counts) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n == 0) return SPG_OK;
    if (!truth) return SPG_E_BADARG;
    const int64_t blocks = std::min<int64_t>(ceil_div64(n, LP_THREADS), 4 * kNumSMs);
    SPG_LAUNCH(K_LP_METRICS, s, lp_count_kernel, (unsigned)blocks, LP_THREADS, 0, truth, pred, n,
               reinterpret_cast<unsigned long long*>(counts));
    return launch_status();
}

int spg_lp_edge_weight(const float* diff, int64_t n_edges, double threshold, double* edge_weight,
                       spg_stream_t stream) {
    if (n_edges < 0) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!diff || !edge_weight) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_WEIGHTS, (cudaStream_t)stream, lp_edge_weight_kernel, grid_of(n_edges), LP_THREADS, 0, diff,
               n_edges, threshold, edge_weight);
    return launch_status();
}

int spg_lp_relax(uint8_t* relaxed, const int64_t* src, const int64_t* tgt, int64_t n_ver, int64_t n_edges,
                 int tolerance, uint8_t* vertex_mark, int32_t* hit, int32_t* status, spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || !hit || !status) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(hit, 0, sizeof(int32_t), s);
    if (e == cudaSuccess && n_ver > 0 && vertex_mark) e = cudaMemsetAsync(vertex_mark, 0, (size_t)n_ver, s);
    if (e != cudaSuccess) return (int)e;
    if (n_edges == 0 || tolerance <= 0) return SPG_OK;
    if (!relaxed || !src || !tgt || (n_ver > 0 && !vertex_mark)) return SPG_E_BADARG;
    for (int it = 0; it < tolerance; ++it) {
        SPG_LAUNCH(K_LP_RELAX, s, lp_relax_mark_kernel, grid_of(n_edges), LP_THREADS, 0, (const uint8_t*)relaxed,
                   src, tgt, n_ver, n_edges, vertex_mark);
        SPG_LAUNCH(K_LP_RELAX, s, lp_relax_spread_kernel, grid_of(n_edges), LP_THREADS, 0, relaxed, src, tgt,
                   (const uint8_t*)vertex_mark, n_ver, n_edges, (int*)hit);
        SPG_LAUNCH(K_LP_RELAX, s, lp_relax_index_kernel, 1, 32, 0, relaxed, n_edges, (int*)hit, (int*)status);
    }
    return launch_status();
}

int spg_lp_perfect_prediction(const int64_t* comp_ptr, const int64_t* point_ids, int64_t n_comp,
                              const int64_t* labels, int64_t ld_labels, int n_classes, int64_t n_ver, int64_t* pred,
                              spg_stream_t stream) {
    if (n_comp < 0 || n_ver < 0 || n_classes <= 0 || ld_labels < n_classes + 1) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    if (n_ver > 0) {
        if (!pred) return SPG_E_BADARG;
        cudaError_t e = cudaMemsetAsync(pred, 0, (size_t)n_ver * sizeof(int64_t), s);
        if (e != cudaSuccess) return (int)e;
    }
    if (n_comp == 0) return SPG_OK;
    if (!comp_ptr || !point_ids || !labels) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_METRICS, s, lp_perfect_kernel, (unsigned)ceil_div64(n_comp * 32, LP_THREADS), LP_THREADS, 0,
               comp_ptr, point_ids, n_comp, labels, ld_labels, n_classes, n_ver, pred);
    return launch_status();
}

}  // extern "C"
