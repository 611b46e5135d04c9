// The l0 cut pursuit of both partition pipelines (ref: partition/cut-pursuit, CutPursuit.h with CutPursuit_L2.h
// for spatial = 0 and CutPursuit_SPG.h for spatial = 1, speed 4), one stage per entry point; the host runs the
// main loop (spg_cut_pursuit.py).  All state lives in one workspace laid out by `layout`:
//
//   cp_graph       the doubled arc list as a CSR (a stable CUB sort by tail vertex; duplicates kept), each arc
//                  with its reverse and its listed edge, and the input checks.
//   cp_members     vertices grouped by component, ascending id within a component (a stable sort by component).
//   cp_kmeans      2-means with k-means++ seeding and 10 restarts per unsaturated component of >= 2 vertices, one
//                  CTA of 512 threads per component of more than 2048 vertices, else one warp; Philox4x32-10 draws
//                  keyed by the seed, counter (iteration, root vertex, restart); fp64 sums.
//   cp_centers     the two centres of every unsaturated component (fp64 sums); one empty side saturates (L2).
//   cp_capacities  the reference's fp32 terminal and edge capacities.
//   cp_maxflow     a maximum preflow in 2^k fixed point (int64): synchronous lock-free push-relabel rounds with a
//                  global relabel (a breadth-first search from the sink in the residual graph) every 16 rounds,
//                  run once forward and once on the reversed problem.
//   cp_colour      sink tree = the vertices with a residual path to the sink (forward problem), source tree = the
//                  vertices reachable from the source (the reversed problem); the binary labels.
//   cp_activate    L2 saturation and edge activation by colour difference.
//   cp_split       connected components of the non-active graph (hooking to the minimum vertex and pointer
//                  jumping), numbered as the reference numbers them.
//   cp_merge       component values, the reduced graph's borders (sorted and reduced by component pair), fp64
//                  gains, the greedy one-merge-per-component selection as rounds of locally dominant borders, and
//                  the renumbering in kept order.
//   cp_energy      fidelity and penalty in fp64, reduced in a fixed order.
//
// Every stage takes the vertex weights mu (`nw`; CutPursuit_SPG.h's vertex weight): 1 for libcp.cutpursuit
// (cutpursuit.cpp:91), the caller's for libcp.cutpursuit2 (cutpursuit.cpp:107-128, spg_cp_node_weights).  Each
// weighted expression is written so that mu = 1 computes bit for bit what the unweighted one computes: products by
// mu are exact there, and where the unweighted form contracts to an FMA the weighted one is an explicit FMA of the
// same operands.  A vertex of weight 0 holds no observation: it adds nothing to any sum, its terminal capacities are
// 0, and a component whose weights are all 0 gets the value 0 / 0 = NaN, which never takes part in a merge (a NaN
// gain is no candidate).
#include <cub/cub.cuh>

#include "common.cuh"
#include "philox.cuh"
#include "workspace.cuh"

namespace spg {

constexpr int CP_T = 256;
constexpr int CP_BIG_T = 512;
constexpr int CP_BIG = 2048;             // components above this size get a CTA of CP_BIG_T threads
constexpr int CP_GR_ROUNDS = 16;         // push-relabel rounds between global relabels
constexpr int CP_BFS_BATCH = 16;         // BFS levels launched between read-backs
constexpr int64_t CP_MAX_BATCHES = 20000; // push-relabel batches before a flow is given up as an error
constexpr int CP_MAX_DIM = 32;
constexpr int64_t CP_CAP_MAX = 1ll << 61;

// scalar words of the workspace (int64)
enum CpWord { W_STATUS = 0, W_TMAX, W_COUNT, W_FLAG, W_NRUNS, W_NCAND, W_Q0, W_Q1, W_Q2, W_SAT, W_WEIGHTED, W_N };

struct CpWs {
    float *obs, *w, *cs, *ct, *ecap, *nw;
    int32_t *eu, *ev;
    uint8_t *active, *label, *plab, *colour, *sat, *sat2, *keep;
    int32_t *arc_off, *arc_dst, *arc_edge, *arc_rev;
    int64_t *res, *excess, *rt;
    int32_t *h, *q0, *q1;
    int32_t *comp, *pid, *parent, *members, *offsets, *root, *root2, *newid, *partner, *best, *nsink, *rank;
    double *value, *value2, *c0, *c1, *partial, *cw;
    uint32_t *ka, *kb;
    int32_t *va, *vb;
    uint64_t *bkey, *bkey2, *gkey, *gkey2;
    double *bw, *bw2, *gain;
    int32_t *gidx, *gidx2;
    int64_t* words;
    double* dwords;
    CubRegion cub;
    size_t bytes;
};

constexpr int CP_PARTIALS = 1024;

static int layout(int64_t n, int64_t E, int D, void* base, CpWs* w) {
    const int64_t A = 2 * E;
    const int64_t M = std::max<int64_t>(std::max<int64_t>(A, n), 1);
    const int Ei = (int)std::max<int64_t>(E, 1);
    size_t cb = 0;
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                  (const int32_t*)nullptr, (int32_t*)nullptr, (int)M);
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const double*)nullptr, (double*)nullptr, Ei);
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int32_t*)nullptr, (int32_t*)nullptr, Ei);
    SPG_CUB_BYTES(cb, cub::DeviceReduce::ReduceByKey, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const double*)nullptr, (double*)nullptr, (int64_t*)nullptr, cub::Sum(), Ei);
    SPG_CUB_BYTES(cb, cub::DeviceScan::ExclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n + 1);
    const size_t N = (size_t)n, ND = (size_t)n * D, En = (size_t)Ei, An = (size_t)std::max<int64_t>(A, 1);
    Planner p(base);
    w->obs = p.take<float>(ND);
    w->w = p.take<float>(En);
    w->cs = p.take<float>(N);
    w->ct = p.take<float>(N);
    w->ecap = p.take<float>(En);
    w->eu = p.take<int32_t>(En);
    w->ev = p.take<int32_t>(En);
    w->active = p.take<uint8_t>(En);
    w->label = p.take<uint8_t>(N);
    w->plab = p.take<uint8_t>(N);
    w->colour = p.take<uint8_t>(N);
    w->sat = p.take<uint8_t>(N);
    w->sat2 = p.take<uint8_t>(N);
    w->keep = p.take<uint8_t>(N);
    w->arc_off = p.take<int32_t>(N + 1);
    w->arc_dst = p.take<int32_t>(An);
    w->arc_edge = p.take<int32_t>(An);
    w->arc_rev = p.take<int32_t>(An);
    w->res = p.take<int64_t>(An);
    w->excess = p.take<int64_t>(N);
    w->rt = p.take<int64_t>(N);
    w->h = p.take<int32_t>(N);
    w->q0 = p.take<int32_t>(N);
    w->q1 = p.take<int32_t>(N);
    w->comp = p.take<int32_t>(N);
    w->pid = p.take<int32_t>(N);
    w->parent = p.take<int32_t>(N);
    w->members = p.take<int32_t>(N);
    w->offsets = p.take<int32_t>(N + 1);
    w->root = p.take<int32_t>(N);
    w->root2 = p.take<int32_t>(N);
    w->newid = p.take<int32_t>(N + 1);
    w->partner = p.take<int32_t>(N);
    w->best = p.take<int32_t>(N);
    w->nsink = p.take<int32_t>(N);
    w->rank = p.take<int32_t>(N + 1);
    w->value = p.take<double>(ND);
    w->value2 = p.take<double>(ND);
    w->c0 = p.take<double>(ND);
    w->c1 = p.take<double>(ND);
    w->partial = p.take<double>(2 * CP_PARTIALS);
    w->ka = p.take<uint32_t>((size_t)M);
    w->kb = p.take<uint32_t>((size_t)M);
    w->va = p.take<int32_t>((size_t)M);
    w->vb = p.take<int32_t>((size_t)M);
    w->bkey = p.take<uint64_t>(En);
    w->bkey2 = p.take<uint64_t>(En);
    w->gkey = p.take<uint64_t>(En);
    w->gkey2 = p.take<uint64_t>(En);
    w->bw = p.take<double>(En);
    w->bw2 = p.take<double>(En);
    w->gain = p.take<double>(En);
    w->gidx = p.take<int32_t>(En);
    w->gidx2 = p.take<int32_t>(En);
    w->nw = p.take<float>(N);
    w->cw = p.take<double>(N);
    w->words = p.take<int64_t>(W_N);
    w->dwords = p.take<double>(4);
    w->cub = p.cub(cb);
    w->bytes = p.bytes;
    return SPG_OK;
}

static int cp_bits(int64_t v) {
    int b = 1;
    while (b < 32 && (v >> b) != 0) ++b;
    return b;
}

static unsigned cp_grid(int64_t m, int t = CP_T) {
    const int64_t g = ceil_div64(m > 0 ? m : 1, t);
    return (unsigned)(g < 16 * kNumSMs ? g : 16 * kNumSMs);
}

#define CP_LOOP(i, m) for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (m); i += (int64_t)gridDim.x * blockDim.x)

// ------------------------------------------------------------------------------------------------ cp_graph
__global__ void cp_check_kernel(const float* __restrict__ obs, const int64_t* __restrict__ src,
                                const int64_t* __restrict__ tgt, const float* __restrict__ ew, int64_t n,
                                int64_t E, int D, int64_t* words) {
    unsigned st = 0;
    CP_LOOP(i, n * D) if (!isfinite(obs[i])) st |= 1u;
    CP_LOOP(e, E) {
        if (!isfinite(ew[e])) st |= 2u;
        if (src[e] < 0 || src[e] >= n || tgt[e] < 0 || tgt[e] >= n) st |= 4u;
    }
    if (st) atomicOr((unsigned long long*)words + W_STATUS, (unsigned long long)st);
}

__global__ void cp_copy_kernel(const float* __restrict__ obs, const int64_t* __restrict__ src,
                               const int64_t* __restrict__ tgt, const float* __restrict__ ew, int64_t n, int64_t E,
                               int D, CpWs w) {
    CP_LOOP(i, n * D) w.obs[i] = obs[i];
    CP_LOOP(e, E) {
        w.eu[e] = (int32_t)src[e];
        w.ev[e] = (int32_t)tgt[e];
        w.w[e] = ew[e];
        w.active[e] = 0;
        w.ka[e] = (uint32_t)src[e];      // arc e: u -> v, arc E + e: v -> u
        w.ka[E + e] = (uint32_t)tgt[e];
        w.va[e] = (int32_t)e;
        w.va[E + e] = (int32_t)(E + e);
    }
    CP_LOOP(v, n) {
        w.comp[v] = 0;
        w.sat[v] = 0;
        w.label[v] = 0;
        w.nw[v] = 1.f;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) w.root[0] = 0;
}

// spg_cp_node_weights: the caller's vertex weights; status 8 marks a negative or non-finite one
__global__ void cp_node_weights_kernel(const float* __restrict__ mu, int64_t n, CpWs w) {
    if (blockIdx.x == 0 && threadIdx.x == 0) w.words[W_WEIGHTED] = 1;
    unsigned st = 0;
    CP_LOOP(v, n) {
        const float m = mu[v];
        if (!isfinite(m) || m < 0.f) st |= 8u;
        w.nw[v] = m;
    }
    if (st) atomicOr((unsigned long long*)w.words + W_STATUS, (unsigned long long)st);
}

// lower bound of v in the sorted keys [0, m)
__device__ __forceinline__ int32_t cp_lower(const uint32_t* __restrict__ keys, int64_t m, uint32_t v) {
    int64_t lo = 0, hi = m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < v) lo = mid + 1; else hi = mid;
    }
    return (int32_t)lo;
}

__global__ void cp_arcs_kernel(int64_t n, int64_t E, CpWs w) {
    const int64_t A = 2 * E;
    CP_LOOP(p, A) {
        const int32_t j = w.vb[p];
        const int32_t e = j < E ? j : (int32_t)(j - E);
        w.arc_dst[p] = j < E ? w.ev[e] : w.eu[e];
        w.arc_edge[p] = e;
        w.va[j] = (int32_t)p;  // position of arc j
    }
    CP_LOOP(v, n + 1) w.arc_off[v] = cp_lower(w.kb, A, (uint32_t)v);
}

__global__ void cp_rev_kernel(int64_t E, CpWs w) {
    CP_LOOP(p, 2 * E) {
        const int32_t j = w.vb[p];
        w.arc_rev[p] = w.va[j < E ? j + E : j - E];
    }
}

// ------------------------------------------------------------------------------------------------ cp_members
__global__ void cp_iota_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) {
        w.ka[v] = (uint32_t)w.comp[v];
        w.va[v] = (int32_t)v;
    }
}

__global__ void cp_offsets_kernel(int64_t n, int64_t n_comp, CpWs w) {
    CP_LOOP(c, n_comp + 1) w.offsets[c] = cp_lower(w.kb, n, (uint32_t)c);
}

static int cp_members(const CpWs& w, int64_t n, int64_t n_comp, cudaStream_t s) {
    SPG_LAUNCH(K_CP_MEMBERS, s, cp_iota_kernel, cp_grid(n), CP_T, 0, n, w);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint32_t*)w.ka, w.kb, (const int32_t*)w.va, w.members,
            (int)n, 0, cp_bits(n_comp), s);
    SPG_LAUNCH(K_CP_MEMBERS, s, cp_offsets_kernel, cp_grid(n_comp + 1), CP_T, 0, n, n_comp, w);
    return launch_status();
}

// ------------------------------------------------------------------------------------------------ block helpers
// Components of more than CP_BIG vertices are served by the NT = CP_BIG_T instantiation, the others by NT = 32;
// every block of the other instantiation returns at once.
template <int NT>
__device__ __forceinline__ bool cp_mine(int size) {
    return NT == 32 ? size <= CP_BIG : size > CP_BIG;
}

// the block's sum, returned to every thread (CUB's reduction holds it in thread 0 only)
template <int NT>
__device__ __forceinline__ double cp_bsum(double v, void* tmp, double* bc) {
    typedef cub::BlockReduce<double, NT> R;
    const double r = R(*reinterpret_cast<typename R::TempStorage*>(tmp)).Sum(v);
    if (threadIdx.x == 0) *bc = r;
    __syncthreads();
    const double out = *bc;
    __syncthreads();
    return out;
}

// a vertex's weight in the per-component kernels, whose member-order gathers skip the load while every weight is 1
// (W_WEIGHTED unset: libcp.cutpursuit)
__device__ __forceinline__ double cp_mu(const CpWs& w, bool weighted, int32_t v) {
    return weighted ? (double)w.nw[v] : 1.0;
}

struct CpSum2 {
    __device__ __forceinline__ double2 operator()(const double2& a, const double2& b) const {
        return make_double2(a.x + b.x, a.y + b.y);
    }
};

// two sums of the block in one reduction, returned to every thread
template <int NT>
__device__ __forceinline__ double2 cp_bsum2(double2 v, void* tmp, double2* bc) {
    typedef cub::BlockReduce<double2, NT> R;
    const double2 r = R(*reinterpret_cast<typename R::TempStorage*>(tmp)).Reduce(v, CpSum2());
    if (threadIdx.x == 0) *bc = r;
    __syncthreads();
    const double2 out = *bc;
    __syncthreads();
    return out;
}

template <int NT>
struct CpShared {
    union {
        typename cub::BlockReduce<double, NT>::TempStorage red;
        typename cub::BlockReduce<double2, NT>::TempStorage red2;
        typename cub::BlockScan<double, NT>::TempStorage scan;
    } t;
    double k[2][CP_MAX_DIM];
    double bc;
    double2 bc2;
    int sel;
};

// compute_value (ref: CutPursuit_SPG.h:439-468): the component value = sum mu x / sum mu (fp64), cw = sum mu (the
// member count at mu = 1); a component whose weights are all 0 gets 0 / 0 = NaN
template <int NT>
__global__ void __launch_bounds__(NT) cp_values_kernel(int D, CpWs w) {
    __shared__ CpShared<NT> sh;
    const int c = blockIdx.x, off = w.offsets[c], size = w.offsets[c + 1] - off;
    if (!cp_mine<NT>(size)) return;
    const bool wt = w.words[W_WEIGHTED] != 0;
    double tw = (double)size;
    if (wt) {
        tw = 0.0;
        for (int i = threadIdx.x; i < size; i += NT) tw += (double)w.nw[w.members[off + i]];
        tw = cp_bsum<NT>(tw, &sh.t, &sh.bc);
    }
    if (threadIdx.x == 0) w.cw[c] = tw;
    for (int d = 0; d < D; ++d) {
        double s = 0.0;
        for (int i = threadIdx.x; i < size; i += NT) {
            const int32_t v = w.members[off + i];
            s = __fma_rn(cp_mu(w, wt, v), (double)w.obs[(int64_t)v * D + d], s);
        }
        s = cp_bsum<NT>(s, &sh.t, &sh.bc);
        if (threadIdx.x == 0) w.value[(int64_t)c * D + d] = s / tw;
    }
}

// ------------------------------------------------------------------------------------------------ cp_kmeans
template <int NT>
__device__ __forceinline__ double cp_d2(const float* __restrict__ x, const double* k, int D) {
    double s = 0.0;
    for (int d = 0; d < D; ++d) {
        const double t = (double)x[d] - k[d];
        s += t * t;
    }
    return s;
}

// init_labels (ref: CutPursuit_L2.h:111-261, CutPursuit_SPG.h:119-275): k-means++ seeding (first kernel the member
// at index u0 % size, the second the first member whose running sum of mu |x - k0|^2 exceeds E0 * u1 / 2^32,
// SPG.h:160-181), 5 Lloyd iterations with the reference's label convention (label = d0 > d1 on unweighted distances,
// SPG.h:191-200; label-true members feed kernel 0 with sums of mu x over sums of mu, SPG.h:202-244; a side of total
// weight 0 stops the iterations with undivided sums), and the restart's labels kept when its energy sum mu |x - k|^2
// is below E0 (SPG.h:247-272).
template <int NT>
__global__ void __launch_bounds__(NT) cp_kmeans_kernel(int D, int iteration, uint64_t seed, CpWs w) {
    __shared__ CpShared<NT> sh;
    const int c = blockIdx.x, off = w.offsets[c], size = w.offsets[c + 1] - off;
    if (!cp_mine<NT>(size) || size <= 1 || w.sat[c]) return;
    const bool wt = w.words[W_WEIGHTED] != 0;
    const int root = w.root[c];
    // contiguous chunk of member positions per thread (the running sum of the seeding is in member order)
    const int per = (size + NT - 1) / NT, lo = min(size, (int)threadIdx.x * per), hi = min(size, lo + per);
    uint8_t* plab = w.plab + off;
    const int32_t* mem = w.members + off;
    for (int r = 0; r < 10; ++r) {
        const Philox4 ph = philox4x32_10((uint32_t)iteration, (uint32_t)root, (uint32_t)r, 0u, (uint32_t)seed,
                                         (uint32_t)(seed >> 32));
        const int first = (int)(ph.v[0] % (uint32_t)size);
        const double u1 = (double)ph.v[1] * (1.0 / 4294967296.0);
        for (int d = threadIdx.x; d < D; d += NT) sh.k[0][d] = (double)w.obs[(int64_t)mem[first] * D + d];
        if (threadIdx.x == 0) sh.sel = size;
        __syncthreads();
        double loc = 0.0;
        for (int i = lo; i < hi; ++i)
            loc = __fma_rn(cp_mu(w, wt, mem[i]), cp_d2<NT>(w.obs + (int64_t)mem[i] * D, sh.k[0], D), loc);
        double before, e0;
        {
            typedef cub::BlockScan<double, NT> S;
            S(sh.t.scan).ExclusiveSum(loc, before, e0);
            __syncthreads();
        }
        const double target = e0 * u1;
        if (before + loc > target) {  // this chunk holds the crossing (the first chunk whose end exceeds target)
            double run = before;
            for (int i = lo; i < hi; ++i) {
                run = __fma_rn(cp_mu(w, wt, mem[i]), cp_d2<NT>(w.obs + (int64_t)mem[i] * D, sh.k[0], D), run);
                if (run > target) {
                    atomicMin(&sh.sel, i);
                    break;
                }
            }
        }
        __syncthreads();
        const int second = sh.sel < size ? sh.sel : 0;
        for (int d = threadIdx.x; d < D; d += NT) sh.k[1][d] = (double)w.obs[(int64_t)mem[second] * D + d];
        __syncthreads();
        for (int it = 0; it < 5; ++it) {
            double2 tw = make_double2(0.0, 0.0);  // the total weight of the label-true and label-false members
            for (int i = threadIdx.x; i < size; i += NT) {
                const float* x = w.obs + (int64_t)mem[i] * D;
                const uint8_t l = cp_d2<NT>(x, sh.k[0], D) > cp_d2<NT>(x, sh.k[1], D);
                plab[i] = l;
                if (l) tw.x += cp_mu(w, wt, mem[i]); else tw.y += cp_mu(w, wt, mem[i]);
            }
            tw = cp_bsum2<NT>(tw, &sh.t, &sh.bc2);
            const double n0 = tw.x, n1 = tw.y;
            for (int d = 0; d < D; ++d) {
                double s0 = 0.0, s1 = 0.0;
                for (int i = threadIdx.x; i < size; i += NT) {
                    const double x = (double)w.obs[(int64_t)mem[i] * D + d], m = cp_mu(w, wt, mem[i]);
                    if (plab[i]) s0 = __fma_rn(m, x, s0); else s1 = __fma_rn(m, x, s1);
                }
                s0 = cp_bsum<NT>(s0, &sh.t, &sh.bc);
                s1 = cp_bsum<NT>(s1, &sh.t, &sh.bc);
                if (threadIdx.x == 0) {
                    const bool empty = n0 == 0.0 || n1 == 0.0;
                    sh.k[0][d] = empty ? s0 : s0 / n0;
                    sh.k[1][d] = empty ? s1 : s1 / n1;
                }
            }
            __syncthreads();
            if (n0 == 0.0 || n1 == 0.0) break;
        }
        double en = 0.0;
        for (int i = threadIdx.x; i < size; i += NT)
            en = __fma_rn(cp_mu(w, wt, mem[i]), cp_d2<NT>(w.obs + (int64_t)mem[i] * D, sh.k[plab[i] ? 0 : 1], D), en);
        en = cp_bsum<NT>(en, &sh.t, &sh.bc);
        if (en < e0)
            for (int i = threadIdx.x; i < size; i += NT) w.label[mem[i]] = plab[i];
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ cp_centers
// compute_center (ref: CutPursuit_L2.h:284-339, CutPursuit_SPG.h:298-352): the weighted means of the label-true
// (c0) and label-false (c1) members; a side of total weight 0 gives c0 = c1 = the component value and saturates the
// component in L2.
template <int NT>
__global__ void __launch_bounds__(NT) cp_centers_kernel(int D, int spatial, CpWs w) {
    __shared__ CpShared<NT> sh;
    const int c = blockIdx.x, off = w.offsets[c], size = w.offsets[c + 1] - off;
    if (!cp_mine<NT>(size) || w.sat[c]) return;
    const bool wt = w.words[W_WEIGHTED] != 0;
    const int32_t* mem = w.members + off;
    double2 tw = make_double2(0.0, 0.0);
    for (int i = threadIdx.x; i < size; i += NT) {
        if (w.label[mem[i]]) tw.x += cp_mu(w, wt, mem[i]); else tw.y += cp_mu(w, wt, mem[i]);
    }
    tw = cp_bsum2<NT>(tw, &sh.t, &sh.bc2);
    const double n0 = tw.x, n1 = tw.y;
    const bool empty = n0 == 0.0 || n1 == 0.0;
    for (int d = 0; d < D; ++d) {
        double s0 = 0.0, s1 = 0.0;
        if (!empty)
            for (int i = threadIdx.x; i < size; i += NT) {
                const double x = (double)w.obs[(int64_t)mem[i] * D + d], m = cp_mu(w, wt, mem[i]);
                if (w.label[mem[i]]) s0 = __fma_rn(m, x, s0); else s1 = __fma_rn(m, x, s1);
            }
        s0 = cp_bsum<NT>(s0, &sh.t, &sh.bc);
        s1 = cp_bsum<NT>(s1, &sh.t, &sh.bc);
        if (threadIdx.x == 0) {
            const int64_t k = (int64_t)c * D + d;
            w.c0[k] = empty ? w.value[k] : s0 / n0;
            w.c1[k] = empty ? w.value[k] : s1 / n1;
        }
    }
    if (threadIdx.x == 0 && empty && !spatial) w.sat[c] = 1;
}

// ------------------------------------------------------------------------------------------------ cp_capacities
// set_capacities (ref: CutPursuit_L2.h:343-417, CutPursuit_SPG.h:360-435): with cb = float(c0), cn = float(c1),
// cost_B = float(cost_B + (0.5 mu) (cb cb - float(2 float(cb x)))) per dimension in fp64, the same for cost_notB; the
// source arc carries cost_B - cost_notB when positive, else the sink arc carries cost_notB - cost_B (fp32).  A
// saturated component (saturateComponent) and a vertex of weight 0 (SPG.h:388-393) get 0 on both.  Edge:
// float(w lambda) when not active (SPG: divided by unary), 0 when active.  W_TMAX = the largest terminal capacity
// (float bits).
__global__ void cp_capacities_kernel(int64_t n, int64_t E, int D, float lambda, float unary, int spatial, CpWs w) {
    unsigned tmax = 0;
    CP_LOOP(v, n) {
        const int c = w.comp[v];
        const float mu = w.nw[v];
        float s = 0.f, t = 0.f;
        if (!w.sat[c] && mu != 0.f) {
            const double hm = __dmul_rn(0.5, (double)mu);
            float cost_b = 0.f, cost_n = 0.f;
            for (int d = 0; d < D; ++d) {
                const float x = w.obs[v * D + d];
                const float cb = (float)w.c0[(int64_t)c * D + d], cn = (float)w.c1[(int64_t)c * D + d];
                const double tb = __dmul_rn(hm, __dsub_rn(__dmul_rn((double)cb, (double)cb),
                                                          (double)__fmul_rn(2.f, __fmul_rn(cb, x))));
                const double tn = __dmul_rn(hm, __dsub_rn(__dmul_rn((double)cn, (double)cn),
                                                          (double)__fmul_rn(2.f, __fmul_rn(cn, x))));
                cost_b = (float)__dadd_rn((double)cost_b, tb);
                cost_n = (float)__dadd_rn((double)cost_n, tn);
            }
            if (cost_b > cost_n) s = __fsub_rn(cost_b, cost_n);
            else t = __fsub_rn(cost_n, cost_b);
        }
        w.cs[v] = s;
        w.ct[v] = t;
        tmax = max(tmax, max(__float_as_uint(s), __float_as_uint(t)));
    }
    if (tmax) atomicMax((unsigned long long*)w.words + W_TMAX, (unsigned long long)tmax);
    CP_LOOP(e, E) {
        const float c = __fmul_rn(w.w[e], lambda);
        w.ecap[e] = w.active[e] ? 0.f : (spatial ? __fdiv_rn(c, unary) : c);
    }
}

// ------------------------------------------------------------------------------------------------ cp_maxflow
// Fixed point: a capacity c becomes rint(c 2^k), k = min(40, 61 - e) with n tmax < 2^e, so that the terminal
// capacities sum below 2^61; arc capacities are clamped at 2^61, above every cut through the terminals alone.
__device__ __forceinline__ int cp_shift(const int64_t* words, int64_t n) {
    const double b = (double)__uint_as_float((unsigned)words[W_TMAX]) * (double)n;
    if (b == 0.0) return 40;
    int e;
    frexp(b, &e);
    return min(40, 61 - e);
}

__device__ __forceinline__ int64_t cp_fix(float c, int k) {
    const double q = rint(ldexp((double)c, k));
    return q >= (double)CP_CAP_MAX ? CP_CAP_MAX : (int64_t)q;
}

__global__ void cp_flow_init_kernel(int64_t n, int reverse, CpWs w) {
    const int k = cp_shift(w.words, n);
    CP_LOOP(v, n) {
        w.excess[v] = cp_fix(reverse ? w.ct[v] : w.cs[v], k);
        w.rt[v] = cp_fix(reverse ? w.cs[v] : w.ct[v], k);
        const int32_t a = w.arc_off[v], b = w.arc_off[v + 1];
        for (int32_t p = a; p < b; ++p) w.res[p] = cp_fix(w.ecap[w.arc_edge[p]], k);
    }
}

// BFS from the sink in the residual graph: h = distance, n where the sink is unreachable.  Level 0 is seeded
// by cp_bfs_seed_kernel; level L reads queue L & 1 (count W_Q0 + L % 3), writes the other queue and clears the
// count of level L + 2.
__global__ void cp_bfs_seed_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) {
        const bool s = w.rt[v] > 0;
        w.h[v] = s ? 1 : (int32_t)n;
        if (s) w.q0[atomicAdd((unsigned long long*)w.words + W_Q0, 1ull)] = (int32_t)v;
    }
}

__global__ void cp_bfs_level_kernel(int64_t n, int level, CpWs w) {
    const int64_t cnt = w.words[W_Q0 + level % 3];
    const int32_t* qin = (level & 1) ? w.q1 : w.q0;
    int32_t* qout = (level & 1) ? w.q0 : w.q1;
    if (blockIdx.x == 0 && threadIdx.x == 0) w.words[W_Q0 + (level + 2) % 3] = 0;
    const int32_t hn = level + 2;
    CP_LOOP(i, cnt) {
        const int32_t x = qin[i];
        for (int32_t p = w.arc_off[x]; p < w.arc_off[x + 1]; ++p) {
            const int32_t y = w.arc_dst[p];
            if (w.res[w.arc_rev[p]] > 0 && w.h[y] == (int32_t)n && atomicCAS(&w.h[y], (int32_t)n, hn) == (int32_t)n)
                qout[atomicAdd((unsigned long long*)w.words + W_Q0 + (level + 1) % 3, 1ull)] = y;
        }
    }
}

// One synchronous round of the lock-free push-relabel (Hong, 2008): every active vertex (excess > 0, h < n)
// pushes to its lowest residual neighbour (the sink has height 0) when it is higher, else relabels to one above
// it.  W_COUNT counts the active vertices.
__global__ void cp_push_kernel(int64_t n, CpWs w) {
    unsigned long long act = 0;
    CP_LOOP(u, n) {
        const int64_t ex = w.excess[u];
        const int32_t hu = w.h[u];
        if (ex <= 0 || hu >= (int32_t)n) continue;
        ++act;
        int32_t hmin = w.rt[u] > 0 ? 0 : (int32_t)n, best = -1;
        for (int32_t p = w.arc_off[u]; p < w.arc_off[u + 1] && hmin > 0; ++p) {
            if (w.res[p] <= 0 || w.arc_dst[p] == u) continue;  // a self-loop arc carries nothing
            const int32_t hv = w.h[w.arc_dst[p]];
            if (hv < hmin) {
                hmin = hv;
                best = p;
            }
        }
        if (hu > hmin) {
            if (best < 0) {
                const int64_t d = min(ex, w.rt[u]);
                w.rt[u] -= d;
                atomicAdd((unsigned long long*)&w.excess[u], (unsigned long long)(-d));
            } else {
                const int64_t d = min(ex, w.res[best]);
                atomicAdd((unsigned long long*)&w.res[best], (unsigned long long)(-d));
                atomicAdd((unsigned long long*)&w.res[w.arc_rev[best]], (unsigned long long)d);
                atomicAdd((unsigned long long*)&w.excess[u], (unsigned long long)(-d));
                atomicAdd((unsigned long long*)&w.excess[w.arc_dst[best]], (unsigned long long)d);
            }
        } else {
            w.h[u] = hmin >= (int32_t)n - 1 ? (int32_t)n : hmin + 1;
        }
    }
    if (act) atomicAdd((unsigned long long*)w.words + W_COUNT, act);
}

// colour (ref: Boykov-Kolmogorov's trees, CutPursuit.h:300-325): forward pass: 4 (sink tree) where the sink
// is reachable, else 1 (free); reverse pass: 0 (source tree) where the reversed sink is reachable.  The binary
// label of an unsaturated component's vertex is colour == sink.
__global__ void cp_colour_kernel(int64_t n, int reverse, CpWs w) {
    CP_LOOP(v, n) {
        const bool hit = w.h[v] < (int32_t)n;
        if (!reverse) {
            w.colour[v] = hit ? 4 : 1;
        } else {
            if (hit) w.colour[v] = 0;
            if (!w.sat[w.comp[v]]) w.label[v] = w.colour[v] == 4;
        }
    }
}

template <class T>
static int cp_read(T* dst, const T* src, int count, cudaStream_t s) {
    cudaError_t e = cudaMemcpyAsync(dst, src, sizeof(T) * count, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return (int)e;
}

// the sink-reachability BFS; h = distance or n
static int cp_bfs(const CpWs& w, int64_t n, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(w.words + W_Q0, 0, 3 * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_MAXFLOW, s, cp_bfs_seed_kernel, cp_grid(n), CP_T, 0, n, w);
    for (int level = 0;; level += CP_BFS_BATCH) {
        for (int l = level; l < level + CP_BFS_BATCH; ++l)
            SPG_LAUNCH(K_CP_MAXFLOW, s, cp_bfs_level_kernel, cp_grid(n), CP_T, 0, n, l, w);
        int64_t q[3];
        int rc = cp_read(q, w.words + W_Q0, 3, s);
        if (rc != SPG_OK) return rc;
        if (q[(level + CP_BFS_BATCH) % 3] == 0) break;
    }
    return launch_status();
}

// a maximum preflow of one direction; rounds += the push-relabel rounds run
static int cp_flow(const CpWs& w, int64_t n, int reverse, int64_t* rounds, cudaStream_t s) {
    SPG_LAUNCH(K_CP_MAXFLOW, s, cp_flow_init_kernel, cp_grid(n), CP_T, 0, n, reverse, w);
    for (int64_t batch = 0;; ++batch) {
        if (batch > CP_MAX_BATCHES) return SPG_E_UNSUPPORTED;  // no preflow after that many rounds
        int rc = cp_bfs(w, n, s);
        if (rc != SPG_OK) return rc;
        cudaError_t e = cudaMemsetAsync(w.words + W_COUNT, 0, sizeof(int64_t), s);
        if (e != cudaSuccess) return (int)e;
        for (int r = 0; r < CP_GR_ROUNDS; ++r)
            SPG_LAUNCH(K_CP_MAXFLOW, s, cp_push_kernel, cp_grid(n), CP_T, 0, n, w);
        *rounds += CP_GR_ROUNDS;
        int64_t act;
        rc = cp_read(&act, w.words + W_COUNT, 1, s);
        if (rc != SPG_OK) return rc;
        if (act == 0) break;
    }
    return cp_bfs(w, n, s);  // the final heights: h < n exactly on the vertices with a residual path to the sink
}

// ------------------------------------------------------------------------------------------------ cp_activate
__global__ void cp_sink_count_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) if (w.colour[v] == 4 && !w.sat[w.comp[v]]) atomicAdd(&w.nsink[w.comp[v]], 1);
}

// activate_edges (ref: CutPursuit.h:256-327): L2 saturates a component whose vertices all lie on one side of
// the sink tree; an edge whose endpoints differ in colour becomes active.  W_SAT = vertices in saturated
// components.
__global__ void cp_activate_kernel(int64_t n, int64_t E, int64_t n_comp, int spatial, CpWs w) {
    CP_LOOP(c, n_comp) {
        const int size = w.offsets[c + 1] - w.offsets[c];
        if (!spatial && !w.sat[c] && (w.nsink[c] == 0 || w.nsink[c] == size)) w.sat[c] = 1;
    }
    CP_LOOP(e, E) if (w.colour[w.eu[e]] != w.colour[w.ev[e]]) w.active[e] = 1;
}

__global__ void cp_sat_count_kernel(int64_t n_comp, CpWs w) {
    unsigned long long s = 0;
    CP_LOOP(c, n_comp) if (w.sat[c]) s += (unsigned long long)(w.offsets[c + 1] - w.offsets[c]);
    if (s) atomicAdd((unsigned long long*)w.words + W_SAT, s);
}

// ------------------------------------------------------------------------------------------------ cp_split
__device__ __forceinline__ int32_t cp_find(const int32_t* parent, int32_t x) {
    int32_t p;
    while ((p = parent[x]) != x) x = p;
    return x;
}

__global__ void cp_cc_init_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) {
        w.parent[v] = (int32_t)v;
        w.pid[v] = -1;
    }
}

__global__ void cp_hook_kernel(int64_t E, CpWs w) {
    unsigned long long changed = 0;
    CP_LOOP(e, E) {
        if (w.active[e]) continue;
        const int32_t u = w.eu[e], v = w.ev[e];
        if (w.sat[w.comp[u]] || w.sat[w.comp[v]]) continue;
        const int32_t ru = cp_find(w.parent, u), rv = cp_find(w.parent, v);
        if (ru == rv) continue;
        atomicMin(&w.parent[max(ru, rv)], min(ru, rv));
        changed = 1;
    }
    if (changed) w.words[W_FLAG] = 1;
}

__global__ void cp_jump_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) w.parent[v] = cp_find(w.parent, (int32_t)v);
}

// the piece holding an unsaturated component's root keeps the component's index (ref: CutPursuit.h:349-400)
__global__ void cp_old_roots_kernel(int64_t n_comp, CpWs w) {
    CP_LOOP(c, n_comp) if (!w.sat[c]) w.pid[w.parent[w.root[c]]] = (int32_t)c;
}

__global__ void cp_new_flags_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n + 1) w.rank[v] = (v < n && !w.sat[w.comp[v]] && w.parent[v] == v && w.pid[v] < 0) ? 1 : 0;
}

__global__ void cp_count_new_kernel(int64_t n, CpWs w) { w.words[W_COUNT] = w.newid[n]; }

// other pieces are appended in the order of their smallest vertex, which becomes their root
__global__ void cp_new_ids_kernel(int64_t n, int64_t n_comp, CpWs w) {
    CP_LOOP(v, n) {
        if (!w.sat[w.comp[v]] && w.parent[v] == v && w.pid[v] < 0) {
            const int32_t id = (int32_t)n_comp + w.newid[v];
            w.pid[v] = id;
            w.root[id] = (int32_t)v;
            w.sat[id] = 0;
        }
    }
}

__global__ void cp_assign_kernel(int64_t n, int64_t n_comp, CpWs w) {
    CP_LOOP(v, n) {
        const int32_t c = w.comp[v];
        if (c < n_comp && w.sat[c]) continue;  // saturated components keep their members
        w.comp[v] = w.pid[w.parent[v]];
    }
}

// ------------------------------------------------------------------------------------------------ cp_merge
__device__ __forceinline__ uint64_t cp_dkey(double g) {
    if (g == 0.0) g = 0.0;  // -0 and +0 are one gain
    const uint64_t u = (uint64_t)__double_as_longlong(g);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

// the merged value and the fidelity change of one dimension, rounded op by op (no contraction), as the oracle
// computes them: m = (w1 v1 + w2 v2) / (w1 + w2), 0.5 (m m (w1 + w2) - v1 v1 w1 - v2 v2 w2)
__device__ __forceinline__ double cp_merged(double v1, double v2, double w1, double w2) {
    return __ddiv_rn(__dadd_rn(__dmul_rn(w1, v1), __dmul_rn(w2, v2)), __dadd_rn(w1, w2));
}

__device__ __forceinline__ double cp_merge_term(double v1, double v2, double w1, double w2) {
    const double m = cp_merged(v1, v2, w1, w2);
    const double t = __dsub_rn(__dsub_rn(__dmul_rn(__dmul_rn(m, m), __dadd_rn(w1, w2)), __dmul_rn(__dmul_rn(v1, v1), w1)),
                               __dmul_rn(__dmul_rn(v2, v2), w2));
    return __dmul_rn(0.5, t);
}

__global__ void cp_border_keys_kernel(int64_t E, CpWs w) {
    CP_LOOP(e, E) {
        const uint32_t a = (uint32_t)w.comp[w.eu[e]], b = (uint32_t)w.comp[w.ev[e]];
        w.bkey[e] = a == b ? ~0ull : ((uint64_t)min(a, b) << 32 | max(a, b));
        w.bw[e] = (double)w.w[e];
    }
}

// compute_merge_gain (ref: CutPursuit_L2.h:455-481, CutPursuit_SPG.h:473-498) with the component weights cw +
// lambda * border weight; candidates: gain > 0, or with is_cutoff either side weighing <= cutoff (CutPursuit.h:
// 473-478).  A gain with a NaN-valued component is NaN and never a candidate, so it takes no place in the ranking.
// gkey sorts candidates by descending gain; ties keep the ascending (comp1, comp2) order of the borders.
__global__ void cp_gain_kernel(int64_t n_runs, int D, double lambda, double cutoff, int is_cutoff, CpWs w) {
    CP_LOOP(b, n_runs) {
        const uint64_t key = w.bkey[b];
        bool cand = false;
        double g = 0.0;
        if (key != ~0ull) {
            const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
            const double w1 = w.cw[c1], w2 = w.cw[c2];
            for (int d = 0; d < D; ++d) {
                const double v1 = w.value[(int64_t)c1 * D + d], v2 = w.value[(int64_t)c2 * D + d];
                g = __dadd_rn(g, cp_merge_term(v1, v2, w1, w2));
            }
            g = __dadd_rn(g, __dmul_rn(w.bw[b], lambda));
            cand = is_cutoff ? (w1 <= cutoff || w2 <= cutoff) && !isnan(g) : g > 0.0;
        }
        w.gain[b] = g;
        w.gkey[b] = cand ? ~cp_dkey(g) : ~0ull;
        w.gidx[b] = (int32_t)b;
        if (cand) atomicAdd((unsigned long long*)w.words + W_NCAND, 1ull);
    }
}

__global__ void cp_match_init_kernel(int64_t n_comp, CpWs w) {
    CP_LOOP(c, n_comp) {
        w.partner[c] = -1;
        w.best[c] = INT_MAX;
    }
}

// one round of the greedy matching: every free component takes the best-ranked candidate still free at both
// ends; a candidate best at both of its components is selected.  The selections of all rounds are exactly the
// ones the sequential pass down the sorted list makes.
__global__ void cp_match_best_kernel(int64_t n_cand, CpWs w) {
    CP_LOOP(p, n_cand) {
        const uint64_t key = w.bkey[w.gidx2[p]];
        const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
        if (w.partner[c1] >= 0 || w.partner[c2] >= 0) continue;
        atomicMin(&w.best[c1], (int)p);
        atomicMin(&w.best[c2], (int)p);
    }
}

__global__ void cp_match_take_kernel(int64_t n_cand, CpWs w) {
    unsigned long long took = 0;
    CP_LOOP(p, n_cand) {
        const uint64_t key = w.bkey[w.gidx2[p]];
        const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
        if (w.best[c1] == (int)p && w.best[c2] == (int)p) {
            w.partner[c1] = c2;
            w.partner[c2] = c1;
            ++took;
        }
    }
    if (took) atomicAdd((unsigned long long*)w.words + W_COUNT, took);
}

__global__ void cp_best_reset_kernel(int64_t n_comp, CpWs w) {
    CP_LOOP(c, n_comp) w.best[c] = INT_MAX;
}

// merge (ref: CutPursuit.h:531-662): comp2 joins comp1 (comp1 < comp2), comp1 takes the merged value (weighted by
// cw, CutPursuit.h:578-619) and is no longer saturated, the border between them is deactivated; the kept components
// are renumbered in order.  cw is not carried over: the next merge recomputes it with the values.
__global__ void cp_merge_apply_kernel(int64_t n_comp, int D, CpWs w) {
    CP_LOOP(c, n_comp + 1) {
        if (c == n_comp) {
            w.newid[c] = 0;
            continue;
        }
        const int q = w.partner[c];
        w.newid[c] = !(q >= 0 && q < c);
        if (q > c) {
            const double w1 = w.cw[c], w2 = w.cw[q];
            for (int d = 0; d < D; ++d) {
                const double v1 = w.value[(int64_t)c * D + d], v2 = w.value[(int64_t)q * D + d];
                w.value[(int64_t)c * D + d] = cp_merged(v1, v2, w1, w2);
            }
            w.sat[c] = 0;
        }
    }
}

__global__ void cp_deactivate_kernel(int64_t E, CpWs w) {
    CP_LOOP(e, E) {
        const int a = w.comp[w.eu[e]], b = w.comp[w.ev[e]];
        if (a != b && w.partner[a] == b) w.active[e] = 0;
    }
}

__global__ void cp_renumber_kernel(int64_t n_comp, int D, CpWs w) {
    CP_LOOP(c, n_comp) {
        const int q = w.partner[c];
        if (q >= 0 && q < c) continue;
        const int id = w.pid[c];
        w.root2[id] = w.root[c];
        w.sat2[id] = w.sat[c];
        for (int d = 0; d < D; ++d) w.value2[(int64_t)id * D + d] = w.value[(int64_t)c * D + d];
    }
}

__global__ void cp_recomp_kernel(int64_t n, CpWs w) {
    CP_LOOP(v, n) {
        const int c = w.comp[v], q = w.partner[c];
        w.comp[v] = w.pid[q >= 0 && q < c ? q : c];
    }
}

// ------------------------------------------------------------------------------------------------ cp_energy
// compute_energy (ref: CutPursuit_L2.h:15-49, CutPursuit_SPG.h:25-34): sum 0.5 mu |x - value|^2 + lambda sum over
// active listed edges of w (each listed edge is two arcs of 0.5 lambda w), fp64, partial sums per thread block
// reduced in a fixed order.  A NaN-valued component makes it NaN, 0 NaN included.
__global__ void __launch_bounds__(CP_T) cp_energy_kernel(int64_t n, int64_t E, int D, CpWs w) {
    typedef cub::BlockReduce<double, CP_T> R;
    __shared__ typename R::TempStorage tmp;
    double f = 0.0, p = 0.0;
    CP_LOOP(v, n) {
        const int c = w.comp[v];
        const double hm = __dmul_rn(0.5, (double)w.nw[v]);
        for (int d = 0; d < D; ++d) {
            const double t = (double)w.obs[v * D + d] - w.value[(int64_t)c * D + d];
            f = __fma_rn(__dmul_rn(hm, t), t, f);
        }
    }
    CP_LOOP(e, E) if (w.active[e]) p += (double)w.w[e];
    f = R(tmp).Sum(f);
    __syncthreads();
    p = R(tmp).Sum(p);
    if (threadIdx.x == 0) {
        w.partial[blockIdx.x] = f;
        w.partial[CP_PARTIALS + blockIdx.x] = p;
    }
}

__global__ void __launch_bounds__(CP_T) cp_energy_final_kernel(int nb, double lambda, CpWs w) {
    typedef cub::BlockReduce<double, CP_T> R;
    __shared__ typename R::TempStorage tmp;
    double f = 0.0, p = 0.0;
    for (int i = threadIdx.x; i < nb; i += CP_T) {
        f += w.partial[i];
        p += w.partial[CP_PARTIALS + i];
    }
    f = R(tmp).Sum(f);
    __syncthreads();
    p = R(tmp).Sum(p);
    if (threadIdx.x == 0) {
        w.dwords[0] = f;
        w.dwords[1] = p;
        w.dwords[2] = f + lambda * p;
    }
}

__global__ void cp_output_kernel(int64_t n, int64_t n_comp, CpWs w, int64_t* in_component, int64_t* offsets,
                                 int64_t* members) {
    CP_LOOP(v, n) {
        in_component[v] = w.comp[v];
        members[v] = w.members[v];
    }
    CP_LOOP(c, n_comp + 1) offsets[c] = w.offsets[c];
}

// ------------------------------------------------------------------------------------------------ plumbing
static int cp_setup_ws(int64_t n, int64_t E, int D, void* ws, int64_t bytes, CpWs* w) {
    if (n <= 0 || E < 0 || D < 1 || D > CP_MAX_DIM) return SPG_E_BADARG;
    if (too_big(2 * E + 1) || too_big(n * D + 1)) return SPG_E_UNSUPPORTED;
    const int rc = layout(n, E, D, ws, w);
    return rc == SPG_OK ? ws_check(ws, bytes, w->bytes) : rc;
}

#define CP_PER_COMP(kid, s, n_comp, kernel, ...)                                                      \
    do {                                                                                             \
        SPG_LAUNCH(kid, s, kernel<32>, (unsigned)(n_comp), 32, 0, __VA_ARGS__);                      \
        SPG_LAUNCH(kid, s, kernel<CP_BIG_T>, (unsigned)(n_comp), CP_BIG_T, 0, __VA_ARGS__);          \
    } while (0)

}  // namespace spg

using namespace spg;

#define CP_WS(n, E, D, ws, bytes)                            \
    CpWs w;                                                  \
    {                                                        \
        const int rc_ = cp_setup_ws(n, E, D, ws, bytes, &w); \
        if (rc_ != SPG_OK) return rc_;                       \
    }                                                        \
    cudaStream_t s = (cudaStream_t)stream;

extern "C" {

int spg_cp_workspace(int64_t n, int64_t n_edges, int dim, int64_t* bytes) {
    if (!bytes || n <= 0 || n_edges < 0 || dim < 1 || dim > CP_MAX_DIM) return SPG_E_BADARG;
    if (too_big(2 * n_edges + 1) || too_big(n * dim + 1)) return SPG_E_UNSUPPORTED;
    CpWs w;
    const int rc = layout(n, n_edges, dim, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_cp_regions(int64_t n, int64_t n_edges, int dim, int64_t* offsets) {
    if (!offsets || n <= 0 || n_edges < 0 || dim < 1 || dim > CP_MAX_DIM) return SPG_E_BADARG;
    CpWs w;
    const int rc = layout(n, n_edges, dim, nullptr, &w);
    if (rc != SPG_OK) return rc;
    const void* r[] = {w.obs, w.comp, w.root, w.sat, w.label, w.colour, w.active, w.value, w.c0, w.c1,
                       w.cs, w.ct, w.ecap, w.members, w.offsets, w.words, w.dwords, w.partner,
                       w.res, w.excess, w.rt, w.arc_off, w.arc_dst, w.arc_rev, w.arc_edge, w.nw, w.cw};
    for (size_t i = 0; i < sizeof(r) / sizeof(r[0]); ++i) offsets[i] = (int64_t)(uintptr_t)r[i];
    return SPG_OK;
}

int spg_cp_setup(const float* obs, const int64_t* source, const int64_t* target, const float* edge_weight,
                 int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t* out,
                 spg_stream_t stream) {
    if (!obs || !out || (n_edges > 0 && (!source || !target || !edge_weight))) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    const int64_t E = n_edges;
    cudaError_t e = cudaMemsetAsync(w.words, 0, W_N * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_GRAPH, s, cp_check_kernel, cp_grid(n * dim + E), CP_T, 0, obs, source, target, edge_weight, n,
               E, dim, w.words);
    int rc = cp_read(out, w.words + W_STATUS, 1, s);
    if (rc != SPG_OK || out[0] != 0) return rc;
    SPG_LAUNCH(K_CP_GRAPH, s, cp_copy_kernel, cp_grid(n * dim + E), CP_T, 0, obs, source, target, edge_weight, n, E,
               dim, w);
    if (E > 0) {
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint32_t*)w.ka, w.kb, (const int32_t*)w.va, w.vb,
                (int)(2 * E), 0, cp_bits(n), s);
    }
    SPG_LAUNCH(K_CP_GRAPH, s, cp_arcs_kernel, cp_grid(2 * E + n + 1), CP_T, 0, n, E, w);
    SPG_LAUNCH(K_CP_GRAPH, s, cp_rev_kernel, cp_grid(2 * E), CP_T, 0, E, w);
    rc = cp_members(w, n, 1, s);
    if (rc != SPG_OK) return rc;
    CP_PER_COMP(K_CP_MERGE, s, 1, cp_values_kernel, dim, w);
    return launch_status();
}

int spg_cp_node_weights(const float* node_weight, int64_t n, int64_t n_edges, int dim, void* workspace,
                        int64_t workspace_bytes, int64_t* out, spg_stream_t stream) {
    if (!node_weight || !out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    cudaError_t e = cudaMemsetAsync(w.words + W_STATUS, 0, sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_GRAPH, s, cp_node_weights_kernel, cp_grid(n), CP_T, 0, node_weight, n, w);
    const int rc = cp_read(out, w.words + W_STATUS, 1, s);
    if (rc != SPG_OK || out[0] != 0) return rc;
    CP_PER_COMP(K_CP_MERGE, s, 1, cp_values_kernel, dim, w);
    return launch_status();
}

int spg_cp_members(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                   spg_stream_t stream) {
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    return cp_members(w, n, n_comp, s);
}

int spg_cp_kmeans(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                  int64_t iteration, int64_t seed, spg_stream_t stream) {
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    cudaError_t e = cudaMemsetAsync(w.label, 0, (size_t)n, s);
    if (e != cudaSuccess) return (int)e;
    CP_PER_COMP(K_CP_KMEANS, s, n_comp, cp_kmeans_kernel, dim, (int)iteration, (uint64_t)seed, w);
    return launch_status();
}

int spg_cp_centers(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                   int spatial, spg_stream_t stream) {
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    CP_PER_COMP(K_CP_CENTERS, s, n_comp, cp_centers_kernel, dim, spatial, w);
    return launch_status();
}

int spg_cp_capacities(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes,
                      float reg_strength, float unary, int spatial, spg_stream_t stream) {
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    cudaError_t e = cudaMemsetAsync(w.words + W_TMAX, 0, sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_CAPACITIES, s, cp_capacities_kernel, cp_grid(n + n_edges), CP_T, 0, n, n_edges, dim,
               reg_strength, unary, spatial, w);
    return launch_status();
}

int spg_cp_maxflow(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t* out,
                   spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    out[0] = 0;
    for (int reverse = 0; reverse < 2; ++reverse) {
        const int rc = cp_flow(w, n, reverse, out, s);
        if (rc != SPG_OK) return rc;
        SPG_LAUNCH(K_CP_COLOUR, s, cp_colour_kernel, cp_grid(n), CP_T, 0, n, reverse, w);
    }
    return launch_status();
}

int spg_cp_activate(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                    int spatial, int64_t* out, spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    cudaError_t e = cudaMemsetAsync(w.nsink, 0, (size_t)n_comp * sizeof(int32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.words + W_SAT, 0, sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_ACTIVATE, s, cp_sink_count_kernel, cp_grid(n), CP_T, 0, n, w);
    SPG_LAUNCH(K_CP_ACTIVATE, s, cp_activate_kernel, cp_grid(n_comp + n_edges), CP_T, 0, n, n_edges, n_comp,
               spatial, w);
    SPG_LAUNCH(K_CP_ACTIVATE, s, cp_sat_count_kernel, cp_grid(n_comp), CP_T, 0, n_comp, w);
    return cp_read(out, w.words + W_SAT, 1, s);
}

int spg_cp_split(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                 int64_t* out, spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    SPG_LAUNCH(K_CP_SPLIT, s, cp_cc_init_kernel, cp_grid(n), CP_T, 0, n, w);
    for (;;) {
        cudaError_t e = cudaMemsetAsync(w.words + W_FLAG, 0, sizeof(int64_t), s);
        if (e != cudaSuccess) return (int)e;
        SPG_LAUNCH(K_CP_SPLIT, s, cp_hook_kernel, cp_grid(n_edges), CP_T, 0, n_edges, w);
        SPG_LAUNCH(K_CP_SPLIT, s, cp_jump_kernel, cp_grid(n), CP_T, 0, n, w);
        int64_t f;
        const int rc = cp_read(&f, w.words + W_FLAG, 1, s);
        if (rc != SPG_OK) return rc;
        if (!f) break;
    }
    SPG_LAUNCH(K_CP_SPLIT, s, cp_old_roots_kernel, cp_grid(n_comp), CP_T, 0, n_comp, w);
    SPG_LAUNCH(K_CP_SPLIT, s, cp_new_flags_kernel, cp_grid(n + 1), CP_T, 0, n, w);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.rank, w.newid, (int)n + 1, s);
    int64_t n_new;
    int rc;
    cudaError_t e = cudaMemsetAsync(w.words + W_COUNT, 0, sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_SPLIT, s, cp_count_new_kernel, 1, 1, 0, n, w);
    rc = cp_read(&n_new, w.words + W_COUNT, 1, s);
    if (rc != SPG_OK) return rc;
    SPG_LAUNCH(K_CP_SPLIT, s, cp_new_ids_kernel, cp_grid(n), CP_T, 0, n, n_comp, w);
    SPG_LAUNCH(K_CP_SPLIT, s, cp_assign_kernel, cp_grid(n), CP_T, 0, n, n_comp, w);
    out[0] = n_comp + n_new;
    return launch_status();
}

int spg_cp_merge(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                 double reg_strength, double cutoff, int is_cutoff, int64_t* out, spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    const int64_t E = n_edges;
    out[0] = 0;
    out[1] = n_comp;
    int rc = cp_members(w, n, n_comp, s);
    if (rc != SPG_OK) return rc;
    CP_PER_COMP(K_CP_MERGE, s, n_comp, cp_values_kernel, dim, w);
    if (E == 0 || n_comp == 1) return launch_status();
    cudaError_t e = cudaMemsetAsync(w.words + W_NRUNS, 0, 2 * sizeof(int64_t), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_MERGE, s, cp_border_keys_kernel, cp_grid(E), CP_T, 0, E, w);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.bkey, w.bkey2, (const double*)w.bw, w.bw2,
            (int)E, 0, 64, s);
    SPG_CUB(w.cub, cub::DeviceReduce::ReduceByKey, (const uint64_t*)w.bkey2, w.bkey, (const double*)w.bw2, w.bw,
            w.words + W_NRUNS, cub::Sum(), (int)E, s);
    int64_t n_runs;
    rc = cp_read(&n_runs, w.words + W_NRUNS, 1, s);
    if (rc != SPG_OK) return rc;
    SPG_LAUNCH(K_CP_MERGE, s, cp_gain_kernel, cp_grid(n_runs), CP_T, 0, n_runs, dim, reg_strength, cutoff,
               is_cutoff, w);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.gkey, w.gkey2, (const int32_t*)w.gidx,
            w.gidx2, (int)n_runs, 0, 64, s);
    int64_t n_cand;
    rc = cp_read(&n_cand, w.words + W_NCAND, 1, s);
    if (rc != SPG_OK || n_cand == 0) return rc;
    SPG_LAUNCH(K_CP_MERGE, s, cp_match_init_kernel, cp_grid(n_comp), CP_T, 0, n_comp, w);
    int64_t n_merged = 0;
    for (;;) {
        e = cudaMemsetAsync(w.words + W_COUNT, 0, sizeof(int64_t), s);
        if (e != cudaSuccess) return (int)e;
        SPG_LAUNCH(K_CP_MERGE, s, cp_match_best_kernel, cp_grid(n_cand), CP_T, 0, n_cand, w);
        SPG_LAUNCH(K_CP_MERGE, s, cp_match_take_kernel, cp_grid(n_cand), CP_T, 0, n_cand, w);
        SPG_LAUNCH(K_CP_MERGE, s, cp_best_reset_kernel, cp_grid(n_comp), CP_T, 0, n_comp, w);
        int64_t took;
        rc = cp_read(&took, w.words + W_COUNT, 1, s);
        if (rc != SPG_OK) return rc;
        if (took == 0) break;
        n_merged += took;
    }
    SPG_LAUNCH(K_CP_MERGE, s, cp_merge_apply_kernel, cp_grid(n_comp + 1), CP_T, 0, n_comp, dim, w);
    SPG_LAUNCH(K_CP_MERGE, s, cp_deactivate_kernel, cp_grid(E), CP_T, 0, E, w);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.newid, w.pid, (int)n_comp + 1, s);
    SPG_LAUNCH(K_CP_MERGE, s, cp_renumber_kernel, cp_grid(n_comp), CP_T, 0, n_comp, dim, w);
    const int64_t m = n_comp - n_merged;
    e = cudaMemcpyAsync(w.root, w.root2, m * sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(w.sat, w.sat2, m, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(w.value, w.value2, m * dim * sizeof(double), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_CP_MERGE, s, cp_recomp_kernel, cp_grid(n), CP_T, 0, n, w);
    out[0] = n_merged;
    out[1] = m;
    return launch_status();
}

int spg_cp_energy(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes,
                  double reg_strength, double* out, spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    const unsigned nb = std::min<unsigned>(cp_grid(n + n_edges), CP_PARTIALS);
    SPG_LAUNCH(K_CP_ENERGY, s, cp_energy_kernel, nb, CP_T, 0, n, n_edges, dim, w);
    SPG_LAUNCH(K_CP_ENERGY, s, cp_energy_final_kernel, 1, CP_T, 0, (int)nb, reg_strength, w);
    return cp_read(out, w.dwords, 3, s);
}

int spg_cp_output(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                  int64_t* in_component, int64_t* offsets, int64_t* members, spg_stream_t stream) {
    if (!in_component || !offsets || !members) return SPG_E_BADARG;
    CP_WS(n, n_edges, dim, workspace, workspace_bytes);
    if (n_comp < 1 || n_comp > n) return SPG_E_BADARG;
    const int rc = cp_members(w, n, n_comp, s);
    if (rc != SPG_OK) return rc;
    SPG_LAUNCH(K_CP_MEMBERS, s, cp_output_kernel, cp_grid(n + 1), CP_T, 0, n, n_comp, w, in_component, offsets,
               members);
    return launch_status();
}

}  // extern "C"
