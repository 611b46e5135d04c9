// Exact 3D Delaunay triangulation of a float32 cloud on the device: parallel Bowyer-Watson cavity insertion with a
// symbolic infinite vertex (spg_delaunay.py runs the rounds).  The predicates and the perturbation are in
// dt_predicates.cuh.
//
//   dt_setup     finiteness, the lexicographic (x, y, z) sort, the duplicates (the smallest index of a group is
//                kept), every unique point's rank, and the insertion order: a Morton key over the bounding box
//   dt_init      the first tetrahedron (the first affinely independent points in insertion order), its four
//                infinite neighbours, and every point located by a visibility walk
//   dt_nominate  every tetrahedron holding uninserted points nominates the one of smallest priority (a bijective
//                hash of its id, so that the nominees of neighbouring tetrahedra are scattered inside them)
//   dt_grow      every nominee grows its cavity over the perturbed in-sphere test and claims its cavity and the
//                tetrahedra across the cavity's boundary with an integer atomicMin of its priority (a bijective
//                hash of its id)
//   dt_check     a nominee that holds all its claims wins and reserves one slot per boundary face
//   dt_commit    winners retriangulate their cavities from the boundary faces, patch the adjacency inside and
//                outside, forward their dead tetrahedra to a new one and push them on the free list
//   dt_relocate  points of dead tetrahedra walk from the forwarded one to a tetrahedron they conflict with
//   dt_output    the finite tetrahedra in original ids, rotated to canonical form and sorted
//
// Claims cover the cavity and its outer ring, so two winners never touch the same tetrahedron and the nominee of
// smallest priority always wins: every round inserts at least one point.  A cavity larger than the per-nominee buffer is
// grown again, alone, over a buffer of the whole store; a round whose winners need more slots than the store has
// writes nothing and reports it, and the host grows the store.
#include <cub/cub.cuh>

#include "common.cuh"
#include "dt_predicates.cuh"
#include "workspace.cuh"

namespace spg {
namespace {

using dt::P3;

constexpr int DT_T = 256;
constexpr int DT_SLOT = 320;       // ints of buffer per nominee, at least: 64 cavity tetrahedra, 128 boundary faces
constexpr int DT_NOM = 1 << 18;    // nominees per round at most
constexpr int INF_V = -1;
constexpr unsigned CAV_MARK = 0x80000000u;
constexpr int DT_WALK = 1 << 20;   // steps of one walk before it is reported as stuck
constexpr int DT_MAX_CAP = 1 << 29;  // adjacency entries hold tet * 4 + face in int32

// state words
enum {
    S_STATUS = 0,   // 1: non-finite coordinate, 2: fewer than 4 affinely independent points, 4: a walk did not end,
                    // 8: a cavity that is not a ball
    S_UNIQUE,
    S_TOP,
    S_NFREE,
    S_NOM,
    S_WIN,
    S_NEW,
    S_OVER,
    S_MIN_OVER,
    S_MAX_CAV,
    S_I2,
    S_I3,
    S_PUSHED,
    S_BIG,
    S_LO,           // 3 words: coordinate minima as float keys
    S_HI = S_LO + 3,
    S_COUNT = S_HI + 3,
    S_WORDS = 32
};

struct DtWs {
    int* state;
    uint64_t *k64a, *k64b;
    uint32_t *k32a, *k32b;
    int *ia, *ib;
    int* uniq;
    float4* wp;  // insertion order: x, y, z, lexicographic rank (int bits)
    int* orig;
    int* pt_tet;  // -1 once inserted
    int *nom_p, *nom_nc, *nom_nb, *nom_base;
    int* buf;
    int64_t buf_ints;
    int4 *tv, *ta;
    unsigned* owner;
    unsigned* nomt;  // per tetrahedron: the smallest priority of the points it holds
    int* freel;
    CubRegion cub;
    size_t bytes;
};

int64_t nom_cap(int64_t n) { return n < DT_NOM ? (n > 0 ? n : 1) : DT_NOM; }

int layout(int64_t n, int64_t cap, void* base, DtWs* w) {
    Planner p(base);
    const int64_t nc = nom_cap(n);
    w->state = p.take<int>(S_WORDS);
    w->k64a = p.take<uint64_t>(n);
    w->k64b = p.take<uint64_t>(n);
    w->k32a = p.take<uint32_t>(n);
    w->k32b = p.take<uint32_t>(n);
    w->ia = p.take<int>(n);
    w->ib = p.take<int>(n);
    w->uniq = p.take<int>(n);
    w->wp = p.take<float4>(n);
    w->orig = p.take<int>(n);
    w->pt_tet = p.take<int>(n);
    w->nom_p = p.take<int>(nc);
    w->nom_nc = p.take<int>(nc);
    w->nom_nb = p.take<int>(nc);
    w->nom_base = p.take<int>(nc);
    const int64_t per = nc * DT_SLOT, whole = 6 * cap;
    w->buf_ints = per > whole ? per : whole;
    w->buf = p.take<int>(w->buf_ints);
    w->tv = p.take<int4>(cap);
    w->ta = p.take<int4>(cap);
    w->owner = p.take<unsigned>(cap);
    w->nomt = p.take<unsigned>(cap);
    w->freel = p.take<int>(cap);
    size_t cb = 0;
    const int ni = (int)n, ci = (int)cap;
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int*)nullptr, (int*)nullptr, ni);
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                  (const int*)nullptr, (int*)nullptr, ni);
    SPG_CUB_BYTES(cb, cub::DeviceSelect::Flagged, (const int*)nullptr, (const int*)nullptr, (int*)nullptr,
                  (int*)nullptr, ni);
    SPG_CUB_BYTES(cb, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int*)nullptr, (int*)nullptr, ci);
    w->cub = p.cub(cb);
    w->bytes = p.bytes;
    return SPG_OK;
}

unsigned grid_of(int64_t n) { return (unsigned)ceil_div64(n > 0 ? n : 1, DT_T); }

__device__ __forceinline__ P3 pt(const float4* wp, int i) {
    const float4 v = wp[i];
    return P3{v.x, v.y, v.z};
}
__device__ __forceinline__ int rank_of(const float4* wp, int i) { return __float_as_int(wp[i].w); }
__device__ __forceinline__ int vget(const int4& v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w)); }
__device__ __forceinline__ void vset(int4& v, int i, int x) {
    if (i == 0) v.x = x;
    else if (i == 1) v.y = x;
    else if (i == 2) v.z = x;
    else v.w = x;
}
__device__ __forceinline__ int vfind(const int4& v, int x) {
    return v.x == x ? 0 : (v.y == x ? 1 : (v.z == x ? 2 : 3));
}
__device__ __forceinline__ bool dead(const int4& v) { return v.x < -1; }

// claim priority of point s: a bijection of [0, 2^31) that scatters the Morton order, so that nearby nominees'
// priorities are uncorrelated and many of them are local minima (below CAV_MARK, so never a cavity mark)
__device__ __forceinline__ unsigned prio(int s) { return ((unsigned)s * 2654435761u) & 0x7fffffffu; }

// nominee k's cavity list, boundary list and cavity hash set (open addressing, -1 empty, at most half full): the
// buffer split evenly over the round's nn nominees, since early rounds have few nominees and large cavities; a big
// round's one nominee takes all of it and marks its cavity in owner[] instead of hashing
struct Slice {
    int *cav, *bnd, *hash;
    int ccap, bcap, hmask;
};
__device__ __forceinline__ Slice slice_of(const DtWs& w, int k, int nn, int big, int64_t cap) {
    if (big) return Slice{w.buf, w.buf + cap, nullptr, (int)cap, (int)(5 * cap), 0};
    int64_t stride = w.buf_ints / (nn > 0 ? nn : 1);
    if (stride > (1 << 15)) stride = 1 << 15;
    int h = 1;
    while (2 * h <= stride * 2 / 5) h *= 2;
    int* base = w.buf + k * stride;
    return Slice{base + h, base + h + h / 2, base, h / 2, (int)(stride - h - h / 2), h - 1};
}

__device__ __forceinline__ unsigned tet_hash(int t) { return (unsigned)t * 2654435761u; }

// inserts t into the set; false if it was there already
__device__ __forceinline__ bool hash_insert(const Slice& sl, int t) {
    for (unsigned i = tet_hash(t) & sl.hmask;; i = (i + 1) & sl.hmask) {
        const int v = sl.hash[i];
        if (v == t) return false;
        if (v < 0) {
            sl.hash[i] = t;
            return true;
        }
    }
}

__device__ __forceinline__ bool hash_has(const Slice& sl, int t) {
    for (unsigned i = tet_hash(t) & sl.hmask;; i = (i + 1) & sl.hmask) {
        const int v = sl.hash[i];
        if (v == t) return true;
        if (v < 0) return false;
    }
}

__device__ __forceinline__ int orient_q(const float4* wp, int4 v, int i, const P3& q) {
    P3 p[4];
    for (int k = 0; k < 4; ++k) p[k] = k == i ? q : pt(wp, vget(v, k));
    return dt::orient3d(p[0], p[1], p[2], p[3]);
}

// whether point s (coordinates q) is in conflict with tetrahedron v
__device__ bool conflict(const float4* wp, int4 v, int s, const P3& q) {
    const int rq = rank_of(wp, s);
    const int k = vfind(v, INF_V);
    if (vget(v, k) == INF_V) {
        const int o = orient_q(wp, v, k, q);
        if (o) return o > 0;
        P3 f[3];
        int r[3], c = 0;
        for (int i = 0; i < 4; ++i)
            if (i != k) {
                f[c] = pt(wp, vget(v, i));
                r[c++] = rank_of(wp, vget(v, i));
            }
        return dt::incircle_perturbed(f, r, q, rq) > 0;
    }
    P3 p[4];
    int r[4];
    for (int i = 0; i < 4; ++i) {
        p[i] = pt(wp, vget(v, i));
        r[i] = rank_of(wp, vget(v, i));
    }
    return dt::insphere_perturbed(p, r, q, rq) > 0;
}

// visibility walk from t to a tetrahedron in conflict with s; -1 if it does not end
__device__ int walk(const DtWs& w, int t, int s) {
    const P3 q = pt(w.wp, s);
    for (int step = 0; step < DT_WALK; ++step) {
        const int4 v = w.tv[t];
        const int k = vfind(v, INF_V);
        if (vget(v, k) == INF_V) {
            if (conflict(w.wp, v, s, q)) return t;
            t = vget(w.ta[t], k) >> 2;
            continue;
        }
        bool moved = false;
        for (int j = 0; j < 4; ++j) {
            const int i = (j + s + step) & 3;
            if (orient_q(w.wp, v, i, q) < 0) {
                t = vget(w.ta[t], i) >> 2;
                moved = true;
                break;
            }
        }
        if (!moved) return t;
    }
    return -1;
}

// ------------------------------------------------------------------------------------------------ dt_setup
__global__ void dt_keys_kernel(const float* __restrict__ xyz, int n, DtWs w) {
    SPG_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = xyz[3 * i] + 0.f, y = xyz[3 * i + 1] + 0.f, z = xyz[3 * i + 2] + 0.f;  // -0 -> +0
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) atomicOr(&w.state[S_STATUS], 1);
    w.k64a[i] = ((uint64_t)float_key(y) << 32) | float_key(z);
    w.ia[i] = i;
}

__global__ void dt_xkeys_kernel(const float* __restrict__ xyz, int n, DtWs w) {
    SPG_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    w.k32a[i] = float_key(xyz[3 * w.ib[i]] + 0.f);
}

// after the x sort (ia: ids in lexicographic order): first of every run of equal points
__global__ void dt_flags_kernel(const float* __restrict__ xyz, int n, DtWs w) {
    SPG_PDL_ENTRY();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int a = w.ia[j];
    int f = 1;
    if (j > 0) {
        const int b = w.ia[j - 1];
        f = !(xyz[3 * a] == xyz[3 * b] && xyz[3 * a + 1] == xyz[3 * b + 1] && xyz[3 * a + 2] == xyz[3 * b + 2]);
    }
    w.ib[j] = f;
}

__global__ void dt_bounds_kernel(const float* __restrict__ xyz, DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= u) return;
    const int i = w.uniq[j];
    for (int c = 0; c < 3; ++c) {
        const unsigned k = float_key(xyz[3 * i + c] + 0.f);
        atomicMin((unsigned*)&w.state[S_LO + c], k);
        atomicMax((unsigned*)&w.state[S_HI + c], k);
    }
}

__device__ __forceinline__ uint64_t spread3(uint64_t v) {  // 16 bits -> every third of 48
    v &= 0xffff;
    v = (v | (v << 16)) & 0x0000ff0000ffull;
    v = (v | (v << 8)) & 0x00f00f00f00full;
    v = (v | (v << 4)) & 0x0c30c30c30c3ull;
    v = (v | (v << 2)) & 0x249249249249ull;
    return v;
}

__global__ void dt_morton_kernel(const float* __restrict__ xyz, DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= u) return;
    const int i = w.uniq[j];
    uint64_t key = 0;
    for (int c = 0; c < 3; ++c) {
        const double lo = float_unkey((unsigned)w.state[S_LO + c]), hi = float_unkey((unsigned)w.state[S_HI + c]);
        const double ext = hi - lo;
        double f = ext > 0 ? ((double)xyz[3 * i + c] - lo) / ext : 0.0;
        const uint64_t q = (uint64_t)fmin(fmax(f * 65535.0, 0.0), 65535.0);
        key |= spread3(q) << c;
    }
    w.k64a[j] = key;
    w.ia[j] = j;
}

__global__ void dt_fill_kernel(const float* __restrict__ xyz, DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u) return;
    const int j = w.ib[s];  // lexicographic rank
    const int i = w.uniq[j];
    w.wp[s] = make_float4(xyz[3 * i] + 0.f, xyz[3 * i + 1] + 0.f, xyz[3 * i + 2] + 0.f, __int_as_float(j));
    w.orig[s] = i;
}

// ------------------------------------------------------------------------------------------------ dt_init
__global__ void dt_find2_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = 2 + blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u) return;
    if (dt::coplanar_orient(pt(w.wp, 0), pt(w.wp, 1), pt(w.wp, s)) != 0) atomicMin(&w.state[S_I2], s);
}

__global__ void dt_find3_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE], i2 = w.state[S_I2];
    const int s = 2 + blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u || i2 >= u) return;
    if (dt::orient3d(pt(w.wp, 0), pt(w.wp, 1), pt(w.wp, i2), pt(w.wp, s)) != 0) atomicMin(&w.state[S_I3], s);
}

__global__ void dt_first_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE], i2 = w.state[S_I2], i3 = w.state[S_I3];
    if (i2 >= u || i3 >= u) {
        w.state[S_STATUS] |= 2;
        return;
    }
    int f[4] = {0, 1, i2, i3};
    if (dt::orient3d(pt(w.wp, f[0]), pt(w.wp, f[1]), pt(w.wp, f[2]), pt(w.wp, f[3])) < 0) {
        f[0] = 1;
        f[1] = 0;
    }
    int4 v0 = make_int4(f[0], f[1], f[2], f[3]);
    w.tv[0] = v0;
    int4 vi[4];
    for (int i = 0; i < 4; ++i) {
        int4 v = v0;
        vset(v, i, INF_V);
        int o[3], c = 0;
        for (int j = 0; j < 4; ++j)
            if (j != i) o[c++] = j;
        const int a = vget(v, o[0]);
        vset(v, o[0], vget(v, o[1]));
        vset(v, o[1], a);
        vi[i] = v;
        w.tv[i + 1] = v;
    }
    int4 a0;
    for (int i = 0; i < 4; ++i) vset(a0, i, ((i + 1) << 2) | i);
    w.ta[0] = a0;
    for (int i = 0; i < 4; ++i) {
        int4 a;
        vset(a, i, (0 << 2) | i);
        for (int j = 0; j < 4; ++j)
            if (j != i) vset(a, vfind(vi[i], f[j]), ((j + 1) << 2) | vfind(vi[j], f[i]));
        w.ta[i + 1] = a;
    }
    w.state[S_TOP] = 5;
    w.state[S_NFREE] = 0;
}

__global__ void dt_locate_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u || (w.state[S_STATUS] & 2)) return;
    const int4 v0 = w.tv[0];
    if (s == v0.x || s == v0.y || s == v0.z || s == v0.w) {
        w.pt_tet[s] = -1;
        return;
    }
    const int t = walk(w, 0, s);
    if (t < 0) atomicOr(&w.state[S_STATUS], 4);
    w.pt_tet[s] = t;
}

// ------------------------------------------------------------------------------------------------ rounds
__global__ void dt_nominate_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u) return;
    const int t = w.pt_tet[s];
    if (t >= 0) atomicMin(&w.nomt[t], prio(s));
}

__global__ void dt_list_kernel(DtWs w, int nc) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u) return;
    const int t = w.pt_tet[s];
    if (t >= 0 && w.nomt[t] == prio(s)) {
        const int k = atomicAdd(&w.state[S_NOM], 1);
        if (k < nc) w.nom_p[k] = s;
    }
}

__global__ void dt_list_big_kernel(DtWs w, int s) {
    SPG_PDL_ENTRY();
    w.nom_p[0] = s;
    w.state[S_NOM] = 1;
    w.state[S_BIG] = 1;
}

// grows nominee k's cavity into its buffer; big: the one nominee of the round, membership marked in owner[]
__global__ void dt_grow_kernel(DtWs w, int nc, int big, int64_t cap) {
    SPG_PDL_ENTRY();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int nn = min(w.state[S_NOM], nc);
    if (k >= nn) return;
    const int s = w.nom_p[k];
    const P3 q = pt(w.wp, s);
    const Slice sl = slice_of(w, k, nn, big, cap);
    int* cav = sl.cav;
    int* bnd = sl.bnd;
    const int ccap = sl.ccap, bcap = sl.bcap;
    const unsigned mark = (unsigned)s | CAV_MARK;
    int c = 1, b = 0;
    cav[0] = w.pt_tet[s];
    if (big) {
        w.owner[cav[0]] = mark;
    } else {
        for (int i = 0; i <= sl.hmask; ++i) sl.hash[i] = -1;
        hash_insert(sl, cav[0]);
    }
    bool over = false;
    for (int i = 0; i < c && !over; ++i) {
        const int t = cav[i];
        const int4 a = w.ta[t];
        for (int f = 0; f < 4; ++f) {
            const int nb = vget(a, f) >> 2;
            if (big ? w.owner[nb] == mark : hash_has(sl, nb)) continue;
            if (conflict(w.wp, w.tv[nb], s, q)) {
                if (c == ccap) {
                    over = true;
                    break;
                }
                cav[c++] = nb;
                if (big) w.owner[nb] = mark;
                else hash_insert(sl, nb);
            } else {
                if (b == bcap) {
                    over = true;
                    break;
                }
                bnd[b++] = t * 4 + f;
            }
        }
    }
    if (over) {
        w.nom_nc[k] = -1;
        atomicAdd(&w.state[S_OVER], 1);
        atomicMin(&w.state[S_MIN_OVER], s);
        return;
    }
    w.nom_nc[k] = c;
    w.nom_nb[k] = b;
    atomicMax(&w.state[S_MAX_CAV], c);
    if (big) return;
    const unsigned pr = prio(s);
    for (int i = 0; i < c; ++i) atomicMin(&w.owner[cav[i]], pr);
    for (int i = 0; i < b; ++i) atomicMin(&w.owner[vget(w.ta[bnd[i] >> 2], bnd[i] & 3) >> 2], pr);
}

__global__ void dt_check_kernel(DtWs w, int nc, int big, int64_t cap) {
    SPG_PDL_ENTRY();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int nn = min(w.state[S_NOM], nc);
    if (k >= nn) return;
    const int c = w.nom_nc[k];
    if (c < 0) return;
    const int s = w.nom_p[k];
    const int b = w.nom_nb[k];
    if (!big) {
        const Slice sl = slice_of(w, k, nn, big, cap);
        const int* cav = sl.cav;
        const int* bnd = sl.bnd;
        const unsigned pr = prio(s);
        for (int i = 0; i < c; ++i)
            if (w.owner[cav[i]] != pr) {
                w.nom_nc[k] = -2;
                return;
            }
        for (int i = 0; i < b; ++i)
            if (w.owner[vget(w.ta[bnd[i] >> 2], bnd[i] & 3) >> 2] != pr) {
                w.nom_nc[k] = -2;
                return;
            }
    }
    w.nom_base[k] = atomicAdd(&w.state[S_NEW], b);
    atomicAdd(&w.state[S_WIN], 1);
}

// slot of the v-th new tetrahedron of the round: the free list from its top, then the bump region
__device__ __forceinline__ int slot_of(const DtWs& w, int v, int nfree, int top) {
    return v < nfree ? w.freel[nfree - 1 - v] : top + (v - nfree);
}

__global__ void dt_commit_kernel(DtWs w, int nc, int big, int64_t cap) {
    SPG_PDL_ENTRY();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int nn = min(w.state[S_NOM], nc);
    if (k >= nn) return;
    const int c = w.nom_nc[k];
    if (c < 0) return;
    const int s = w.nom_p[k], b = w.nom_nb[k], base = w.nom_base[k];
    const int nfree = w.state[S_NFREE], top = w.state[S_TOP];
    const Slice sl = slice_of(w, k, nn, big, cap);
    const int* cav = sl.cav;
    const int* bnd = sl.bnd;
    const unsigned mark = (unsigned)s | CAV_MARK;
    if (!big)
        for (int i = 0; i < c; ++i) w.owner[cav[i]] = mark;
    // the new tetrahedra: boundary face (t, j) with s in place of vertex j; the outside neighbour is patched, and
    // the dead face forwards to the new tetrahedron for the rotations below
    for (int f = 0; f < b; ++f) {
        const int t = bnd[f] >> 2, j = bnd[f] & 3;
        const int nid = slot_of(w, base + f, nfree, top);
        int4 v = w.tv[t];
        vset(v, j, s);
        w.tv[nid] = v;
        int4 ta = w.ta[t];
        const int out = vget(ta, j);
        int4 a = make_int4(-1, -1, -1, -1);
        vset(a, j, out);
        w.ta[nid] = a;
        int4 oa = w.ta[out >> 2];
        vset(oa, out & 3, (nid << 2) | j);
        w.ta[out >> 2] = oa;
        vset(ta, j, (nid << 2) | j);
        w.ta[t] = ta;
    }
    // the faces through s: rotate around the edge inside the cavity to the next boundary face
    for (int f = 0; f < b; ++f) {
        const int t = bnd[f] >> 2, j = bnd[f] & 3;
        const int nid = slot_of(w, base + f, nfree, top);
        const int4 vt = w.tv[t];
        int4 a = w.ta[nid];
        for (int kk = 0; kk < 4; ++kk) {
            if (kk == j) continue;
            int e0 = -2, e1 = -2;
            for (int i = 0; i < 4; ++i)
                if (i != j && i != kk) (e0 == -2 ? e0 : e1) = vget(vt, i);
            int cur = t, face = kk;
            for (int step = 0;; ++step) {
                if (step > c) {  // the cavity is not a ball: reported, never looped on
                    atomicOr(&w.state[S_STATUS], 8);
                    break;
                }
                const int4 vc = w.tv[cur];
                int x = -2;  // the vertex of face `face` of cur off the edge
                for (int i = 0; i < 4; ++i) {
                    const int vv = vget(vc, i);
                    if (i != face && vv != e0 && vv != e1) x = vv;
                }
                const int e = vget(w.ta[cur], face);
                const int nt = e >> 2;
                if (w.owner[nt] == mark) {
                    cur = nt;
                    face = vfind(w.tv[nt], x);
                } else {
                    // nt was built on boundary face (cur, face); its face through s and the edge is opposite x
                    vset(a, kk, (nt << 2) | vfind(vc, x));
                    break;
                }
            }
        }
        w.ta[nid] = a;
    }
    const int fwd = slot_of(w, base, nfree, top);
    for (int i = 0; i < c; ++i) {
        int4 v = w.tv[cav[i]];
        v.x = -2 - fwd;
        w.tv[cav[i]] = v;
    }
    w.pt_tet[s] = -1;
}

__global__ void dt_push_kernel(DtWs w, int nc, int big, int64_t cap) {
    SPG_PDL_ENTRY();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int nn = min(w.state[S_NOM], nc);
    if (k >= nn) return;
    const int c = w.nom_nc[k];
    if (c < 0) return;
    const int* cav = slice_of(w, k, nn, big, cap).cav;
    const int used = min(w.state[S_NEW], w.state[S_NFREE]);
    const int pos = w.state[S_NFREE] - used + atomicAdd(&w.state[S_PUSHED], c);
    for (int i = 0; i < c; ++i) w.freel[pos + i] = cav[i];
}

__global__ void dt_relocate_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int u = w.state[S_UNIQUE];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= u) return;
    const int t = w.pt_tet[s];
    if (t < 0) return;
    const int4 v = w.tv[t];
    if (!dead(v)) return;
    const int r = walk(w, -2 - v.x, s);
    if (r < 0) atomicOr(&w.state[S_STATUS], 4);
    w.pt_tet[s] = r < 0 ? -1 : r;
}

__global__ void dt_round_end_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int nw = w.state[S_NEW], nf = w.state[S_NFREE];
    const int used = min(nw, nf);
    w.state[S_TOP] += nw - used;
    w.state[S_NFREE] = nf - used + w.state[S_PUSHED];
}

// ------------------------------------------------------------------------------------------------ dt_output
__global__ void dt_count_kernel(DtWs w) {
    SPG_PDL_ENTRY();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= w.state[S_TOP]) return;
    const int4 v = w.tv[t];
    if (dead(v) || v.x == INF_V || v.y == INF_V || v.z == INF_V || v.w == INF_V) return;
    atomicAdd(&w.state[S_COUNT], 1);
}

// rows in original ids, rotated by an even permutation to (smallest, second smallest, ...); keys for the sort
__global__ void dt_emit_kernel(DtWs w, int4* rows, uint64_t* lo, int* idx) {
    SPG_PDL_ENTRY();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= w.state[S_TOP]) return;
    const int4 v = w.tv[t];
    if (dead(v) || v.x == INF_V || v.y == INF_V || v.z == INF_V || v.w == INF_V) return;
    int r[4] = {w.orig[v.x], w.orig[v.y], w.orig[v.z], w.orig[v.w]};
    int m = 0;
    for (int i = 1; i < 4; ++i)
        if (r[i] < r[m]) m = i;
    static const int front[4][4] = {{0, 1, 2, 3}, {1, 0, 3, 2}, {2, 3, 0, 1}, {3, 2, 1, 0}};
    int a[4];
    for (int i = 0; i < 4; ++i) a[i] = r[front[m][i]];
    int m2 = 1;
    for (int i = 2; i < 4; ++i)
        if (a[i] < a[m2]) m2 = i;
    int o[4];
    o[0] = a[0];
    for (int i = 0; i < 3; ++i) o[1 + i] = a[1 + (m2 - 1 + i) % 3];
    const int j = atomicAdd(&w.state[S_COUNT], 1);
    rows[j] = make_int4(o[0], o[1], o[2], o[3]);
    lo[j] = ((uint64_t)(uint32_t)o[2] << 32) | (uint32_t)o[3];
    idx[j] = j;
}

__global__ void dt_hikeys_kernel(const int4* rows, const int* idx, uint64_t* hi, int m) {
    SPG_PDL_ENTRY();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int4 r = rows[idx[j]];
    hi[j] = ((uint64_t)(uint32_t)r.x << 32) | (uint32_t)r.y;
}

__global__ void dt_gather_kernel(const int4* rows, const int* idx, int4* out, int m) {
    SPG_PDL_ENTRY();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    out[j] = rows[idx[j]];
}

int dt_read(int* dst, const int* src, int count, cudaStream_t s) {
    cudaError_t e = cudaMemcpyAsync(dst, src, sizeof(int) * count, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return (int)e;
}

int dt_bits(int64_t v) {
    int b = 1;
    while (b < 32 && (1ll << b) <= v) ++b;
    return b;
}

bool bad_dims(int64_t n, int64_t cap) { return n < 1 || too_big(n) || cap < 8 || cap > DT_MAX_CAP; }

}  // namespace
}  // namespace spg

using namespace spg;

#define DT_WS(n, cap, ws, ws_bytes)                                  \
    if (bad_dims(n, cap)) return SPG_E_BADARG;                    \
    DtWs w;                                                       \
    {                                                             \
        int rc_ = layout(n, cap, nullptr, &w);                    \
        if (rc_ != SPG_OK) return rc_;                            \
        rc_ = ws_check(ws, ws_bytes, w.bytes);                       \
        if (rc_ != SPG_OK) return rc_;                            \
        layout(n, cap, ws, &w);                                   \
    }                                                             \
    cudaStream_t s = (cudaStream_t)stream;

extern "C" {

int spg_dt_workspace(int64_t n, int64_t cap, int64_t* bytes) {
    if (!bytes || bad_dims(n, cap)) return SPG_E_BADARG;
    DtWs w;
    const int rc = layout(n, cap, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_dt_setup(const float* xyz, int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                 spg_stream_t stream) {
    if (!xyz || !out) return SPG_E_BADARG;
    DT_WS(n, cap, workspace, workspace_bytes);
    const int ni = (int)n;
    cudaError_t e = cudaMemsetAsync(w.state, 0, S_WORDS * sizeof(int), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.state + S_LO, 0xff, 3 * sizeof(int), s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_DT_SETUP, s, dt_keys_kernel, grid_of(n), DT_T, 0, xyz, ni, w);
    int st[2];
    int rc = dt_read(st, w.state, 1, s);
    if (rc != SPG_OK) return rc;
    out[0] = st[0];
    out[1] = 0;
    if (st[0]) return SPG_OK;
    // lexicographic (x, y, z) order, stable in the index: (y, z) first, then x
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.k64a, w.k64b, (const int*)w.ia, w.ib, ni, 0,
            64, s);
    SPG_LAUNCH(K_DT_SETUP, s, dt_xkeys_kernel, grid_of(n), DT_T, 0, xyz, ni, w);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint32_t*)w.k32a, w.k32b, (const int*)w.ib, w.ia, ni, 0,
            32, s);
    SPG_LAUNCH(K_DT_SETUP, s, dt_flags_kernel, grid_of(n), DT_T, 0, xyz, ni, w);
    SPG_CUB(w.cub, cub::DeviceSelect::Flagged, (const int*)w.ia, (const int*)w.ib, w.uniq, w.state + S_UNIQUE, ni,
            s);
    SPG_LAUNCH(K_DT_SETUP, s, dt_bounds_kernel, grid_of(n), DT_T, 0, xyz, w);
    SPG_LAUNCH(K_DT_SETUP, s, dt_morton_kernel, grid_of(n), DT_T, 0, xyz, w);
    rc = dt_read(st, w.state, 2, s);
    if (rc != SPG_OK) return rc;
    const int u = st[1];
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.k64a, w.k64b, (const int*)w.ia, w.ib, u, 0,
            48, s);
    SPG_LAUNCH(K_DT_SETUP, s, dt_fill_kernel, grid_of(u), DT_T, 0, xyz, w);
    out[1] = u;
    return launch_status();
}

int spg_dt_init(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    DT_WS(n, cap, workspace, workspace_bytes);
    int st[2];
    int rc = dt_read(st, w.state, 2, s);
    if (rc != SPG_OK) return rc;
    const int u = st[1];
    if (u < 4) {
        out[0] = 2;
        return SPG_OK;
    }
    const int big[2] = {0x7fffffff, 0x7fffffff};
    cudaError_t e = cudaMemcpyAsync(w.state + S_I2, big, 2 * sizeof(int), cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_DT_INIT, s, dt_find2_kernel, grid_of(u), DT_T, 0, w);
    SPG_LAUNCH(K_DT_INIT, s, dt_find3_kernel, grid_of(u), DT_T, 0, w);
    SPG_LAUNCH(K_DT_INIT, s, dt_first_kernel, 1, 1, 0, w);
    SPG_LAUNCH(K_DT_INIT, s, dt_locate_kernel, grid_of(u), DT_T, 0, w);
    rc = dt_read(st, w.state, 1, s);
    if (rc != SPG_OK) return rc;
    out[0] = st[0];
    return launch_status();
}

int spg_dt_cavities(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t big_point,
                    int64_t* out, spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    DT_WS(n, cap, workspace, workspace_bytes);
    const int nc = (int)nom_cap(n);
    const int big = big_point >= 0;
    if (big_point >= n) return SPG_E_BADARG;
    cudaError_t e = cudaMemsetAsync(w.owner, 0xff, (size_t)cap * sizeof(unsigned), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.nomt, 0xff, (size_t)cap * sizeof(unsigned), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.state + S_NOM, 0, (S_MAX_CAV - S_NOM) * sizeof(int), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.state + S_MIN_OVER, 0x7f, sizeof(int), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.state + S_PUSHED, 0, 2 * sizeof(int), s);
    if (e != cudaSuccess) return (int)e;
    int st[2];
    int rc = dt_read(st, w.state, 2, s);
    if (rc != SPG_OK) return rc;
    const int u = st[1];
    if (big) {
        SPG_LAUNCH(K_DT_NOMINATE, s, dt_list_big_kernel, 1, 1, 0, w, (int)big_point);
    } else {
        SPG_LAUNCH(K_DT_NOMINATE, s, dt_nominate_kernel, grid_of(u), DT_T, 0, w);
        SPG_LAUNCH(K_DT_NOMINATE, s, dt_list_kernel, grid_of(u), DT_T, 0, w, nc);
    }
    SPG_LAUNCH(K_DT_GROW, s, dt_grow_kernel, grid_of(big ? 1 : nc), big ? 1 : DT_T, 0, w, nc, big, cap);
    SPG_LAUNCH(K_DT_CHECK, s, dt_check_kernel, grid_of(big ? 1 : nc), big ? 1 : DT_T, 0, w, nc, big, cap);
    int v[S_WORDS];
    rc = dt_read(v, w.state, S_WORDS, s);
    if (rc != SPG_OK) return rc;
    // out: nominees, winners, new tetrahedra, overflowing nominees, smallest overflowing, free slots, top, largest
    // cavity
    out[0] = v[S_NOM] < nc ? v[S_NOM] : nc;
    out[1] = v[S_WIN];
    out[2] = v[S_NEW];
    out[3] = v[S_OVER];
    out[4] = v[S_MIN_OVER];
    out[5] = v[S_NFREE];
    out[6] = v[S_TOP];
    out[7] = v[S_MAX_CAV];
    return launch_status();
}

int spg_dt_commit(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                  spg_stream_t stream) {
    if (!out) return SPG_E_BADARG;
    DT_WS(n, cap, workspace, workspace_bytes);
    int v[S_WORDS];
    int rc = dt_read(v, w.state, S_WORDS, s);
    if (rc != SPG_OK) return rc;
    // nothing is written unless every winner's slots are free
    if ((int64_t)v[S_NEW] > (int64_t)v[S_NFREE] + cap - v[S_TOP]) {
        out[0] = 1;
        return SPG_OK;
    }
    out[0] = 0;
    const int nc = (int)nom_cap(n);
    const int big = v[S_BIG];
    const unsigned g = grid_of(big ? 1 : nc), b = big ? 1 : DT_T;
    SPG_LAUNCH(K_DT_COMMIT, s, dt_commit_kernel, g, b, 0, w, nc, big, cap);
    SPG_LAUNCH(K_DT_COMMIT, s, dt_push_kernel, g, b, 0, w, nc, big, cap);
    SPG_LAUNCH(K_DT_RELOCATE, s, dt_relocate_kernel, grid_of(v[S_UNIQUE]), DT_T, 0, w);
    SPG_LAUNCH(K_DT_COMMIT, s, dt_round_end_kernel, 1, 1, 0, w);
    rc = dt_read(v, w.state, 1, s);
    if (rc != SPG_OK) return rc;
    out[1] = v[S_STATUS];
    return launch_status();
}

int spg_dt_grow(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t new_cap,
                void* new_workspace, int64_t new_workspace_bytes, spg_stream_t stream) {
    DT_WS(n, cap, workspace, workspace_bytes);
    if (new_cap < cap || bad_dims(n, new_cap)) return SPG_E_BADARG;
    DtWs d;
    layout(n, new_cap, nullptr, &d);
    const int rc = ws_check(new_workspace, new_workspace_bytes, d.bytes);
    if (rc != SPG_OK) return rc;
    layout(n, new_cap, new_workspace, &d);
    struct R {
        void* dst;
        const void* src;
        size_t bytes;
    } r[] = {{d.state, w.state, S_WORDS * sizeof(int)},        {d.wp, w.wp, (size_t)n * sizeof(float4)},
             {d.orig, w.orig, (size_t)n * sizeof(int)},        {d.pt_tet, w.pt_tet, (size_t)n * sizeof(int)},
             {d.tv, w.tv, (size_t)cap * sizeof(int4)},          {d.ta, w.ta, (size_t)cap * sizeof(int4)},
             {d.freel, w.freel, (size_t)cap * sizeof(int)}};
    for (const R& x : r) {
        const cudaError_t e = cudaMemcpyAsync(x.dst, x.src, x.bytes, cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return (int)e;
    }
    return SPG_OK;
}

int spg_dt_output(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* count, int* simplices,
                  spg_stream_t stream) {
    if (!count) return SPG_E_BADARG;
    DT_WS(n, cap, workspace, workspace_bytes);
    cudaError_t e = cudaMemsetAsync(w.state + S_COUNT, 0, sizeof(int), s);
    if (e != cudaSuccess) return (int)e;
    int v[S_WORDS];
    int rc = dt_read(v, w.state, S_WORDS, s);
    if (rc != SPG_OK) return rc;
    const int top = v[S_TOP];
    if (!simplices) {
        SPG_LAUNCH(K_DT_OUTPUT, s, dt_count_kernel, grid_of(top), DT_T, 0, w);
        rc = dt_read(v, w.state + S_COUNT, 1, s);
        if (rc != SPG_OK) return rc;
        *count = v[0];
        return launch_status();
    }
    // the adjacency is not needed any more: its region holds the rows
    int4* rows = w.ta;
    uint64_t* lo_a = (uint64_t*)w.buf;
    uint64_t* lo_b = lo_a + cap;
    int* ia = (int*)(lo_b + cap);
    int* ib = ia + cap;
    SPG_LAUNCH(K_DT_OUTPUT, s, dt_emit_kernel, grid_of(top), DT_T, 0, w, rows, lo_a, ia);
    rc = dt_read(v, w.state + S_COUNT, 1, s);
    if (rc != SPG_OK) return rc;
    const int m = v[0];
    if (m != *count) return SPG_E_BADARG;
    const int bits = dt_bits(n);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)lo_a, lo_b, (const int*)ia, ib, m, 0, 32 + bits,
            s);
    SPG_LAUNCH(K_DT_OUTPUT, s, dt_hikeys_kernel, grid_of(m), DT_T, 0, (const int4*)rows, (const int*)ib, lo_a, m);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)lo_a, lo_b, (const int*)ib, ia, m, 0, 32 + bits,
            s);
    SPG_LAUNCH(K_DT_OUTPUT, s, dt_gather_kernel, grid_of(m), DT_T, 0, (const int4*)rows, (const int*)ia,
               (int4*)simplices, m);
    return launch_status();
}

}  // extern "C"
