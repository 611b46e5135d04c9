// A point cloud's k-nearest-neighbour graphs and geometric features (ref: partition/graphs.py:11-70
// `compute_graph_nn`, `compute_graph_nn_2`; partition/ply_c/ply_c.cpp:384-462 `compute_geof`), the first phase of
// both partition pipelines (partition/partition.py:146-152, supervized_partition/graph_processing.py:146,176):
//
//   geo_bounds  the bounding box of the cloud (order-free integer min / max of an order-preserving map of the
//               floats) and a status word: bit 0 is set for a non-finite coordinate
//   geo_grid    one 63-bit cell key (21 bits per axis, x major) per point and the sorted cloud: CUB's stable radix
//               sort of (key, index), so indices stay ascending within a cell, xyz gathered in that order, the
//               table of occupied cells (run-length encode + scan: key, first sorted position)
//   geo_knn     one thread per query, queries in sorted (cell) order so that neighbouring threads read the same
//               cells; its k best candidates live in shared memory as a sorted list of (d2, id) (slot-major, so the
//               threads of a warp hit distinct banks).  Cells are visited ring by ring (Chebyshev distance in
//               cells); a column (cx, cy) of a ring is one contiguous range of sorted points, found by two binary
//               searches of the cell table.  The search stops when the k-th best d2 is below the square of a
//               conservative lower bound on the distance to any cell not yet visited, so the result never
//               depends on the cell size; only the work does.  A query still unfinished after kRingColumns columns
//               (a stray point far from the cloud, a sparse region) sweeps the occupied-cell table once instead,
//               pruned by the same bound, so no query's work grows with the empty space around it.
//   geo_geof    one thread per vertex: the vertex and its k neighbours, fp64 mean and covariance (centred on the
//               vertex first: translation-free, and exactly zero for coincident points), a cyclic Jacobi
//               eigen-solve, the four features of ply_c.cpp:436-446 in fp64, rounded once to float32
//
// Ranking follows the reference's kd-tree: d2 = (dx dx + dy dy) + dz dz in float64 from float32 coordinates,
// every step rounded explicitly (no contraction), ties broken by the smaller index, the vertex itself excluded
// (sklearn returns it first and the reference drops that column).  The reported distance is float32(sqrt(d2)).
// No float atomics anywhere: every output is reproducible bit for bit.
#include <cub/cub.cuh>

#include "workspace.cuh"
#include "eig3.cuh"

namespace spg {

constexpr int GEO_THREADS = 256;
constexpr int KNN_THREADS = 128;
constexpr int kKnnMaxK = 64;       // neighbours per query (the vertex itself not counted)
constexpr int kGridBits = 21;      // per axis
constexpr double kRingMargin = 1e-6;  // in cells: far above the rounding of a point's cell coordinate (< 2^-30)
constexpr int kRingColumns = 128;     // (x, y) columns a query visits ring by ring before it sweeps the cell table

// ------------------------------------------------------------------------------------------------ bounds
// words[0..2] min keys (preset to 0xffffffff), words[3..5] max keys (preset to 0), words[6] status (preset to 0)
__global__ void __launch_bounds__(GEO_THREADS) geo_bounds_kernel(const float* __restrict__ xyz, int64_t n,
                                                                 unsigned* __restrict__ words) {
    SPG_PDL_ENTRY();
    unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u}, bad = 0u;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = __ldg(xyz + 3 * i + c);
            if (!isfinite(v)) {
                bad = 1u;
                continue;
            }
            const unsigned k = float_key(v);
            lo[c] = min(lo[c], k);
            hi[c] = max(hi[c], k);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            lo[c] = min(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
            hi[c] = max(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
        }
        bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (lo[c] != 0xffffffffu) atomicMin(words + c, lo[c]);
            if (hi[c] != 0u) atomicMax(words + 3 + c, hi[c]);
        }
        if (bad) atomicOr(words + 6, 1u);
    }
}

// ------------------------------------------------------------------------------------------------ grid
struct Grid {
    double o[3];   // origin (the box minimum)
    double inv_h;  // 1 / cell size
    int dim[3];    // cells per axis, each < 2^21
};

__device__ __forceinline__ int geo_cell(const Grid& g, float v, int c) {
    const double u = __dmul_rn(__dsub_rn((double)v, g.o[c]), g.inv_h);
    const int64_t q = (int64_t)floor(u);
    return (int)(q < 0 ? 0 : (q >= g.dim[c] ? g.dim[c] - 1 : q));
}

__device__ __forceinline__ uint64_t geo_key(int cx, int cy, int cz) {
    return ((uint64_t)cx << (2 * kGridBits)) | ((uint64_t)cy << kGridBits) | (uint64_t)cz;
}

__global__ void __launch_bounds__(GEO_THREADS) geo_keys_kernel(const float* __restrict__ xyz, int64_t n, const Grid g,
                                                               uint64_t* __restrict__ keys, int32_t* __restrict__ idx) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = geo_key(geo_cell(g, __ldg(xyz + 3 * i), 0), geo_cell(g, __ldg(xyz + 3 * i + 1), 1),
                      geo_cell(g, __ldg(xyz + 3 * i + 2), 2));
    idx[i] = (int32_t)i;
}

__global__ void __launch_bounds__(GEO_THREADS) geo_gather_kernel(const float* __restrict__ xyz, int64_t n,
                                                                 const int32_t* __restrict__ order,
                                                                 float4* __restrict__ sorted_xyz) {
    SPG_PDL_ENTRY();
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t i = __ldg(order + p);
    sorted_xyz[p] = make_float4(__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2), 0.f);
}

// ------------------------------------------------------------------------------------------------ query
struct KnnArgs {
    Grid g;
    int64_t n;
    int k;                      // neighbours searched (k_nn2)
    int k1;                     // neighbours of the graph outputs (k_nn1 <= k)
    const float4* sorted_xyz;   // [n]
    const int32_t* order;       // [n] original index of every sorted position
    const uint64_t* keys;       // [n] sorted cell keys
    const uint64_t* cell_keys;  // [n_cells] occupied cells, ascending
    const int32_t* cell_start;  // [n_cells + 1] first sorted position of every cell, n last
    const int32_t* n_cells;     // [1]
    int64_t* source;            // [n k1]
    int64_t* target;            // [n k1]
    float* distances;           // [n k1]
    int64_t* target2;           // [n k] or null
};

// first cell index with key >= x
__device__ __forceinline__ int geo_lower_bound(const uint64_t* __restrict__ a, int n, uint64_t x) {
    int lo = 0, len = n;
    while (len > 0) {
        const int half = len >> 1;
        if (__ldg(a + lo + half) < x) {
            lo += half + 1;
            len -= half + 1;
        } else {
            len = half;
        }
    }
    return lo;
}

// (d, j) ranks before (e, l): smaller d2, then smaller index
__device__ __forceinline__ bool geo_before(double d, int j, double e, int l) { return d < e || (d == e && j < l); }

__global__ void __launch_bounds__(KNN_THREADS) geo_knn_kernel(const KnnArgs a) {
    SPG_PDL_ENTRY();
    extern __shared__ unsigned char geo_smem[];
    const int t = threadIdx.x, T = blockDim.x;
    const int64_t p = (int64_t)blockIdx.x * T + t;
    if (p >= a.n) return;
    double* D = reinterpret_cast<double*>(geo_smem);  // [k][T]
    int* I = reinterpret_cast<int*>(D + (size_t)a.k * T);  // [k][T]
    const int k = a.k, n_cells = __ldg(a.n_cells);
    const float4 q = __ldg(a.sorted_xyz + p);
    const int self = __ldg(a.order + p);
    const uint64_t key = __ldg(a.keys + p);
    const int mask = (1 << kGridBits) - 1;
    const int c[3] = {(int)(key >> (2 * kGridBits)), (int)(key >> kGridBits) & mask, (int)key & mask};
    const double qd[3] = {(double)q.x, (double)q.y, (double)q.z};
    // the query's coordinates in cell units, for the lower bound on unvisited cells
    double u[3];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) u[ax] = __dmul_rn(__dsub_rn(qd[ax], a.g.o[ax]), a.g.inv_h);
    const double h = 1.0 / a.g.inv_h;
    int count = 0;
    double worst = 0.0;  // D[k - 1] once count == k
    int worst_id = 0;

    auto scan_points = [&](int s0, int s1) {
        for (int s = s0; s < s1; ++s) {
            if (s == p) continue;
            const float4 v = __ldg(a.sorted_xyz + s);
            const double dx = __dsub_rn(qd[0], (double)v.x);
            const double dy = __dsub_rn(qd[1], (double)v.y);
            const double dz = __dsub_rn(qd[2], (double)v.z);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            if (count == k && d2 > worst) continue;
            const int j = __ldg(a.order + s);
            if (count == k && !geo_before(d2, j, worst, worst_id)) continue;
            int pos = count < k ? count : k - 1;
            while (pos > 0) {
                const double e = D[(size_t)(pos - 1) * T + t];
                const int l = I[(size_t)(pos - 1) * T + t];
                if (!geo_before(d2, j, e, l)) break;
                D[(size_t)pos * T + t] = e;
                I[(size_t)pos * T + t] = l;
                --pos;
            }
            D[(size_t)pos * T + t] = d2;
            I[(size_t)pos * T + t] = j;
            if (count < k) ++count;
            if (count == k) {
                worst = D[(size_t)(k - 1) * T + t];
                worst_id = I[(size_t)(k - 1) * T + t];
            }
        }
    };
    auto scan = [&](int cx, int cy, int z0, int z1) {
        const int c0 = geo_lower_bound(a.cell_keys, n_cells, geo_key(cx, cy, z0));
        const int c1 = geo_lower_bound(a.cell_keys, n_cells, geo_key(cx, cy, z1) + 1);
        if (c0 < c1) scan_points(__ldg(a.cell_start + c0), __ldg(a.cell_start + c1));
    };
    // true when no point at `gap` cells (minus the margin) or more from the query can rank among the k best
    auto beyond = [&](double gap2) { return count == k && gap2 * h * h * (1.0 - 1e-12) > worst; };
    auto axis_gap = [&](int cc, int ax) {
        const double g = cc > c[ax] ? (double)cc - u[ax] : (cc < c[ax] ? u[ax] - (double)(cc + 1) : 0.0);
        return fmax(g - kRingMargin, 0.0);
    };

    int r_done = -1;  // every cell within Chebyshev distance r_done of the query's cell has been scanned
    bool done = false;
    int columns = 0;
    for (int r = 0; !done; ++r) {
        const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, a.g.dim[0] - 1);
        const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, a.g.dim[1] - 1);
        const int z0 = max(c[2] - r, 0), z1 = min(c[2] + r, a.g.dim[2] - 1);
        columns += (x1 - x0 + 1) * (y1 - y0 + 1);
        if (columns > kRingColumns) break;  // far from its neighbours: sweep the cell table instead
        for (int cx = x0; cx <= x1; ++cx) {
            const bool xs = abs(cx - c[0]) == r;
            for (int cy = y0; cy <= y1; ++cy) {
                if (xs || abs(cy - c[1]) == r) {
                    scan(cx, cy, z0, z1);  // a column on the ring's xy shell: all of its z
                } else {
                    if (c[2] - r >= 0) scan(cx, cy, c[2] - r, c[2] - r);  // inside: only the two z caps
                    if (r > 0 && c[2] + r < a.g.dim[2]) scan(cx, cy, c[2] + r, c[2] + r);
                }
            }
        }
        r_done = r;
        // every unvisited cell lies beyond the box of cells [c - r, c + r] along some axis that still has cells
        // there; its points are at least `gap` cells from the query along that axis
        double gap = 1e300;
        bool more = false;
#pragma unroll
        for (int ax = 0; ax < 3; ++ax) {
            if (c[ax] - r > 0) {
                gap = fmin(gap, u[ax] - (double)(c[ax] - r));
                more = true;
            }
            if (c[ax] + r < a.g.dim[ax] - 1) {
                gap = fmin(gap, (double)(c[ax] + r + 1) - u[ax]);
                more = true;
            }
        }
        const double L = fmax(gap - kRingMargin, 0.0);
        done = !more || (L > 0.0 && beyond(L * L));
    }
    if (!done) {
        // One sweep of the occupied-cell table outwards from the query's own cell, in both directions, always
        // taking the side whose next cell is nearer along x.  The table is x-major, so along each side the x gap
        // only grows: a side stops once that gap alone rules its cells out.  Cells already scanned by the rings are
        // skipped, and every other cell is scanned unless its lower bound rules it out.  The work is at most one
        // pass over the table, whatever the empty space around the query.
        const int own = geo_lower_bound(a.cell_keys, n_cells, key);
        int up = own, dn = own - 1;
        while (true) {
            double gu = 1e300, gd = 1e300;
            uint64_t ku = 0, kd = 0;
            if (up < n_cells) {
                ku = __ldg(a.cell_keys + up);
                gu = axis_gap((int)(ku >> (2 * kGridBits)), 0);
                if (beyond(gu * gu)) up = n_cells;
            }
            if (dn >= 0) {
                kd = __ldg(a.cell_keys + dn);
                gd = axis_gap((int)(kd >> (2 * kGridBits)), 0);
                if (beyond(gd * gd)) dn = -1;
            }
            const bool has_up = up < n_cells, has_dn = dn >= 0;
            if (!has_up && !has_dn) break;
            const bool take_up = has_up && (!has_dn || gu <= gd);
            const int ci = take_up ? up++ : dn--;
            const uint64_t kc = take_up ? ku : kd;
            const int cc[3] = {(int)(kc >> (2 * kGridBits)), (int)(kc >> kGridBits) & mask, (int)kc & mask};
            if (max(abs(cc[0] - c[0]), max(abs(cc[1] - c[1]), abs(cc[2] - c[2]))) <= r_done) continue;
            const double g0 = axis_gap(cc[0], 0), g1 = axis_gap(cc[1], 1), g2 = axis_gap(cc[2], 2);
            if (beyond(g0 * g0 + g1 * g1 + g2 * g2)) continue;
            scan_points(__ldg(a.cell_start + ci), __ldg(a.cell_start + ci + 1));
        }
    }
    const int64_t i = self;
    for (int j = 0; j < k; ++j) {
        const int id = I[(size_t)j * T + t];
        if (a.target2) a.target2[i * k + j] = id;
        if (j < a.k1) {
            a.source[i * a.k1 + j] = i;
            a.target[i * a.k1 + j] = id;
            a.distances[i * a.k1 + j] = __double2float_rn(__dsqrt_rn(D[(size_t)j * T + t]));
        }
    }
}

// ------------------------------------------------------------------------------------------------ geof
__global__ void __launch_bounds__(GEO_THREADS) geo_geof_kernel(const float* __restrict__ xyz, int64_t n,
                                                               const int64_t* __restrict__ target, int k,
                                                               float* __restrict__ geof, unsigned* __restrict__ status) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x0 = __ldg(xyz + 3 * i), y0 = __ldg(xyz + 3 * i + 1), z0 = __ldg(xyz + 3 * i + 2);
    // positions relative to the vertex: the first pass sums them, the second the centred products
    double sx = 0.0, sy = 0.0, sz = 0.0;
    bool bad = false;
    for (int j = 0; j < k; ++j) {
        const int64_t u = __ldg(target + i * k + j);
        if (u < 0 || u >= n) {
            bad = true;
            continue;
        }
        sx += (double)__ldg(xyz + 3 * u) - x0;
        sy += (double)__ldg(xyz + 3 * u + 1) - y0;
        sz += (double)__ldg(xyz + 3 * u + 2) - z0;
    }
    float4 out = make_float4(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff), __int_as_float(0x7fffffff),
                             __int_as_float(0x7fffffff));
    if (bad) {
        atomicOr(status, 2u);
        reinterpret_cast<float4*>(geof)[i] = out;
        return;
    }
    const double inv = 1.0 / (double)(k + 1);
    const double mx = sx * inv, my = sy * inv, mz = sz * inv;
    // the vertex itself, at relative position 0
    double cxx = mx * mx, cxy = mx * my, cxz = mx * mz, cyy = my * my, cyz = my * mz, czz = mz * mz;
    for (int j = 0; j < k; ++j) {
        const int64_t u = __ldg(target + i * k + j);
        const double dx = (double)__ldg(xyz + 3 * u) - x0 - mx;
        const double dy = (double)__ldg(xyz + 3 * u + 1) - y0 - my;
        const double dz = (double)__ldg(xyz + 3 * u + 2) - z0 - mz;
        cxx += dx * dx;
        cxy += dx * dy;
        cxz += dx * dz;
        cyy += dy * dy;
        cyz += dy * dz;
        czz += dz * dz;
    }
    double A[3][3] = {{cxx * inv, cxy * inv, cxz * inv}, {cxy * inv, cyy * inv, cyz * inv},
                      {cxz * inv, cyz * inv, czz * inv}};
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    geo_jacobi(A, V);
    // eigenvalues descending with their vectors (ply_c.cpp:418-422), clamped at 0 (:423-425)
    double e[3] = {A[0][0], A[1][1], A[2][2]};
    double v[3][3] = {{V[0][0], V[1][0], V[2][0]}, {V[0][1], V[1][1], V[2][1]}, {V[0][2], V[1][2], V[2][2]}};
    geo_order(e, v, 0, 1);
    geo_order(e, v, 1, 2);
    geo_order(e, v, 0, 1);
    const double l0 = fmax(e[0], 0.0), l1 = fmax(e[1], 0.0), l2 = fmax(e[2], 0.0);
    const double s0 = sqrt(l0), s1 = sqrt(l1), s2 = sqrt(l2);
    // ply_c.cpp:436-446; l0 == 0 gives 0 / 0 in every column, as in the reference
    double uv[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) uv[r] = l0 * fabs(v[0][r]) + l1 * fabs(v[1][r]) + l2 * fabs(v[2][r]);
    const double norm = sqrt(uv[0] * uv[0] + uv[1] * uv[1] + uv[2] * uv[2]);
    out.x = (float)((s0 - s1) / s0);
    out.y = (float)((s1 - s2) / s0);
    out.z = (float)(s2 / s0);
    out.w = (float)(uv[2] / norm);
    reinterpret_cast<float4*>(geof)[i] = out;
}

// ------------------------------------------------------------------------------------------------ plan
struct KnnWs {
    uint64_t *keys_in, *keys;
    int32_t *idx_in, *order;
    float4* sorted_xyz;
    uint64_t* cell_keys;
    int32_t *cell_count, *cell_start, *n_cells;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n, void* base, KnnWs* w) {
    const int m = (int)(n > 0 ? n : 1);
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (const int32_t*)nullptr, (int32_t*)nullptr, m, 0, 3 * kGridBits);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRunLengthEncode::Encode, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                  (int32_t*)nullptr, (int32_t*)nullptr, m);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int32_t*)nullptr, (int32_t*)nullptr, m + 1);
    const size_t N = (size_t)m;
    Planner p(base);
    w->keys_in = p.take<uint64_t>(N);
    w->keys = p.take<uint64_t>(N);
    w->idx_in = p.take<int32_t>(N);
    w->order = p.take<int32_t>(N);
    w->sorted_xyz = p.take<float4>(N);
    w->cell_keys = p.take<uint64_t>(N);
    w->cell_count = p.take<int32_t>(N + 1);
    w->cell_start = p.take<int32_t>(N + 1);
    w->n_cells = p.take<int32_t>(1);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

static int make_grid(double ox, double oy, double oz, double cell, int64_t dx, int64_t dy, int64_t dz, Grid* g) {
    if (!(cell > 0.0) || !isfinite(cell)) return SPG_E_BADARG;
    const int64_t lim = 1ll << kGridBits;
    if (dx < 1 || dy < 1 || dz < 1 || dx >= lim || dy >= lim || dz >= lim) return SPG_E_UNSUPPORTED;
    g->o[0] = ox;
    g->o[1] = oy;
    g->o[2] = oz;
    g->inv_h = 1.0 / cell;
    g->dim[0] = (int)dx;
    g->dim[1] = (int)dy;
    g->dim[2] = (int)dz;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_knn_max_k(void) { return kKnnMaxK; }

int spg_knn_workspace(int64_t n, int64_t* bytes) {
    if (!bytes || n < 0) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    KnnWs w;
    const int rc = layout(n, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_knn_bounds(const float* xyz, int64_t n, uint32_t* words, spg_stream_t stream) {
    if (n < 0 || !words || (n > 0 && !xyz)) return SPG_E_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(words, 0xff, 3 * sizeof(uint32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(words + 3, 0, 5 * sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n == 0) return SPG_OK;
    const int64_t blocks = ceil_div64(n, GEO_THREADS);
    SPG_LAUNCH(K_GEO_BOUNDS, s, geo_bounds_kernel, (unsigned)(blocks < 4 * kNumSMs ? blocks : 4 * kNumSMs),
               GEO_THREADS, 0, xyz, n, (unsigned*)words);
    return launch_status();
}

int spg_knn_grid(const float* xyz, int64_t n, double ox, double oy, double oz, double cell, int64_t dim_x,
                 int64_t dim_y, int64_t dim_z, void* workspace, int64_t workspace_bytes, int32_t* n_cells,
                 spg_stream_t stream) {
    if (n <= 0 || !xyz || !n_cells) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    KnnWs w;
    int rc = layout(n, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    Grid g;
    rc = make_grid(ox, oy, oz, cell, dim_x, dim_y, dim_z, &g);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)ceil_div64(n, GEO_THREADS);
    SPG_LAUNCH(K_GEO_GRID, s, geo_keys_kernel, blocks, GEO_THREADS, 0, xyz, n, g, w.keys_in, w.idx_in);
    SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const uint64_t*)w.keys_in, w.keys, (const int32_t*)w.idx_in,
            w.order, (int)n, 0, 3 * kGridBits, s);
    SPG_LAUNCH(K_GEO_GRID, s, geo_gather_kernel, blocks, GEO_THREADS, 0, xyz, n, (const int32_t*)w.order,
               w.sorted_xyz);
    // counts beyond the last cell stay 0, so the scan puts n at cell_start[n_cells] (and after it)
    cudaError_t e = cudaMemsetAsync(w.cell_count, 0, ((size_t)n + 1) * 4, s);
    if (e != cudaSuccess) return (int)e;
    SPG_CUB(w.cub, cub::DeviceRunLengthEncode::Encode, (const uint64_t*)w.keys, w.cell_keys, w.cell_count, w.n_cells,
            (int)n, s);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int32_t*)w.cell_count, w.cell_start, (int)n + 1, s);
    e = cudaMemcpyAsync(n_cells, w.n_cells, sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return (int)e;
    return launch_status();
}

int spg_knn_query(int64_t n, int k, int k1, double ox, double oy, double oz, double cell, int64_t dim_x,
                  int64_t dim_y, int64_t dim_z, const void* workspace, int64_t workspace_bytes, int64_t* source,
                  int64_t* target, float* distances, int64_t* target2, spg_stream_t stream) {
    if (n <= 0 || k <= 0 || k1 <= 0 || k1 > k || !source || !target || !distances) return SPG_E_BADARG;
    if (k > kKnnMaxK || too_big(n)) return SPG_E_UNSUPPORTED;
    if (n < (int64_t)k + 1) return SPG_E_BADARG;
    KnnWs w;
    int rc = layout(n, const_cast<void*>(workspace), &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    KnnArgs a;
    rc = make_grid(ox, oy, oz, cell, dim_x, dim_y, dim_z, &a.g);
    if (rc != SPG_OK) return rc;
    a.n = n;
    a.k = k;
    a.k1 = k1;
    a.sorted_xyz = w.sorted_xyz;
    a.order = w.order;
    a.keys = w.keys;
    a.cell_keys = w.cell_keys;
    a.cell_start = w.cell_start;
    a.n_cells = w.n_cells;
    a.source = source;
    a.target = target;
    a.distances = distances;
    a.target2 = target2;
    const size_t smem = (size_t)k * KNN_THREADS * (sizeof(double) + sizeof(int));
    const cudaError_t e = cudaFuncSetAttribute(geo_knn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(K_GEO_KNN, (cudaStream_t)stream, geo_knn_kernel, (unsigned)ceil_div64(n, KNN_THREADS), KNN_THREADS,
               smem, a);
    return launch_status();
}

int spg_geof(const float* xyz, int64_t n, const int64_t* target, int k, float* geof, uint32_t* status,
             spg_stream_t stream) {
    if (n < 0 || k <= 0 || !status) return SPG_E_BADARG;
    if (too_big(n)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(status, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return (int)e;
    if (n == 0) return SPG_OK;
    if (!xyz || !target || !geof) return SPG_E_BADARG;
    if ((reinterpret_cast<uintptr_t>(geof) & 15) != 0) return SPG_E_ALIGN;
    SPG_LAUNCH(K_GEO_GEOF, s, geo_geof_kernel, (unsigned)ceil_div64(n, GEO_THREADS), GEO_THREADS, 0, xyz, n, target,
               k, geof, (unsigned*)status);
    return launch_status();
}

}  // extern "C"
