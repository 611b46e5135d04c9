// The learned partition's batch builder (ref: supervized_partition/graph_processing.py:347-436 `graph_loader`,
// :439-472 `graph_collate`, :534-546 `augment_cloud_whole`; partition/ply_c/random_subgraph.cpp:91-95), for the
// learned-embedding branch.  The per-file arrays stay resident in HBM; every launch below serves one file of the
// batch and writes its slice of the collated outputs:
//
//   lp_augment       rgb / 255, and for training the rotation about z around a reference vertex and the jitter
//                    (host noise, or Philox4x32-10 keyed by (seed, file position)), into batch scratch
//   lp_subgraph      vertex renumbering by a scan of the vertex mask, the edge mask sel[u] * sel[v] and its scan,
//                    the stable compaction of the kept edges (plus the collate's vertex offset), the per-file
//                    object maximum (integer atomicMax: order-free) and the collate's object offsets
//   lp_local_clouds  one warp per selected vertex: the k neighbours' xyz (and rgb), numpy's sequential fp32
//                    mean / variance, the normalised [F, k] cloud, the global-feature row, labels, objects, xyz
//
// Floating point follows numpy's evaluation order exactly (every step plain sequential fp32, rounded
// explicitly so that nvcc cannot contract a multiply-add), so everything but the rotation is bit-identical to
// the reference; the rotation is BLAS's float32 matmul on the host, whose last bit is not promised.
#include <cub/cub.cuh>

#include "workspace.cuh"
#include "philox.cuh"

namespace spg {

constexpr int LPL_THREADS = 256;
constexpr int kLclWarps = 8;  // warps (selected vertices) per CTA of lp_local_clouds
constexpr int kLclMaxK = 256;

enum { LPL_GLOBAL_E = 1, LPL_GLOBAL_RGB = 2, LPL_GLOBAL_XYN = 4, LPL_GLOBAL_XY = 8 };

// ------------------------------------------------------------------------------------------------ augment
// Standard normal from two 32-bit words (Box-Muller, u in (0, 1)); `second` picks the sine branch.
__device__ __forceinline__ float lpl_normal(uint32_t w0, uint32_t w1, bool second) {
    const float u0 = ((float)(w0 >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u1 = ((float)(w1 >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float r = sqrtf(-2.f * logf(u0));
    return second ? r * sinpif(2.f * u1) : r * cospif(2.f * u1);
}

// clip(sigma * N(0, 1), -clip, clip) for the three coordinates of vertex v (stream 0: xyz, 1: rgb)
__device__ __forceinline__ void lpl_device_noise(uint64_t seed, uint64_t file_pos, int64_t v, uint32_t which,
                                                 float sigma, float clip, float out[3]) {
    const Philox4 w = philox4x32_10((uint32_t)v, (uint32_t)((uint64_t)v >> 32), (uint32_t)file_pos,
                                    which, (uint32_t)seed, (uint32_t)(seed >> 32));
    const float g[3] = {lpl_normal(w.v[0], w.v[1], false), lpl_normal(w.v[0], w.v[1], true),
                        lpl_normal(w.v[2], w.v[3], false)};
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = fminf(fmaxf(__fmul_rn(sigma, g[c]), -clip), clip);
}

struct AugmentArgs {
    const float* xyz;  // [n, 3] resident
    const float* rgb;  // [n, 3] resident (0..255)
    int64_t n;
    const float* rot;  // [9]: M row-major (float32), or null
    int64_t ref_index;
    const float* noise_xyz;  // [n, 3] clipped host noise, or null
    const float* noise_rgb;  // [n, 3] or null
    int device_noise;        // 1: Philox noise for xyz (and rgb when rgb_jitter)
    int rgb_jitter;
    float sigma, clip;
    uint64_t seed, file_pos;
    float* xyz_out;  // [n, 3]
    float* rgb_out;  // [n, 3]
};

__global__ void __launch_bounds__(LPL_THREADS) lp_augment_kernel(const AugmentArgs a) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= a.n) return;
    float p[3], q[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = __ldg(a.xyz + 3 * v + c);
    if (a.rot) {
        // ref_point is a view of xyz in the reference (:537-538): its own z is 0 when the rotation reads it
        if (v == a.ref_index) p[2] = 0.f;
        const float ref[3] = {__ldg(a.xyz + 3 * a.ref_index), __ldg(a.xyz + 3 * a.ref_index + 1), 0.f};
        const float d[3] = {__fsub_rn(p[0], ref[0]), __fsub_rn(p[1], ref[1]), __fsub_rn(p[2], ref[2])};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float acc = __fmul_rn(d[0], a.rot[j]);
            acc = __fmaf_rn(d[1], a.rot[3 + j], acc);
            acc = __fmaf_rn(d[2], a.rot[6 + j], acc);
            q[j] = __fadd_rn(acc, ref[j]);
        }
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c] = p[c];
    }
    float r[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = __fdiv_rn(__ldg(a.rgb + 3 * v + c), 255.f);
    float nz[3];
    if (a.noise_xyz || a.device_noise) {
        if (a.device_noise) lpl_device_noise(a.seed, a.file_pos, v, 0u, a.sigma, a.clip, nz);
        else
#pragma unroll
            for (int c = 0; c < 3; ++c) nz[c] = __ldg(a.noise_xyz + 3 * v + c);
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c] = __fadd_rn(q[c], nz[c]);
        if (a.rgb_jitter) {
            if (a.device_noise) lpl_device_noise(a.seed, a.file_pos, v, 1u, a.sigma, a.clip, nz);
            else
#pragma unroll
                for (int c = 0; c < 3; ++c) nz[c] = __ldg(a.noise_rgb + 3 * v + c);
#pragma unroll
            for (int c = 0; c < 3; ++c) r[c] = fminf(fmaxf(__fadd_rn(r[c], nz[c]), -1.f), 1.f);
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        a.xyz_out[3 * v + c] = q[c];
        a.rgb_out[3 * v + c] = r[c];
    }
}

// ------------------------------------------------------------------------------------------------ subgraph
// object maxima are kept as uint32 (id ^ 0x80000000), an order-preserving map, so that a zeroed word is
// below every id
__device__ __forceinline__ unsigned obj_key(int o) { return (unsigned)o ^ 0x80000000u; }

__global__ void __launch_bounds__(LPL_THREADS)
lp_subgraph_flags_kernel(const uint8_t* __restrict__ mask, int64_t n_ver, const int32_t* __restrict__ src,
                         const int32_t* __restrict__ tgt, int64_t n_edges, int* __restrict__ vflag,
                         int* __restrict__ eflag) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_ver) vflag[i] = mask[i] != 0;
    if (i < n_edges) eflag[i] = (mask[__ldg(src + i)] != 0) & (mask[__ldg(tgt + i)] != 0);  // random_subgraph.cpp:91-95
}

// selected[new_index[v]] = v for the kept vertices; object maximum over them (all vertices without a mask)
__global__ void __launch_bounds__(LPL_THREADS)
lp_subgraph_vertices_kernel(const uint8_t* __restrict__ mask, int64_t n_ver, const int32_t* __restrict__ new_index,
                            const int32_t* __restrict__ objects, int32_t* __restrict__ selected,
                            unsigned* __restrict__ object_max) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned m = 0u;
    if (v < n_ver && (!mask || mask[v])) {
        if (mask) selected[new_index[v]] = (int32_t)v;
        m = obj_key(__ldg(objects + v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(object_max, m);
}

// the kept edges in their order, renumbered and shifted by the file's first vertex in the batch
__global__ void __launch_bounds__(LPL_THREADS)
lp_subgraph_edges_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ tgt,
                         const uint8_t* __restrict__ is_tr, int64_t n_edges, const int32_t* __restrict__ new_index,
                         const int32_t* __restrict__ edge_pos, int64_t vertex_offset, int64_t* __restrict__ src_out,
                         int64_t* __restrict__ tgt_out, uint8_t* __restrict__ tr_out) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    int64_t s = __ldg(src + e), t = __ldg(tgt + e), o = e;
    if (new_index) {
        o = __ldg(edge_pos + e);
        if (__ldg(edge_pos + e + 1) == o) return;  // not kept
        s = __ldg(new_index + s);
        t = __ldg(new_index + t);
    }
    src_out[o] = s + vertex_offset;
    tgt_out[o] = t + vertex_offset;
    tr_out[o] = is_tr[e];
}

// graph_collate's object offsets (:447,467): offset[b] = sum over b' < b of max(objects of b'), an empty file
// adding 0
__global__ void lp_object_offsets_kernel(const unsigned* __restrict__ object_max, const int64_t* __restrict__ counts,
                                         int64_t n_files, int64_t* __restrict__ offsets) {
    SPG_PDL_ENTRY();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int64_t acc = 0;
    for (int64_t b = 0; b < n_files; ++b) {
        offsets[b] = acc;
        if (counts[b] > 0) acc += (int64_t)(int)(object_max[b] ^ 0x80000000u);
    }
}

// ------------------------------------------------------------------------------------------------ clouds
struct LocalCloudArgs {
    const float* xyz;  // [n, 3] augmented (or resident) xyz of the whole file
    const float* rgb;  // [n, 3]
    int rgb_scale;     // 1: rgb is the resident 0..255 array, divided by 255 here
    const int32_t* geometry;  // [n, ld_geometry] neighbour ids of the file
    int64_t ld_geometry;
    int k;
    const int32_t* selected;  // [n_sel] kept vertices in increasing order, or null (all)
    int64_t n_sel;
    const float* elevation;   // [n]
    const float* xyn;         // [n, 2]
    const int32_t* labels;    // [n, n_label_cols]
    int64_t n_label_cols;
    const int32_t* objects;   // [n]
    const int64_t* object_offset;  // [1]
    int use_rgb, global_flags;
    float* clouds;          // [n_sel, 3 + 3 use_rgb, k]
    float* clouds_global;   // [n_sel, ld_global]
    int64_t ld_global;
    float* xyz_out;         // [n_sel, 3]
    int64_t* labels_out;    // [n_sel, n_label_cols]
    int64_t* objects_out;   // [n_sel]
};

__device__ __forceinline__ float lpl_rgb(const LocalCloudArgs& a, int64_t v, int c) {
    const float r = __ldg(a.rgb + 3 * v + c);
    return a.rgb_scale ? __fdiv_rn(r, 255.f) : r;
}

__global__ void __launch_bounds__(kLclWarps * 32) lp_local_clouds_kernel(const LocalCloudArgs a) {
    SPG_PDL_ENTRY();
    __shared__ float sm[kLclWarps][3 * kLclMaxK + 8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kLclWarps + warp;
    if (i >= a.n_sel) return;
    const int k = a.k;
    float* pts = sm[warp];         // [k][3]
    float* red = pts + 3 * k;      // the variances of x, y, z
    const int64_t v = a.selected ? (int64_t)__ldg(a.selected + i) : i;
    const int32_t* nei = a.geometry + v * a.ld_geometry;
    for (int j = lane; j < k; j += 32) {
        const int64_t u = __ldg(nei + j);
#pragma unroll
        for (int c = 0; c < 3; ++c) pts[3 * j + c] = __ldg(a.xyz + 3 * u + c);
    }
    __syncwarp();
    // np.sqrt(clouds.var(1).sum(1)): per coordinate sequential sums over the k neighbours
    if (lane < 3) {
        float s = 0.f;
        for (int j = 0; j < k; ++j) s = __fadd_rn(s, pts[3 * j + lane]);
        const float m = __fdiv_rn(s, (float)k);
        float q = 0.f;
        for (int j = 0; j < k; ++j) {
            const float d = __fsub_rn(pts[3 * j + lane], m);
            q = __fadd_rn(q, __fmul_rn(d, d));
        }
        red[lane] = __fdiv_rn(q, (float)k);
    }
    __syncwarp();
    const float diam = __fsqrt_rn(__fadd_rn(__fadd_rn(red[0], red[1]), red[2]));
    const float den = __fadd_rn(diam, 1e-10f);
    const float cx = __ldg(a.xyz + 3 * v), cy = __ldg(a.xyz + 3 * v + 1), cz = __ldg(a.xyz + 3 * v + 2);
    const int F = a.use_rgb ? 6 : 3;
    float* out = a.clouds + i * F * k;
    for (int j = lane; j < k; j += 32) {
        out[j] = __fdiv_rn(__fsub_rn(pts[3 * j], cx), den);
        out[k + j] = __fdiv_rn(__fsub_rn(pts[3 * j + 1], cy), den);
        out[2 * k + j] = __fdiv_rn(__fsub_rn(pts[3 * j + 2], cz), den);
        if (a.use_rgb) {
            const int64_t u = __ldg(nei + j);
#pragma unroll
            for (int c = 0; c < 3; ++c) out[(3 + c) * k + j] = lpl_rgb(a, u, c);
        }
    }
    // clouds_global = [diameter | elevation | rgb | xyn | xy] (:403-411)
    float* g = a.clouds_global + i * a.ld_global;
    if (lane == 0) {
        int col = 0;
        g[col++] = diam;
        if (a.global_flags & LPL_GLOBAL_E) g[col++] = __ldg(a.elevation + v);
        if (a.global_flags & LPL_GLOBAL_RGB)
            for (int c = 0; c < 3; ++c) g[col++] = lpl_rgb(a, v, c);
        if (a.global_flags & LPL_GLOBAL_XYN) {
            g[col++] = __ldg(a.xyn + 2 * v);
            g[col++] = __ldg(a.xyn + 2 * v + 1);
        }
        if (a.global_flags & LPL_GLOBAL_XY) {
            g[col++] = cx;
            g[col++] = cy;
        }
        a.xyz_out[3 * i] = cx;
        a.xyz_out[3 * i + 1] = cy;
        a.xyz_out[3 * i + 2] = cz;
        a.objects_out[i] = (int64_t)__ldg(a.objects + v) + a.object_offset[0];
    }
    for (int64_t c = lane; c < a.n_label_cols; c += 32)
        a.labels_out[i * a.n_label_cols + c] = (int64_t)__ldg(a.labels + v * a.n_label_cols + c);
}

struct SubgraphWs {
    int *vflag, *eflag;
    CubRegion cub;
    size_t bytes;
};

static int layout(int64_t n_ver, int64_t n_edges, void* base, SubgraphWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::InclusiveSum, (const int*)nullptr, (int*)nullptr,
                  (int)(n_ver > 0 ? n_ver : 1));
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::InclusiveSum, (const int*)nullptr, (int*)nullptr,
                  (int)(n_edges > 0 ? n_edges : 1));
    Planner p(base);
    w->vflag = p.take<int>(n_ver);
    w->eflag = p.take<int>(n_edges);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_lp_augment(const float* xyz, const float* rgb, int64_t n_ver, const float* rot, int64_t ref_index,
                   const float* noise_xyz, const float* noise_rgb, int device_noise, int rgb_jitter, float sigma,
                   float clip, int64_t seed, int64_t file_pos, float* xyz_out, float* rgb_out, spg_stream_t stream) {
    if (n_ver < 0) return SPG_E_BADARG;
    if (n_ver == 0) return SPG_OK;
    if (!xyz || !rgb || !xyz_out || !rgb_out) return SPG_E_BADARG;
    if (rot && (ref_index < 0 || ref_index >= n_ver)) return SPG_E_BADARG;
    // rgb is jittered only together with xyz (graph_processing.py:541-545): without xyz noise the flag is moot
    rgb_jitter = (noise_xyz || device_noise) && rgb_jitter;
    if (rgb_jitter && !device_noise && !noise_rgb) return SPG_E_BADARG;
    AugmentArgs a;
    a.xyz = xyz;
    a.rgb = rgb;
    a.n = n_ver;
    a.rot = rot;
    a.ref_index = ref_index;
    a.noise_xyz = noise_xyz;
    a.noise_rgb = noise_rgb;
    a.device_noise = device_noise;
    a.rgb_jitter = rgb_jitter;
    a.sigma = sigma;
    a.clip = clip;
    a.seed = (uint64_t)seed;
    a.file_pos = (uint64_t)file_pos;
    a.xyz_out = xyz_out;
    a.rgb_out = rgb_out;
    SPG_LAUNCH(K_LP_AUGMENT, (cudaStream_t)stream, lp_augment_kernel, (unsigned)ceil_div64(n_ver, LPL_THREADS),
               LPL_THREADS, 0, a);
    return launch_status();
}

int spg_lp_subgraph_workspace(int64_t n_ver, int64_t n_edges, int64_t* bytes) {
    if (!bytes || n_ver < 0 || n_edges < 0) return SPG_E_BADARG;
    if (too_big(n_ver) || too_big(n_edges)) return SPG_E_UNSUPPORTED;
    SubgraphWs w;
    const int rc = layout(n_ver, n_edges, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_lp_subgraph_select(const uint8_t* mask, const int32_t* objects, int64_t n_ver, const int32_t* src,
                           const int32_t* tgt, int64_t n_edges, int32_t* new_index, int32_t* selected,
                           int32_t* edge_pos, uint32_t* object_max, void* workspace, int64_t workspace_bytes,
                           spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || !object_max) return SPG_E_BADARG;
    if (too_big(n_ver) || too_big(n_edges)) return SPG_E_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(object_max, 0, sizeof(unsigned), s);
    if (e != cudaSuccess) return (int)e;
    if (n_ver > 0 && !objects) return SPG_E_BADARG;
    if (mask) {
        if (!new_index || !edge_pos || (n_ver > 0 && !selected) || (n_edges > 0 && (!src || !tgt)))
            return SPG_E_BADARG;
        SubgraphWs w;
        int rc = layout(n_ver, n_edges, workspace, &w);
        if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
        if (rc != SPG_OK) return rc;
        e = cudaMemsetAsync(new_index, 0, sizeof(int), s);
        if (e == cudaSuccess) e = cudaMemsetAsync(edge_pos, 0, sizeof(int), s);
        if (e != cudaSuccess) return (int)e;
        const int64_t nm = n_ver > n_edges ? n_ver : n_edges;
        if (nm > 0)
            SPG_LAUNCH(K_LP_SUBGRAPH, s, lp_subgraph_flags_kernel, (unsigned)ceil_div64(nm, LPL_THREADS), LPL_THREADS,
                       0, mask, n_ver, src, tgt, n_edges, w.vflag, w.eflag);
        if (n_ver > 0)
            SPG_CUB(w.cub, cub::DeviceScan::InclusiveSum, (const int*)w.vflag, new_index + 1, (int)n_ver, s);
        if (n_edges > 0)
            SPG_CUB(w.cub, cub::DeviceScan::InclusiveSum, (const int*)w.eflag, edge_pos + 1, (int)n_edges, s);
    }
    if (n_ver > 0)
        SPG_LAUNCH(K_LP_SUBGRAPH, s, lp_subgraph_vertices_kernel, (unsigned)ceil_div64(n_ver, LPL_THREADS),
                   LPL_THREADS, 0, mask, n_ver, (const int32_t*)new_index, objects, selected, object_max);
    return launch_status();
}

int spg_lp_subgraph_edges(const int32_t* src, const int32_t* tgt, const uint8_t* is_transition, int64_t n_edges,
                          const int32_t* new_index, const int32_t* edge_pos, int64_t vertex_offset, int64_t* src_out,
                          int64_t* tgt_out, uint8_t* is_transition_out, spg_stream_t stream) {
    if (n_edges < 0 || too_big(n_edges)) return SPG_E_BADARG;
    if (n_edges == 0) return SPG_OK;
    if (!src || !tgt || !is_transition || !src_out || !tgt_out || !is_transition_out) return SPG_E_BADARG;
    if (new_index && !edge_pos) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_SUBGRAPH, (cudaStream_t)stream, lp_subgraph_edges_kernel,
               (unsigned)ceil_div64(n_edges, LPL_THREADS), LPL_THREADS, 0, src, tgt, is_transition, n_edges,
               new_index, edge_pos, vertex_offset, src_out, tgt_out, is_transition_out);
    return launch_status();
}

int spg_lp_object_offsets(const uint32_t* object_max, const int64_t* counts, int64_t n_files, int64_t* offsets,
                          spg_stream_t stream) {
    if (n_files < 0) return SPG_E_BADARG;
    if (n_files == 0) return SPG_OK;
    if (!object_max || !counts || !offsets) return SPG_E_BADARG;
    SPG_LAUNCH(K_LP_SUBGRAPH, (cudaStream_t)stream, lp_object_offsets_kernel, 1, 32, 0, object_max, counts, n_files,
               offsets);
    return launch_status();
}

int spg_lp_local_clouds(const float* xyz, const float* rgb, int rgb_scale, const int32_t* local_geometry,
                        int64_t ld_geometry, int k, const int32_t* selected, int64_t n_sel, const float* elevation,
                        const float* xyn, const int32_t* labels, int64_t n_label_cols, const int32_t* objects,
                        const int64_t* object_offset, int use_rgb, int global_flags, float* clouds,
                        float* clouds_global, int64_t ld_global, float* xyz_out, int64_t* labels_out,
                        int64_t* objects_out, spg_stream_t stream) {
    if (n_sel < 0 || k <= 0 || ld_geometry < k || n_label_cols < 0) return SPG_E_BADARG;
    if (k > kLclMaxK || n_sel >= (1ll << 31)) return SPG_E_UNSUPPORTED;
    if (n_sel == 0) return SPG_OK;
    if (!xyz || !rgb || !local_geometry || !objects || !object_offset || !clouds || !clouds_global || !xyz_out ||
        !objects_out || (n_label_cols > 0 && (!labels || !labels_out)))
        return SPG_E_BADARG;
    if (((global_flags & LPL_GLOBAL_E) && !elevation) || ((global_flags & LPL_GLOBAL_XYN) && !xyn))
        return SPG_E_BADARG;
    const int need = 1 + ((global_flags & LPL_GLOBAL_E) ? 1 : 0) + ((global_flags & LPL_GLOBAL_RGB) ? 3 : 0) +
                     ((global_flags & LPL_GLOBAL_XYN) ? 2 : 0) + ((global_flags & LPL_GLOBAL_XY) ? 2 : 0);
    if (ld_global < need) return SPG_E_BADARG;
    LocalCloudArgs a;
    a.xyz = xyz;
    a.rgb = rgb;
    a.rgb_scale = rgb_scale;
    a.geometry = local_geometry;
    a.ld_geometry = ld_geometry;
    a.k = k;
    a.selected = selected;
    a.n_sel = n_sel;
    a.elevation = elevation;
    a.xyn = xyn;
    a.labels = labels;
    a.n_label_cols = n_label_cols;
    a.objects = objects;
    a.object_offset = object_offset;
    a.use_rgb = use_rgb;
    a.global_flags = global_flags;
    a.clouds = clouds;
    a.clouds_global = clouds_global;
    a.ld_global = ld_global;
    a.xyz_out = xyz_out;
    a.labels_out = labels_out;
    a.objects_out = objects_out;
    SPG_LAUNCH(K_LP_LOCAL_CLOUDS, (cudaStream_t)stream, lp_local_clouds_kernel,
               (unsigned)ceil_div64(n_sel, kLclWarps), kLclWarps * 32, 0, a);
    return launch_status();
}

}  // extern "C"
