// The superpoint graph's batch builder (ref: learning/spg.py:114-143 `random_neighborhoods`, `k_big_enough` and
// the vertex permutation of `loader`, :178-193 `eccpc_collate`, learning/ecc/GraphConvInfo.py:33-69 `set_batch`).
// The graphs stay resident in HBM; the host draws the permutation and the centres (Python's `random`, in the
// reference's order) and every call below serves one graph of the batch:
//
//   sb_select  inverse permutation, a level-synchronous multi-source BFS of depth `order` over the undirected
//              adjacency (the target CSR and the stable source CSR of spg_graph_build; integer atomicCAS on the
//              level word), one int64 scan over permuted positions of the packed (kept, kept and s >= minpts)
//              flags: the sub-graph numbering and the k_big_enough cut at once, then the kept edges' scan
//   sb_edges   stable compaction of the kept edges in file order, CUB's stable radix sort by new target, and the
//              gather of the collated idxn / target rows, in-degrees (integer atomics), edge-feature rows and
//              target rows into the graph's slice of the batch
//
// Integer work only: the outputs are exact.  Within one target the edges keep the file's order (a stable sort),
// where the reference's default-kind argsort leaves it to numpy's unstable sort (DESIGN.md §4).
#include <cub/cub.cuh>

#include "workspace.cuh"

namespace spg {

constexpr int SB_THREADS = 256;
constexpr int kUnseen = 0x7fffffff;

__global__ void __launch_bounds__(SB_THREADS)
sb_init_kernel(const int* __restrict__ perm, int64_t n, int all, int* __restrict__ inv, int* __restrict__ level,
               int* __restrict__ out) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 2) out[i] = 0;
    if (i >= n) return;
    inv[perm ? perm[i] : (int)i] = (int)i;  // perm[i] is the new id of vertex i (igraph's permute_vertices)
    level[i] = all ? 0 : kUnseen;
}

__global__ void __launch_bounds__(SB_THREADS)
sb_centres_kernel(const int* __restrict__ centres, int64_t n_centres, const int* __restrict__ inv,
                  int* __restrict__ level) {
    SPG_PDL_ENTRY();
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n_centres) level[inv[centres[c]]] = 0;
}

// thread per vertex of level l: claims every unseen neighbour, in either edge direction, for level l + 1
__global__ void __launch_bounds__(SB_THREADS)
sb_bfs_kernel(const int* __restrict__ tgt_rowptr, const int* __restrict__ in_src, const int* __restrict__ src_rowptr,
              const int* __restrict__ src_perm, const int* __restrict__ edge_tgt, int64_t n, int l,
              int* __restrict__ level) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n || level[v] != l) return;
    for (int p = tgt_rowptr[v]; p < tgt_rowptr[v + 1]; ++p) {
        const int u = __ldg(in_src + p);
        if (level[u] == kUnseen) atomicCAS(level + u, kUnseen, l + 1);
    }
    for (int p = src_rowptr[v]; p < src_rowptr[v + 1]; ++p) {
        const int u = __ldg(edge_tgt + __ldg(src_perm + p));
        if (level[u] == kUnseen) atomicCAS(level + u, kUnseen, l + 1);
    }
}

// permuted position j: low word 1 if kept by the BFS, high word 1 if also s >= minpts
__global__ void __launch_bounds__(SB_THREADS)
sb_flags_kernel(const int* __restrict__ inv, const int* __restrict__ level, const int64_t* __restrict__ sizes,
                int64_t n, int64_t minpts, long long* __restrict__ packed) {
    SPG_PDL_ENTRY();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int v = inv[j];
    const long long kept = level[v] != kUnseen;
    packed[j] = kept | ((kept && sizes[v] >= minpts) ? (1ll << 32) : 0ll);
}

// k_big_enough keeps the sub-graph vertices whose running count of s >= minpts is <= k (a prefix)
__global__ void __launch_bounds__(SB_THREADS)
sb_number_kernel(const int* __restrict__ inv, const int* __restrict__ level, const long long* __restrict__ scan,
                 int64_t n, int64_t cut, int* __restrict__ new_index, int* __restrict__ out) {
    SPG_PDL_ENTRY();
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int v = inv[j];
    const long long c = scan[j];
    const int sub = (int)(c & 0xffffffffll);
    const bool keep = level[v] != kUnseen && (cut <= 0 || (c >> 32) <= cut);
    new_index[v] = keep ? sub - 1 : -1;
    if (keep) {
        out[2 + sub - 1] = v;
        atomicMax(out, sub);
    }
}

__global__ void __launch_bounds__(SB_THREADS)
sb_edge_flags_kernel(const int* __restrict__ src, const int* __restrict__ tgt, int64_t n_edges,
                     const int* __restrict__ new_index, int* __restrict__ flags) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e > n_edges) return;
    flags[e] = e < n_edges && new_index[src[e]] >= 0 && new_index[tgt[e]] >= 0;
}

__global__ void sb_edge_count_kernel(const int* __restrict__ edge_pos, int64_t n_edges, int* __restrict__ out) {
    SPG_PDL_ENTRY();
    out[1] = edge_pos[n_edges];
}

__global__ void __launch_bounds__(SB_THREADS)
sb_compact_kernel(const int* __restrict__ src, const int* __restrict__ tgt, int64_t n_edges,
                  const int* __restrict__ new_index, const int* __restrict__ edge_pos, int64_t n_kept,
                  int* __restrict__ keys, int* __restrict__ vals, int64_t* __restrict__ degs) {
    SPG_PDL_ENTRY();
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_kept) degs[e] = 0;
    if (e >= n_edges || edge_pos[e + 1] == edge_pos[e]) return;
    keys[edge_pos[e]] = new_index[tgt[e]];
    vals[edge_pos[e]] = (int)e;
}

// elements [0, kE * F): edge-feature rows; [kE * F, + n_kept * T): target rows; thread i < kE also writes
// edge i's collated (source, target) and counts its target's in-degree
__global__ void __launch_bounds__(SB_THREADS)
sb_gather_kernel(const int* __restrict__ src, const int* __restrict__ new_index, const int* __restrict__ keys,
                 const int* __restrict__ vals, int64_t n_kept_edges, int64_t vertex_offset,
                 const float* __restrict__ feats, int64_t n_feats, const int* __restrict__ kept,
                 int64_t n_kept, const int64_t* __restrict__ targets, int64_t n_target_cols,
                 int64_t* __restrict__ idxn_out, int64_t* __restrict__ tgt_out, int64_t* __restrict__ degs_out,
                 float* __restrict__ feats_out, int64_t* __restrict__ targets_out) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_kept_edges) {
        const int t = keys[i];
        idxn_out[i] = vertex_offset + new_index[src[vals[i]]];
        tgt_out[i] = vertex_offset + t;
        atomicAdd(reinterpret_cast<unsigned long long*>(degs_out + t), 1ull);
    }
    const int64_t nf = n_kept_edges * n_feats;
    if (i < nf) {
        const int64_t r = i / n_feats;
        feats_out[i] = __ldg(feats + (int64_t)vals[r] * n_feats + (i - r * n_feats));
    } else if (i < nf + n_kept * n_target_cols) {
        const int64_t k = i - nf, r = k / n_target_cols;
        targets_out[k] = __ldg(targets + (int64_t)kept[r] * n_target_cols + (k - r * n_target_cols));
    }
}

static int key_bits(int64_t n) {
    int b = 1;
    while (b < 31 && (1ll << b) < n) ++b;
    return b;
}

struct SelectWs {
    int *inv, *level, *flags;
    long long *packed, *scan;
    CubRegion cub;
    size_t bytes;
};

static int select_layout(int64_t n, int64_t n_edges, void* base, SelectWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::InclusiveSum, (const long long*)nullptr, (long long*)nullptr, (int)n);
    SPG_CUB_BYTES(cub_bytes, cub::DeviceScan::ExclusiveSum, (const int*)nullptr, (int*)nullptr, (int)n_edges + 1);
    Planner p(base);
    w->inv = p.take<int>(n);
    w->level = p.take<int>(n);
    w->flags = p.take<int>(n_edges + 1);
    w->packed = p.take<long long>(n);
    w->scan = p.take<long long>(n);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

struct EdgesWs {
    int *keys, *vals, *keys_sorted, *vals_sorted;
    CubRegion cub;
    size_t bytes;
};

static int edges_layout(int64_t n_kept, int64_t n_kept_edges, void* base, EdgesWs* w) {
    size_t cub_bytes = 0;
    SPG_CUB_BYTES(cub_bytes, cub::DeviceRadixSort::SortPairs, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                  (int*)nullptr, (int)n_kept_edges, 0, key_bits(n_kept));
    Planner p(base);
    w->keys = p.take<int>(n_kept_edges);
    w->vals = p.take<int>(n_kept_edges);
    w->keys_sorted = p.take<int>(n_kept_edges);
    w->vals_sorted = p.take<int>(n_kept_edges);
    w->cub = p.cub(cub_bytes);
    w->bytes = p.bytes;
    return SPG_OK;
}

static unsigned blocks(int64_t n) { return (unsigned)ceil_div64(n > 0 ? n : 1, SB_THREADS); }

}  // namespace spg

using namespace spg;

extern "C" {

int spg_batch_select_workspace(int64_t n_ver, int64_t n_edges, int64_t* bytes) {
    if (!bytes || n_ver < 0 || n_edges < 0) return SPG_E_BADARG;
    if (too_big(n_ver) || too_big(n_edges + 1)) return SPG_E_UNSUPPORTED;
    SelectWs w;
    const int rc = select_layout(n_ver, n_edges, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_batch_select(const int32_t* src, const int32_t* tgt, int64_t n_ver, int64_t n_edges,
                     const int32_t* tgt_rowptr, const int32_t* in_src, const int32_t* src_rowptr,
                     const int32_t* src_perm, const int32_t* edge_tgt, const int64_t* sizes, const int32_t* perm,
                     const int32_t* centres, int64_t n_centres, int order, int64_t minpts, int64_t cut,
                     int32_t* new_index, int32_t* edge_pos, int32_t* out, void* workspace, int64_t workspace_bytes,
                     spg_stream_t stream) {
    if (n_ver < 0 || n_edges < 0 || n_centres < 0 || order < 0) return SPG_E_BADARG;
    if (too_big(n_ver) || too_big(n_edges + 1)) return SPG_E_UNSUPPORTED;
    if (!tgt_rowptr || !src_rowptr || !new_index || !edge_pos || !out || (n_ver > 0 && !sizes)) return SPG_E_BADARG;
    if (n_edges > 0 && (!src || !tgt || !in_src || !src_perm || !edge_tgt)) return SPG_E_BADARG;
    if (centres == nullptr && n_centres > 0) return SPG_E_BADARG;
    SelectWs w;
    int rc = select_layout(n_ver, n_edges, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int all = centres == nullptr;
    SPG_LAUNCH(K_SB_SELECT, s, sb_init_kernel, blocks(n_ver > 2 ? n_ver : 2), SB_THREADS, 0, perm, n_ver, all, w.inv,
               w.level, out);
    if (!all) {
        if (n_centres > 0)
            SPG_LAUNCH(K_SB_SELECT, s, sb_centres_kernel, blocks(n_centres), SB_THREADS, 0, centres, n_centres,
                       (const int*)w.inv, w.level);
        for (int l = 0; l < order; ++l)
            SPG_LAUNCH(K_SB_SELECT, s, sb_bfs_kernel, blocks(n_ver), SB_THREADS, 0, tgt_rowptr, in_src, src_rowptr,
                       src_perm, edge_tgt, n_ver, l, w.level);
    }
    if (n_ver > 0) {
        SPG_LAUNCH(K_SB_SELECT, s, sb_flags_kernel, blocks(n_ver), SB_THREADS, 0, (const int*)w.inv,
                   (const int*)w.level, sizes, n_ver, minpts, w.packed);
        SPG_CUB(w.cub, cub::DeviceScan::InclusiveSum, (const long long*)w.packed, w.scan, (int)n_ver, s);
        SPG_LAUNCH(K_SB_SELECT, s, sb_number_kernel, blocks(n_ver), SB_THREADS, 0, (const int*)w.inv,
                   (const int*)w.level, (const long long*)w.scan, n_ver, cut, new_index, out);
    }
    SPG_LAUNCH(K_SB_SELECT, s, sb_edge_flags_kernel, blocks(n_edges + 1), SB_THREADS, 0, src, tgt, n_edges,
               (const int*)new_index, w.flags);
    SPG_CUB(w.cub, cub::DeviceScan::ExclusiveSum, (const int*)w.flags, edge_pos, (int)n_edges + 1, s);
    SPG_LAUNCH(K_SB_SELECT, s, sb_edge_count_kernel, 1, 1, 0, (const int*)edge_pos, n_edges, out);
    return launch_status();
}

int spg_batch_edges_workspace(int64_t n_kept, int64_t n_kept_edges, int64_t* bytes) {
    if (!bytes || n_kept < 0 || n_kept_edges < 0) return SPG_E_BADARG;
    if (too_big(n_kept) || too_big(n_kept_edges)) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    const int rc = edges_layout(n_kept, n_kept_edges, nullptr, &w);
    if (rc == SPG_OK) *bytes = (int64_t)w.bytes;
    return rc;
}

int spg_batch_edges(const int32_t* src, const int32_t* tgt, int64_t n_edges, const int32_t* new_index,
                    const int32_t* edge_pos, const int32_t* kept, int64_t n_kept, int64_t n_kept_edges,
                    int64_t vertex_offset, const float* edge_feats, int64_t n_feats, const int64_t* targets,
                    int64_t n_target_cols, int64_t* idxn_out, int64_t* tgt_out, int64_t* degs_out,
                    float* feats_out, int64_t* targets_out, void* workspace, int64_t workspace_bytes,
                    spg_stream_t stream) {
    if (n_edges < 0 || n_kept < 0 || n_kept_edges < 0 || n_kept_edges > n_edges || n_feats < 0 ||
        n_target_cols < 0 || vertex_offset < 0)
        return SPG_E_BADARG;
    if (too_big(n_kept) || too_big(n_edges + 1)) return SPG_E_UNSUPPORTED;
    if (n_kept_edges > 0 && (!src || !tgt || !new_index || !edge_pos || !idxn_out || !tgt_out || !degs_out ||
                             (n_feats > 0 && (!edge_feats || !feats_out))))
        return SPG_E_BADARG;
    if (n_kept > 0 && (!degs_out || (n_target_cols > 0 && (!kept || !targets || !targets_out)))) return SPG_E_BADARG;
    if ((n_kept_edges * n_feats + n_kept * n_target_cols) >= (1ll << 40)) return SPG_E_UNSUPPORTED;
    EdgesWs w;
    int rc = edges_layout(n_kept, n_kept_edges, workspace, &w);
    if (rc == SPG_OK) rc = ws_check(workspace, workspace_bytes, w.bytes);
    if (rc != SPG_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SPG_LAUNCH(K_SB_EDGES, s, sb_compact_kernel, blocks(n_edges > n_kept ? n_edges : n_kept), SB_THREADS, 0, src,
               tgt, n_edges, new_index, edge_pos, n_kept, w.keys, w.vals, degs_out);
    if (n_kept_edges > 0)
        SPG_CUB(w.cub, cub::DeviceRadixSort::SortPairs, (const int*)w.keys, w.keys_sorted, (const int*)w.vals,
                w.vals_sorted, (int)n_kept_edges, 0, key_bits(n_kept), s);
    const int64_t n_elems = n_kept_edges * n_feats + n_kept * n_target_cols;
    const int64_t n_threads = n_elems > n_kept_edges ? n_elems : n_kept_edges;
    SPG_LAUNCH(K_SB_EDGES, s, sb_gather_kernel, blocks(n_threads), SB_THREADS, 0, src, new_index,
               (const int*)w.keys_sorted, (const int*)w.vals_sorted, n_kept_edges, vertex_offset, edge_feats, n_feats,
               kept, n_kept, targets, n_target_cols, idxn_out, tgt_out, degs_out, feats_out, targets_out);
    return launch_status();
}

}  // extern "C"
