// Connected components by union-find, shared by the learned partition's crosspartition weights (partition.cu) and
// connected_comp (structure.cu).  Parents only ever point to smaller vertices, so every root is its component's
// smallest vertex and components are numbered by it, in vertex order: what boost's connected_components gives
// libply_c's connected_comp (partition/ply_c/connected_components.cpp:31).  Hooks are integer CAS, so the result
// does not depend on the order in which edges are processed.
#pragma once
#include "common.cuh"

namespace spg {

constexpr int CC_THREADS = 256;

__device__ __forceinline__ int cc_find(int* p, int x) {
    volatile int* vp = p;
    int cur = vp[x];
    if (cur != x) {
        int prev = x, next;
        while (cur > (next = vp[cur])) {  // path halving; parents point to smaller vertices, roots to themselves
            vp[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

// joins the components of s and t: the larger root is hooked under the smaller one
__device__ __forceinline__ void cc_union(int* parent, int s, int t) {
    int ru = cc_find(parent, s), rv = cc_find(parent, t);
    while (ru != rv) {
        const int hi = ru > rv ? ru : rv, lo = ru > rv ? rv : ru;
        if (atomicCAS(parent + hi, hi, lo) == hi) break;
        ru = cc_find(parent, ru);
        rv = cc_find(parent, rv);
    }
}

// parent[v] = root of v, is_root[v] = (root == v)
static __global__ void __launch_bounds__(CC_THREADS)
cc_flatten_kernel(int* __restrict__ parent, int64_t n_ver, int* __restrict__ is_root) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_ver) return;
    const int r = cc_find(parent, (int)v);
    parent[v] = r;
    is_root[v] = r == (int)v;
}

// components numbered by their smallest vertex (root_rank: exclusive scan of is_root); sizes by integer atomics
template <class C>
__global__ void __launch_bounds__(CC_THREADS)
cc_label_kernel(const int* __restrict__ parent, const int* __restrict__ root_rank, const int* __restrict__ is_root,
                int64_t n_ver, C* __restrict__ in_comp, int* __restrict__ comp_size, C* __restrict__ n_comp) {
    SPG_PDL_ENTRY();
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_ver) return;
    int r = parent[v];
    while (parent[r] != r) r = parent[r];
    const int c = root_rank[r];
    in_comp[v] = c;
    atomicAdd(comp_size + c, 1);
    if (v == n_ver - 1) *n_comp = root_rank[v] + is_root[v];
}

}  // namespace spg
