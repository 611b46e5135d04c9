// Shared helpers for libspg_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/spg_b200.h"

namespace spg {

// Kernel ids for launch accounting (order must match kKernelNames in runtime.cu).
enum KernelId {
    K_ECC_VV_FWD = 0,
    K_ECC_MAT_FWD,
    K_ECC_GEN_FWD,
    K_ECC_VV_BWD_W,
    K_ECC_MAT_BWD_W,
    K_ECC_GEN_BWD_W,
    K_ECC_VV_BWD_X,
    K_ECC_MAT_BWD_X,
    K_ECC_GEN_BWD_X,
    K_GRU_FWD,
    K_GRU_BWD,
    K_GEMM,
    K_GEMM_SPLITK_REDUCE,
    K_COLSTATS_PARTIAL,
    K_COLSTATS_FINAL,
    K_BN_FOLD,
    K_AFFINE_ACT,
    K_COLSUM_PARTIAL,
    K_COLSUM_FINAL,
    K_ACT_BWD_REDUCE,
    K_ACT_BWD_REDUCE_FINAL,
    K_ACT_BWD_APPLY,
    K_CLOUD_ROWS,
    K_SEGMAX_FWD,
    K_SEGMAX_BWD,
    K_STN_APPLY_BWD,
    K_ROWS_SCATTER,
    K_ROWS_GATHER,
    K_CE_LOSS,
    K_CE_LOSS_FINAL,
    K_CLAMP_ADAM,
    K_TC_GEMM,
    K_TC_PACK,
    K_TC_DW,
    K_RNN_FWD,
    K_RNN_BWD,
    K_CLOUD_BUILD,
    K_CONFUSION,
    K_TC_MERGE,
    K_POINTNET_FUSED,
    K_GRAPH_BUILD,
    K_COUNT
};

// Brackets one launch with CUDA events when profiling is enabled; always counts it.
struct LaunchScope {
    int kid;
    cudaStream_t stream;
    int slot;
    LaunchScope(int kernel_id, cudaStream_t s);
    ~LaunchScope();
};

// cudaGetLastError() -> return code of the C-ABI call.
inline int launch_status() { return (int)cudaGetLastError(); }

constexpr int kNumSMs = 132;  // H100 SXM

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float4 ld_stream4(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream4(float4* p, float4 v) { __stcs(p, v); }

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// 128-bit vectorised variants (dense_vec.cu); return false if the shape/alignment does not fit.
bool vec_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                        const float* scale, const float* shift, const float* mean,
                        const float* var, float eps, int relu, float* s1, float* s2, float* ws,
                        int64_t M, int C, cudaStream_t s, int* rc);
bool vec_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* ws,
                cudaStream_t s, int* rc);
bool vec_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, int has_bn, const float* s1,
                       const float* s2, float* dY, int64_t lddy, int64_t M, int C,
                       cudaStream_t s, int* rc);
bool vec_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                    float* out, int64_t ldo, int64_t M, int C, cudaStream_t s, int* rc);

}  // namespace spg

// Programmatic dependent launch (sm_90+): every kernel of this library starts with pdl_entry() — wait until
// the kernels it depends on have completed and flushed, then allow the NEXT kernel of the stream to be
// scheduled — and is launched with programmaticStreamSerialization, so that the launch latency, block
// scheduling and pre-wait set-up (barrier init, descriptor prefetch) of kernel n+1 overlap kernel n.
// The trigger comes AFTER the wait on purpose: at most one dependent grid is resident and waiting.
// spg_set_pdl(0) switches the attribute off (plain stream order; the device instructions are then no-ops).
#define SPG_PDL_ENTRY()                                          \
    do {                                                         \
        asm volatile("griddepcontrol.wait;" ::: "memory");       \
        asm volatile("griddepcontrol.launch_dependents;" :::);   \
    } while (0)

namespace spg {
bool pdl_enabled(int kernel_id);

template <typename... KArgs, typename... Args>
inline void launch_kernel(int kid, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                          Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl_enabled(kid) ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
}  // namespace spg

#define SPG_LAUNCH(kid, stream_, kernel, grid, block, smem, ...)                                  \
    do {                                                                                           \
        ::spg::LaunchScope _scope((kid), (stream_));                                               \
        ::spg::launch_kernel((kid), kernel, dim3(grid), dim3(block), (size_t)(smem), (stream_), __VA_ARGS__); \
    } while (0)
