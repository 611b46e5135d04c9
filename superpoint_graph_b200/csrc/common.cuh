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
    K_DROPOUT_RNG_NEXT,
    K_DROPOUT_FWD,
    K_DROPOUT_MASK,
    K_DROPOUT_BWD_REDUCE,
    K_DROPOUT_BWD_REDUCE_FINAL,
    K_DROPOUT_BWD_APPLY,
    K_CRF_FWD,
    K_CRF_BWD,
    K_CRF_SOFTMAX,
    K_LSTM_FWD,
    K_LSTM_BWD,
    K_RNN_LSTM_FWD,
    K_RNN_LSTM_BWD,
    K_GN_FWD,
    K_GN_BWD,
    K_GN_BWD_FINAL,
    K_LP_INCIDENCE,
    K_LP_DIST_FWD,
    K_LP_DIST_BWD,
    K_LP_LOSS_FWD,
    K_LP_LOSS_BWD,
    K_LP_CC,
    K_LP_XPART,
    K_LP_SEAL,
    K_LP_WEIGHTS,
    K_LP_RELAX,
    K_LP_METRICS,
    K_LP_AUGMENT,
    K_LP_SUBGRAPH,
    K_LP_LOCAL_CLOUDS,
    K_GEO_BOUNDS,
    K_GEO_GRID,
    K_GEO_KNN,
    K_GEO_GEOF,
    K_SP_SCAN,
    K_SP_SORT_KEYS,
    K_SP_POINTS,
    K_SP_TETS,
    K_SP_PAIRS,
    K_SP_EDGES,
    K_PRUNE_BOUNDS,
    K_PRUNE_KEYS,
    K_PRUNE_ROWS,
    K_PRUNE_REDUCE,
    K_CP_GRAPH,
    K_CP_MEMBERS,
    K_CP_KMEANS,
    K_CP_CENTERS,
    K_CP_CAPACITIES,
    K_CP_MAXFLOW,
    K_CP_COLOUR,
    K_CP_ACTIVATE,
    K_CP_SPLIT,
    K_CP_MERGE,
    K_CP_ENERGY,
    K_DT_SETUP,
    K_DT_INIT,
    K_DT_NOMINATE,
    K_DT_GROW,
    K_DT_CHECK,
    K_DT_COMMIT,
    K_DT_RELOCATE,
    K_DT_OUTPUT,
    K_ST_VOR,
    K_ST_CC,
    K_ST_LABELS,
    K_ST_SELECT,
    K_ST_POINTS,
    K_SB_SELECT,
    K_SB_EDGES,
    K_SB_DRAW,
    K_SB_PERM,
    K_SB_FLAGS,
    K_SB_CLOUD_DRAW,
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

// Order-preserving map float -> uint32 and its inverse: unsigned order of the keys is the order of the floats
// (-0 below +0), so integer min / max / sorts of keys are min / max / sorts of the floats.
__device__ __forceinline__ unsigned float_key(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_unkey(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ---- BatchNorm/ReLU elements shared by the dense, max-pool and tensor-core kernels

// Gradient through relu(y*sc + sh): g where the pre-activation is > 0, else 0 (NaN included).
__device__ __forceinline__ float relu_bwd(float g, float y, float sc, float sh) {
    return fmaf(y, sc, sh) > 0.f ? g : 0.f;
}

// BatchNorm backward of one element: sc*(g - s1/M - xhat*s2/M), xhat = (y - mu)*rstd, m1 = s1/M, m2 = s2/M.
__device__ __forceinline__ float bn_bwd(float g, float y, float sc, float mu, float rstd, float m1, float m2) {
    return sc * (g - m1 - (y - mu) * rstd * m2);
}

// BatchNorm fold of a column from its batch statistics: scale = gamma/sqrt(var+eps), shift =
// beta - mean*scale, running = (1-momentum)*running + momentum*{mean, var*unbias}, nbt += 1.
// gamma, beta, rmean, rvar and nbt may be NULL; `enabled` says whether a merge folds at all.
struct FoldArgs {
    const float *gamma, *beta;
    float *scale, *shift, *rmean, *rvar;
    long long* nbt;
    float eps, momentum, unbias;
    int enabled;
};

// unbias = M/(M-1) for a batch of M rows; enabled if scale != NULL
inline FoldArgs fold_args(const float* gamma, const float* beta, float eps, float* scale, float* shift,
                          float* rmean, float* rvar, int64_t* nbt, float momentum, int64_t M) {
    FoldArgs f;
    f.gamma = gamma; f.beta = beta; f.scale = scale; f.shift = shift;
    f.rmean = rmean; f.rvar = rvar; f.nbt = (long long*)nbt;
    f.eps = eps; f.momentum = momentum;
    f.unbias = M > 1 ? (float)((double)M / (double)(M - 1)) : 1.f;
    f.enabled = scale != nullptr;
    return f;
}

__device__ __forceinline__ void bn_fold_col(const FoldArgs& f, int c, float mu, float var) {
    const float rstd = 1.f / sqrtf(var + f.eps);
    const float sc = (f.gamma ? f.gamma[c] : 1.f) * rstd;
    f.scale[c] = sc;
    f.shift[c] = (f.beta ? f.beta[c] : 0.f) - mu * sc;
    if (f.rmean) f.rmean[c] = (1.f - f.momentum) * f.rmean[c] + f.momentum * mu;
    if (f.rvar) f.rvar[c] = (1.f - f.momentum) * f.rvar[c] + f.momentum * var * f.unbias;
    if (c == 0 && f.nbt) f.nbt[0] += 1;
}

// out[c] = sum_k ws[k*C + c] for k < chunks (fp64, fixed order; bn_act.cu), counted as kernel `kid`.
int colsum_merge(int kid, const float* ws, int64_t chunks, int C, float* out, cudaStream_t s);

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
