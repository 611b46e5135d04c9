// Weight images of the wgmma GEMMs (tc_gemm2.cu): pre-split (tf32 hi / lo) and pre-swizzled copies
// of a weight matrix in exactly the shared-memory layout the MMA reads, so that the resident-weight
// load of the GEMM is a plain TMA box copy.
//
// Reference semantics: the weights of the nn.Conv1d(k=1) / nn.Linear layers of
// learning/pointnet.py:27-37,83-96 (forward: W, data gradient: W^T).
#include "common.cuh"
#include "tc_common.cuh"

namespace spg {

constexpr int TC_KC = 32;       // floats per K chunk (128 B swizzle row)

// Weight image: for every K chunk kc: [hi: N rows x 128 B][lo: N rows x 128 B], each block laid
// out exactly as the shared-memory tile (SWIZZLE_128B).  transpose=0: B[n][k] = W[n*ldw + k];
// transpose=1: B[n][k] = W[k*ldw + n] (the data-gradient GEMM consumes W^T).
__global__ void tc_pack_weights_kernel(const float* __restrict__ W, int64_t ldw, int transpose,
                                       int N, int K, int k_valid, float* __restrict__ img) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * K) return;
    const int n = (int)(i / K), k = (int)(i % K);
    float v = 0.f;  // k >= k_valid: zero padding of the reduction dimension
    if (k < k_valid) v = transpose ? W[(int64_t)k * ldw + n] : W[(int64_t)n * ldw + k];
    const uint32_t hi = to_tf32(v);
    const uint32_t lo = to_tf32(v - __uint_as_float(hi));
    const int kc = k / TC_KC, kk = k % TC_KC;
    const int64_t base = (int64_t)kc * 2 * N * TC_KC;
    const int64_t off = (int64_t)(sw128_off(n, kk >> 2) >> 2) + (kk & 3);
    img[base + off] = __uint_as_float(hi);
    img[base + (int64_t)N * TC_KC + off] = __uint_as_float(lo);
}

// Same image from W[n][k] * row_scale[n]: eval-mode BatchNorm folded into the weights
// (scale = gamma / sqrt(running_var + eps)); consumed by pointnet_fused.cu.
__global__ void tc_pack_weights_scaled_kernel(const float* __restrict__ W, int64_t ldw,
                                              const float* __restrict__ row_scale, int N, int K, int k_valid,
                                              float* __restrict__ img) {
    SPG_PDL_ENTRY();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * K) return;
    const int n = (int)(i / K), k = (int)(i % K);
    float v = 0.f;
    if (k < k_valid) v = W[(int64_t)n * ldw + k] * (row_scale ? row_scale[n] : 1.f);
    const uint32_t hi = to_tf32(v);
    const uint32_t lo = to_tf32(v - __uint_as_float(hi));
    const int kc = k / TC_KC, kk = k % TC_KC;
    const int64_t base = (int64_t)kc * 2 * N * TC_KC;
    const int64_t off = (int64_t)(sw128_off(n, kk >> 2) >> 2) + (kk & 3);
    img[base + off] = __uint_as_float(hi);
    img[base + (int64_t)N * TC_KC + off] = __uint_as_float(lo);
}

// Batched variant: one launch packs every weight matrix of a model (forward images and the
// transposed images of the data-gradient GEMMs).  table[j] = {W, ldw, transpose, N, K, k_valid,
// image, first element index of job j}; a thread finds its job by a linear scan (<= 64 jobs).
__global__ void tc_pack_weights_multi_kernel(const long long* __restrict__ table, int n_jobs,
                                             long long total) {
    SPG_PDL_ENTRY();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int j = 0;
    while (j + 1 < n_jobs && i >= table[(j + 1) * 8 + 7]) ++j;
    const long long* d = table + j * 8;
    const float* W = reinterpret_cast<const float*>(d[0]);
    const long long ldw = d[1];
    const int transpose = (int)d[2], N = (int)d[3], K = (int)d[4], k_valid = (int)d[5];
    float* img = reinterpret_cast<float*>(d[6]);
    const long long e = i - d[7];
    const int n = (int)(e / K), k = (int)(e % K);
    float v = 0.f;
    if (k < k_valid) v = transpose ? W[(long long)k * ldw + n] : W[(long long)n * ldw + k];
    const uint32_t hi = to_tf32(v);
    const uint32_t lo = to_tf32(v - __uint_as_float(hi));
    const int kc = k / TC_KC, kk = k % TC_KC;
    const long long base = (long long)kc * 2 * N * TC_KC;
    const long long off = (long long)(sw128_off(n, kk >> 2) >> 2) + (kk & 3);
    img[base + off] = __uint_as_float(hi);
    img[base + (long long)N * TC_KC + off] = __uint_as_float(lo);
}

}  // namespace spg

using namespace spg;

extern "C" {

int64_t spg_tc_weight_image_floats(int N, int K) { return (int64_t)2 * N * K; }

int spg_tc_pack_weights(const float* W, int64_t ldw, int transpose, int N, int K, int k_valid,
                        float* image, spg_stream_t stream) {
    if (!W || !image || N <= 0 || K <= 0 || k_valid <= 0 || k_valid > K) return SPG_E_BADARG;
    if (K % TC_KC != 0 || N % 8 != 0) return SPG_E_UNSUPPORTED;
    const int64_t total = (int64_t)N * K;
    SPG_LAUNCH(K_TC_PACK, (cudaStream_t)stream, tc_pack_weights_kernel,
               (unsigned)ceil_div64(total, 256), 256, 0, W, ldw, transpose, N, K, k_valid, image);
    return launch_status();
}

int spg_tc_pack_weights_scaled(const float* W, int64_t ldw, const float* row_scale, int N, int K, int k_valid,
                               float* image, spg_stream_t stream) {
    if (!W || !image || N <= 0 || K <= 0 || k_valid <= 0 || k_valid > K) return SPG_E_BADARG;
    if (K % TC_KC != 0 || N % 8 != 0) return SPG_E_UNSUPPORTED;
    const int64_t total = (int64_t)N * K;
    SPG_LAUNCH(K_TC_PACK, (cudaStream_t)stream, tc_pack_weights_scaled_kernel,
               (unsigned)ceil_div64(total, 256), 256, 0, W, ldw, row_scale, N, K, k_valid, image);
    return launch_status();
}

int spg_tc_pack_weights_multi(const int64_t* table, int n_jobs, int64_t total, spg_stream_t stream) {
    if (!table || n_jobs <= 0 || n_jobs > 64 || total <= 0) return SPG_E_BADARG;
    SPG_LAUNCH(K_TC_PACK, (cudaStream_t)stream, tc_pack_weights_multi_kernel,
               (unsigned)ceil_div64(total, 256), 256, 0, (const long long*)table, n_jobs,
               (long long)total);
    return launch_status();
}

}  // extern "C"
