// Training-mode dropout of a fused Linear/Conv1d [+BatchNorm] [+ReLU] layer (ref: learning/pointnet.py:109-110,
// learning/graphnet.py:54-55: nn.Dropout after the activation).
//
// The mask is a pure function of (seed, ctr, i) with i = m*C + c the logical index of element (m, c) of the
// [M, C] activation: Philox4x32-10 with key (seed_lo, seed_hi) and counter (i>>2 low word, i>>34, ctr_lo,
// ctr_hi), word i & 3; kept iff word >= floor(p * 2^32), kept elements scaled by 1/(1-p), p >= 1 drops all.
// It depends on neither grid size, leading dimension nor launch order, so the backward regenerates it instead
// of storing it.  (seed, ctr) live in device memory: spg_dropout_rng_next copies the device generator state
// into a per-site slot and advances the counter, every other kernel reads the slot — nothing about the stream
// position is baked into launch parameters, so replays of a captured CUDA graph draw fresh masks.
// The masked forward and backward are the DROP instantiations of the activation kernels
// (bn_act.cu); this file holds the slot kernel and the mask export.
#include "common.cuh"
#include "philox.cuh"

namespace spg {

__global__ void dropout_rng_next_kernel(int64_t* state, int64_t* slot, int64_t key_xor) {
    SPG_PDL_ENTRY();
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        slot[0] = state[0] ^ key_xor;
        slot[1] = state[1];
        state[1] = state[1] + 1;
    }
}

__global__ void __launch_bounds__(256)
dropout_mask_kernel(const int64_t* __restrict__ slot, float p, int64_t M, int C, uint8_t* __restrict__ mask) {
    SPG_PDL_ENTRY();
    const DropParams d = drop_params(slot, p);
    const int64_t n = M * C, groups = (n + 3) >> 2;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (int64_t)gridDim.x * blockDim.x) {
        const Philox4 w = dropout_words(d.seed, d.ctr, (uint64_t)q);
        for (int j = 0; j < 4 && (q << 2) + j < n; ++j) mask[(q << 2) + j] = kept(d, w.v[j]) ? 1 : 0;
    }
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_dropout_rng_next(int64_t* state, int64_t* slot, int64_t key_xor, spg_stream_t stream) {
    if (!state || !slot) return SPG_E_BADARG;
    SPG_LAUNCH(K_DROPOUT_RNG_NEXT, (cudaStream_t)stream, dropout_rng_next_kernel, 1, 32, 0, state, slot, key_xor);
    return launch_status();
}

int spg_dropout_mask(const int64_t* slot, float p, int64_t M, int C, uint8_t* mask, spg_stream_t stream) {
    if (M < 0 || C <= 0 || !(p >= 0.f)) return SPG_E_BADARG;
    if (M == 0) return SPG_OK;
    if (!slot || !mask) return SPG_E_BADARG;
    int64_t grid = ceil_div64(ceil_div64(M * C, 4), 256);
    if (grid > 16 * kNumSMs) grid = 16 * kNumSMs;
    SPG_LAUNCH(K_DROPOUT_MASK, (cudaStream_t)stream, dropout_mask_kernel, (unsigned)grid, 256, 0, slot, p, M, C,
               mask);
    return launch_status();
}

}  // extern "C"
