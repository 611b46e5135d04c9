// Fused recurrent cells with an input gate and an affine-free layer norm of both gate
// pre-activations: GRUCellEx and LSTMCellEx, forward and backward, one kernel each, plus the
// persistent R x {ECC, cell} recurrence.
//
// Reference semantics: learning/modules.py:205-251 (GRUCellEx) and :262-308 (LSTMCellEx).  There a
// cell is ~20 torch ops per call (3 GEMMs, 2 InstanceNorm1d, chunk/sigmoid/tanh/elementwise); here
// the three weight matrices ((2G+1)*H*H floats for G gates: 28 KB for the GRU, 37 KB for the LSTM
// at H=32) live in shared memory, a warp owns RW rows at a time and every intermediate stays on chip.
// 14 kFLOP and 384 B per GRU row: latency/L2-bound, so no tensor cores.
//
// Everything but the pointwise gate formulas is shared by the two cells: the weight load, the input
// gate, the two row GEMVs, the layer-norm statistics and their backward, the d_x'/d_h/d_q GEMVs and
// the persistent recurrence.  What differs is a compile-time cell policy (GruCell, LstmCell): the
// gate count G, where the biases enter, the pointwise forward and backward, and where the backward
// keeps the gate gradients between its pointwise stage and the layer-norm backward.
#include "ecc_rows.cuh"

namespace spg {

constexpr int kCellWarps = 8;  // warps per block (both cells)

// The LSTM's cell state c, which the GRU does not have (all members are null for the GRU).
struct CellState {
    const float* c;    // c_r [n,H]
    float* c_out;      // forward: c_{r+1}; backward: dL/dc_r (may alias g_c: read before written)
    const float* g_c;  // backward: dL/dc_{r+1}; null = 0 (a state that leaves the module unused)
};

// shared-memory layout (floats), G = Cell::kGates:
//   Wig_t [H][H+1]    Wig_t[k*(H+1)+c]   = ig_weight[c][k]
//   Wih_t [H][GH+1]   Wih_t[k*(GH+1)+j]  = weight_ih[j][k]
//   Whh_t [H][GH+1]
//   per warp scratch: hrow[RW][H], xrow[RW][H], srow[RW][H], gi[RW][GH], gh[RW][GH]
//                     and, if Cell::kDyScratch, dy[RW][GH]
template <class Cell>
__host__ __device__ inline int cell_weight_floats(int H) {
    return H * (H + 1) + 2 * H * (Cell::kGates * H + 1);
}
template <class Cell>
__host__ __device__ inline int cell_scratch_floats(int H, int rw) {
    return rw * (3 * H + (2 + Cell::kDyScratch) * Cell::kGates * H);
}

template <class Cell>
__device__ __forceinline__ void cell_load_weights(float* sm, const float* __restrict__ w_ih,
                                                  const float* __restrict__ w_hh,
                                                  const float* __restrict__ w_ig, int H,
                                                  int ingate) {
    const int GH = Cell::kGates * H;
    float* Wig_t = sm;
    float* Wih_t = Wig_t + H * (H + 1);
    float* Whh_t = Wih_t + H * (GH + 1);
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < GH * H; i += nt) {
        const int j = i / H, k = i % H;
        Wih_t[k * (GH + 1) + j] = w_ih[i];
        Whh_t[k * (GH + 1) + j] = w_hh[i];
    }
    if (ingate) {
        for (int i = tid; i < H * H; i += nt) {
            const int c = i / H, k = i % H;
            Wig_t[k * (H + 1) + c] = w_ig[i];
        }
    }
}

// Recomputes everything up to the normalised gate inputs for RW rows.
// On return (per row i): hrow = h, xrow = gated input x', srow = sigmoid(q) (or 1),
// gi/gh = raw (pre-norm) gate inputs, biases included where the cell adds them before the norm,
// stats = {mean_i, rstd_i, mean_h, rstd_h}.
template <class Cell, int kRW>
__device__ __forceinline__ void cell_rows_forward(const float* sm, float* scratch, int H, int flags,
                                                  const float* x, const float* h,
                                                  const float* __restrict__ b_ih,
                                                  const float* __restrict__ b_hh,
                                                  const float* __restrict__ b_ig, int64_t row0,
                                                  int64_t n_rows, int lane, float stats[kRW][4]) {
    const int GH = Cell::kGates * H;
    const float* Wig_t = sm;
    const float* Wih_t = Wig_t + H * (H + 1);
    const float* Whh_t = Wih_t + H * (GH + 1);
    float* hrow = scratch;
    float* xrow = hrow + kRW * H;
    float* srow = xrow + kRW * H;
    float* gi = srow + kRW * H;
    float* gh = gi + kRW * GH;

    for (int i = 0; i < kRW; ++i) {
        const int64_t row = row0 + i;
        for (int c = lane; c < H; c += 32) {
            hrow[i * H + c] = row < n_rows ? h[row * H + c] : 0.f;
            xrow[i * H + c] = row < n_rows ? x[row * H + c] : 0.f;
        }
    }
    __syncwarp();
    if (flags & SPG_GRU_INGATE) {
        for (int c = lane; c < H; c += 32) {
            float acc[kRW];
#pragma unroll
            for (int i = 0; i < kRW; ++i) acc[i] = b_ig[c];
            for (int k = 0; k < H; ++k) {
                const float wv = Wig_t[k * (H + 1) + c];
#pragma unroll
                for (int i = 0; i < kRW; ++i) acc[i] = fmaf(wv, hrow[i * H + k], acc[i]);
            }
#pragma unroll
            for (int i = 0; i < kRW; ++i) {
                const float sg = sigmoidf_(acc[i]);
                srow[i * H + c] = sg;
                xrow[i * H + c] *= sg;  // only this lane touches xrow[.][c]
            }
        }
    } else {
        for (int c = lane; c < H; c += 32)
#pragma unroll
            for (int i = 0; i < kRW; ++i) srow[i * H + c] = 1.f;
    }
    __syncwarp();
    const bool pre_bias = Cell::kBiasPreNorm && (flags & SPG_GRU_BIAS);
    for (int j = lane; j < GH; j += 32) {
        const float bi = pre_bias ? b_ih[j] : 0.f, bh = pre_bias ? b_hh[j] : 0.f;
        float ai[kRW], ah[kRW];
#pragma unroll
        for (int i = 0; i < kRW; ++i) {
            ai[i] = bi;
            ah[i] = bh;
        }
        for (int k = 0; k < H; ++k) {
            const float wi = Wih_t[k * (GH + 1) + j];
            const float wh = Whh_t[k * (GH + 1) + j];
#pragma unroll
            for (int i = 0; i < kRW; ++i) {
                ai[i] = fmaf(wi, xrow[i * H + k], ai[i]);
                ah[i] = fmaf(wh, hrow[i * H + k], ah[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < kRW; ++i) {
            gi[i * GH + j] = ai[i];
            gh[i * GH + j] = ah[i];
        }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kRW; ++i) {
        if (flags & SPG_GRU_LAYERNORM) {
            float si = 0.f, sh = 0.f;
            for (int j = lane; j < GH; j += 32) {
                si += gi[i * GH + j];
                sh += gh[i * GH + j];
            }
            si = warp_sum(si) / (float)GH;
            sh = warp_sum(sh) / (float)GH;
            float vi = 0.f, vh = 0.f;
            for (int j = lane; j < GH; j += 32) {
                const float di = gi[i * GH + j] - si, dh = gh[i * GH + j] - sh;
                vi = fmaf(di, di, vi);
                vh = fmaf(dh, dh, vh);
            }
            vi = warp_sum(vi) / (float)GH;
            vh = warp_sum(vh) / (float)GH;
            stats[i][0] = si;
            stats[i][1] = rsqrtf(vi + 1e-5f);
            stats[i][2] = sh;
            stats[i][3] = rsqrtf(vh + 1e-5f);
        } else {
            stats[i][0] = 0.f;
            stats[i][1] = 1.f;
            stats[i][2] = 0.f;
            stats[i][3] = 1.f;
        }
    }
}

// ------------------------------------------------------------------ cell policies
// Each policy provides, for the RW rows whose gate inputs cell_rows_forward left in `scratch`:
//   emit: the new state (hy, and c_{r+1} for the LSTM);
//   grad: from dL/dhy (and dL/dc_{r+1}), the gradient w.r.t. each normalised gate input (dy, kept
//         where dy_row points), the direct part of dL/dh, the cell-state gradient; it also replaces
//         gi/gh by their normalised values (y-hat) when the layer norm is on;
//   dy_row / dy_i / dy_h: where the layer-norm backward reads dy for the input and hidden side.

// GRUCellEx (ref: learning/modules.py:239-250): biases after the norm; dy lives in dpre_out,
// which doubles as the bias gradients' summands [d_pr, d_pz, d_pn, d_pn*r].
struct GruCell {
    static constexpr int kGates = 3;
    static constexpr bool kBiasPreNorm = false;
    static constexpr int kDyScratch = 0;
    static constexpr int kDpreCols = 4;  // dpre_out [n, 4H]
    // Large row counts always take 4 rows per warp; widths where those do not fit are unsupported.
    static constexpr bool kFewerRowsIfFull = false;

    __device__ static CellState fwd_state(float*, int, size_t) { return CellState{}; }
    __device__ static CellState bwd_state(const float*, float*, int, int, size_t) {
        return CellState{};
    }

    template <int kRW>
    __device__ static __forceinline__ void emit(const float* scratch, int H, int flags,
                                                const float* __restrict__ b_ih,
                                                const float* __restrict__ b_hh, float* hy,
                                                CellState, int64_t row0, int64_t n_rows, int lane,
                                                const float st[kRW][4]) {
        const float* hrow = scratch;
        const float* gi = scratch + 3 * kRW * H;
        const float* gh = gi + kRW * 3 * H;
        const int H3 = 3 * H;
        const bool has_bias = flags & SPG_GRU_BIAS;
        for (int c = lane; c < H; c += 32) {
            const float bir = has_bias ? b_ih[c] : 0.f, biz = has_bias ? b_ih[H + c] : 0.f,
                        bin = has_bias ? b_ih[2 * H + c] : 0.f;
            const float bhr = has_bias ? b_hh[c] : 0.f, bhz = has_bias ? b_hh[H + c] : 0.f,
                        bhn = has_bias ? b_hh[2 * H + c] : 0.f;
#pragma unroll
            for (int i = 0; i < kRW; ++i) {
                const int64_t row = row0 + i;
                if (row >= n_rows) break;
                const float i_r = (gi[i * H3 + c] - st[i][0]) * st[i][1];
                const float i_z = (gi[i * H3 + H + c] - st[i][0]) * st[i][1];
                const float i_n = (gi[i * H3 + 2 * H + c] - st[i][0]) * st[i][1];
                const float h_r = (gh[i * H3 + c] - st[i][2]) * st[i][3];
                const float h_z = (gh[i * H3 + H + c] - st[i][2]) * st[i][3];
                const float h_n = (gh[i * H3 + 2 * H + c] - st[i][2]) * st[i][3];
                const float rg = sigmoidf_(i_r + bir + h_r + bhr);
                const float zg = sigmoidf_(i_z + biz + h_z + bhz);
                const float ng = tanhf(i_n + bin + rg * (h_n + bhn));
                const float hv = hrow[i * H + c];
                hy[row * H + c] = ng + zg * (hv - ng);
            }
        }
        __syncwarp();
    }

    template <int NU, int kRW>
    __device__ static __forceinline__ void grad(const float* hrow, float* gi, float* gh, float*,
                                                int H, int flags, const float* __restrict__ b_ih,
                                                const float* __restrict__ b_hh, const float* gy,
                                                float* dpre_out, CellState, int64_t row0,
                                                int64_t n_rows, int lane, const float st[kRW][4],
                                                float dh_direct[kRW][NU]) {
        const int H3 = 3 * H;
        const bool has_bias = flags & SPG_GRU_BIAS;
        const bool ln = flags & SPG_GRU_LAYERNORM;
#pragma unroll
        for (int i = 0; i < kRW; ++i) {
            const int64_t row = row0 + i;
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const int c = lane + 32 * u;
                if (c >= H) continue;
                const float bir = has_bias ? b_ih[c] : 0.f, biz = has_bias ? b_ih[H + c] : 0.f,
                            bin = has_bias ? b_ih[2 * H + c] : 0.f;
                const float bhr = has_bias ? b_hh[c] : 0.f, bhz = has_bias ? b_hh[H + c] : 0.f,
                            bhn = has_bias ? b_hh[2 * H + c] : 0.f;
                const float i_r = (gi[i * H3 + c] - st[i][0]) * st[i][1];
                const float i_z = (gi[i * H3 + H + c] - st[i][0]) * st[i][1];
                const float i_n = (gi[i * H3 + 2 * H + c] - st[i][0]) * st[i][1];
                const float h_r = (gh[i * H3 + c] - st[i][2]) * st[i][3];
                const float h_z = (gh[i * H3 + H + c] - st[i][2]) * st[i][3];
                const float h_n = (gh[i * H3 + 2 * H + c] - st[i][2]) * st[i][3];
                const float rg = sigmoidf_(i_r + bir + h_r + bhr);
                const float zg = sigmoidf_(i_z + biz + h_z + bhz);
                const float ng = tanhf(i_n + bin + rg * (h_n + bhn));
                const float hv = hrow[i * H + c];
                const float g = row < n_rows ? gy[row * H + c] : 0.f;
                const float d_n = g * (1.f - zg);
                const float d_z = g * (hv - ng);
                dh_direct[i][u] = g * zg;
                const float d_pn = d_n * (1.f - ng * ng);
                const float d_r = d_pn * (h_n + bhn);
                const float d_pz = d_z * zg * (1.f - zg);
                const float d_pr = d_r * rg * (1.f - rg);
                if (row < n_rows) {
                    float* dp = dpre_out + row * 4 * H;
                    dp[c] = d_pr;
                    dp[H + c] = d_pz;
                    dp[2 * H + c] = d_pn;
                    dp[3 * H + c] = d_pn * rg;
                }
                // y-hat replaces the raw gate inputs only after this lane has read all of its own
                // entries (each lane owns columns c, H+c, 2H+c of both arrays)
                gi[i * H3 + c] = ln ? i_r : 0.f;
                gi[i * H3 + H + c] = ln ? i_z : 0.f;
                gi[i * H3 + 2 * H + c] = ln ? i_n : 0.f;
                gh[i * H3 + c] = ln ? h_r : 0.f;
                gh[i * H3 + H + c] = ln ? h_z : 0.f;
                gh[i * H3 + 2 * H + c] = ln ? h_n : 0.f;
            }
        }
    }

    __device__ static __forceinline__ const float* dy_row(const float* dpre_out, const float*,
                                                          int64_t row, bool live, int H) {
        return dpre_out + (live ? row : 0) * 4 * H;
    }
    // the hidden side's n-gate gradient is d_pn * r (the reset gate scales h_n)
    __device__ static __forceinline__ float dy_i(const float* dp, int j, int) { return dp[j]; }
    __device__ static __forceinline__ float dy_h(const float* dp, int j, int H) {
        return j < 2 * H ? dp[j] : dp[j + H];
    }
};

// LSTMCellEx (ref: learning/modules.py:296-307): biases inside the linears, before the norm, so
// d_gi/d_gh are the bias gradients' summands and no dpre is needed.  Gates (i, f, g, o) = chunks
// of gi + gh; dy is the same for both sides and lives in the per-warp scratch.
struct LstmCell {
    static constexpr int kGates = 4;
    static constexpr bool kBiasPreNorm = true;
    static constexpr int kDyScratch = 1;
    static constexpr int kDpreCols = 0;
    // H = 64 leaves room for 1 row per warp next to the 148 KB of weights: take it.
    static constexpr bool kFewerRowsIfFull = true;

    // fused recurrence: the cell states live in cs [R+1,n,H]; the backward carries dL/dc in dc [n,H]
    __device__ static CellState fwd_state(float* cs, int r, size_t plane) {
        return CellState{cs + r * plane, cs + (r + 1) * plane, nullptr};
    }
    __device__ static CellState bwd_state(const float* cs, float* dc, int r, int R, size_t plane) {
        return CellState{cs + r * plane, dc, r == R - 1 ? nullptr : dc};
    }

    template <int kRW>
    __device__ static __forceinline__ void emit(const float* scratch, int H, int, const float*,
                                                const float*, float* hy, CellState cs,
                                                int64_t row0, int64_t n_rows, int lane,
                                                const float st[kRW][4]) {
        const float* gi = scratch + 3 * kRW * H;
        const float* gh = gi + kRW * 4 * H;
        const int H4 = 4 * H;
        for (int c = lane; c < H; c += 32) {
#pragma unroll
            for (int i = 0; i < kRW; ++i) {
                const int64_t row = row0 + i;
                if (row >= n_rows) break;
                float a[4];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    a[q] = (gi[i * H4 + q * H + c] - st[i][0]) * st[i][1] +
                           (gh[i * H4 + q * H + c] - st[i][2]) * st[i][3];
                const float ig = sigmoidf_(a[0]), fg = sigmoidf_(a[1]), gg = tanhf(a[2]),
                            og = sigmoidf_(a[3]);
                const float cy = fg * cs.c[row * H + c] + ig * gg;
                cs.c_out[row * H + c] = cy;
                hy[row * H + c] = og * tanhf(cy);
            }
        }
        __syncwarp();
    }

    template <int NU, int kRW>
    __device__ static __forceinline__ void grad(const float*, float* gi, float* gh, float* dy,
                                                int H, int flags, const float*, const float*,
                                                const float* gy, float*, CellState cs,
                                                int64_t row0, int64_t n_rows, int lane,
                                                const float st[kRW][4], float dh_direct[kRW][NU]) {
        const int H4 = 4 * H;
        const bool ln = flags & SPG_GRU_LAYERNORM;
#pragma unroll
        for (int i = 0; i < kRW; ++i) {
            const int64_t row = row0 + i;
            const bool live = row < n_rows;
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const int c = lane + 32 * u;
                if (c >= H) continue;
                float yi[4], yh[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    yi[q] = (gi[i * H4 + q * H + c] - st[i][0]) * st[i][1];
                    yh[q] = (gh[i * H4 + q * H + c] - st[i][2]) * st[i][3];
                }
                const float ig = sigmoidf_(yi[0] + yh[0]), fg = sigmoidf_(yi[1] + yh[1]),
                            gg = tanhf(yi[2] + yh[2]), og = sigmoidf_(yi[3] + yh[3]);
                const float cprev = live ? cs.c[row * H + c] : 0.f;
                const float th = tanhf(fg * cprev + ig * gg);
                const float g = live ? gy[row * H + c] : 0.f;
                const float gc = live && cs.g_c ? cs.g_c[row * H + c] : 0.f;
                const float dcy = fmaf(g * og, 1.f - th * th, gc);
                dy[i * H4 + c] = dcy * gg * ig * (1.f - ig);
                dy[i * H4 + H + c] = dcy * cprev * fg * (1.f - fg);
                dy[i * H4 + 2 * H + c] = dcy * ig * (1.f - gg * gg);
                dy[i * H4 + 3 * H + c] = g * th * og * (1.f - og);
                if (live) cs.c_out[row * H + c] = dcy * fg;
                dh_direct[i][u] = 0.f;  // h enters only through W_hh and the input gate
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    gi[i * H4 + q * H + c] = ln ? yi[q] : 0.f;
                    gh[i * H4 + q * H + c] = ln ? yh[q] : 0.f;
                }
            }
        }
    }

    __device__ static __forceinline__ const float* dy_row(const float*, const float* dy_smem,
                                                          int64_t, bool, int) {
        return dy_smem;
    }
    __device__ static __forceinline__ float dy_i(const float* dp, int j, int) { return dp[j]; }
    __device__ static __forceinline__ float dy_h(const float* dp, int j, int) { return dp[j]; }
};

// ------------------------------------------------------------------ per-step kernels
template <class Cell, int kRW>
__global__ void __launch_bounds__(kCellWarps * 32)
cell_fwd_kernel(const float* __restrict__ x, const float* __restrict__ h,
                const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                const float* __restrict__ b_ih, const float* __restrict__ b_hh,
                const float* __restrict__ w_ig, const float* __restrict__ b_ig,
                float* __restrict__ hy, int64_t n_rows, int H, int flags, CellState cs) {
    SPG_PDL_ENTRY();
    extern __shared__ float sm[];
    cell_load_weights<Cell>(sm, w_ih, w_hh, w_ig, H, flags & SPG_GRU_INGATE);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* scratch = sm + cell_weight_floats<Cell>(H) + warp * cell_scratch_floats<Cell>(H, kRW);
    const int64_t warps_total = (int64_t)gridDim.x * kCellWarps;
    for (int64_t row0 = ((int64_t)blockIdx.x * kCellWarps + warp) * kRW; row0 < n_rows;
         row0 += warps_total * kRW) {
        float st[kRW][4];
        cell_rows_forward<Cell, kRW>(sm, scratch, H, flags, x, h, b_ih, b_hh, b_ig, row0, n_rows,
                                     lane, st);
        Cell::template emit<kRW>(scratch, H, flags, b_ih, b_hh, hy, cs, row0, n_rows, lane, st);
    }
}

// Backward of the cell for the RW rows starting at row0 (one warp).  x, h and gy may have been
// written earlier in the same kernel (fused recurrent kernels), hence no __restrict__ on them.
template <class Cell, int NU, int kRW>
__device__ __forceinline__ void cell_rows_backward(
    const float* sm, float* scratch, int H, int flags, const float* x, const float* h,
    const float* gy, const float* __restrict__ b_ih, const float* __restrict__ b_hh,
    const float* __restrict__ b_ig, float* d_x, float* d_h, float* __restrict__ d_gi_out,
    float* __restrict__ d_gh_out, float* __restrict__ d_q_out, float* __restrict__ xprime_out,
    float* dpre_out, CellState cs, int64_t row0, int64_t n_rows, int lane) {
    const int GH = Cell::kGates * H;
    const float* Wig_t = sm;
    const float* Wih_t = Wig_t + H * (H + 1);
    const float* Whh_t = Wih_t + H * (GH + 1);
    float* hrow = scratch;
    float* xrow = hrow + kRW * H;   // x' (gated input)
    float* srow = xrow + kRW * H;   // sigmoid(q); reused below for d_q
    float* gi = srow + kRW * H;     // raw gate inputs -> y-hat -> d_gi
    float* gh = gi + kRW * GH;      // raw gate inputs -> y-hat -> d_gh
    float* dys = gh + kRW * GH;     // the cell's dy scratch, if it has one
    const bool ln = flags & SPG_GRU_LAYERNORM;
    const bool ingate = flags & SPG_GRU_INGATE;
    {
        float st[kRW][4];
        cell_rows_forward<Cell, kRW>(sm, scratch, H, flags, x, h, b_ih, b_hh, b_ig, row0, n_rows,
                                     lane, st);
        // ---- gate gradients (w.r.t. the normalised gate inputs)
        float dh_direct[kRW][NU];  // column c = lane + 32*u
        Cell::template grad<NU, kRW>(hrow, gi, gh, dys, H, flags, b_ih, b_hh, gy, dpre_out, cs, row0,
                                     n_rows, lane, st, dh_direct);
        __syncwarp();
        // ---- layer-norm backward: d_u = rstd * (dy - mean(dy) - yhat*mean(dy*yhat))
#pragma unroll
        for (int i = 0; i < kRW; ++i) {
            const int64_t row = row0 + i;
            const bool live = row < n_rows;
            const float* dp = Cell::dy_row(dpre_out, dys + i * GH, row, live, H);
            float m1i = 0.f, m2i = 0.f, m1h = 0.f, m2h = 0.f;
            if (ln) {
                for (int j = lane; j < GH; j += 32) {
                    const float dyi = live ? Cell::dy_i(dp, j, H) : 0.f;
                    const float dyh = live ? Cell::dy_h(dp, j, H) : 0.f;
                    m1i += dyi;
                    m2i = fmaf(dyi, gi[i * GH + j], m2i);
                    m1h += dyh;
                    m2h = fmaf(dyh, gh[i * GH + j], m2h);
                }
                m1i = warp_sum(m1i) / (float)GH;
                m2i = warp_sum(m2i) / (float)GH;
                m1h = warp_sum(m1h) / (float)GH;
                m2h = warp_sum(m2h) / (float)GH;
            }
            for (int j = lane; j < GH; j += 32) {
                const float dyi = live ? Cell::dy_i(dp, j, H) : 0.f;
                const float dyh = live ? Cell::dy_h(dp, j, H) : 0.f;
                float dui, duh;
                if (ln) {
                    dui = st[i][1] * (dyi - m1i - gi[i * GH + j] * m2i);
                    duh = st[i][3] * (dyh - m1h - gh[i * GH + j] * m2h);
                } else {
                    dui = dyi;
                    duh = dyh;
                }
                gi[i * GH + j] = dui;
                gh[i * GH + j] = duh;
                if (live) {
                    d_gi_out[row * GH + j] = dui;
                    d_gh_out[row * GH + j] = duh;
                }
            }
        }
        __syncwarp();
        // ---- d_x' = d_gi * W_ih ; d_h += d_gh * W_hh
        {
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const int k = lane + 32 * u;
                if (k >= H) continue;
                float ax[kRW], ah[kRW];
#pragma unroll
                for (int i = 0; i < kRW; ++i) ax[i] = ah[i] = 0.f;
                for (int j = 0; j < GH; ++j) {
                    const float wi = Wih_t[k * (GH + 1) + j];
                    const float wh = Whh_t[k * (GH + 1) + j];
#pragma unroll
                    for (int i = 0; i < kRW; ++i) {
                        ax[i] = fmaf(wi, gi[i * GH + j], ax[i]);
                        ah[i] = fmaf(wh, gh[i * GH + j], ah[i]);
                    }
                }
#pragma unroll
                for (int i = 0; i < kRW; ++i) {
                    const int64_t row = row0 + i;
                    const float sg = srow[i * H + k];
                    const float xp = xrow[i * H + k];       // x' = s*x
                    float dq = 0.f;
                    float dxv = ax[i];
                    if (ingate) {
                        // x = x'/s is not safe when s underflows: reload the raw input.
                        const float xin = row < n_rows ? x[row * H + k] : 0.f;
                        const float ds = ax[i] * xin;
                        dxv = ax[i] * sg;
                        dq = ds * sg * (1.f - sg);
                    }
                    dh_direct[i][u] += ah[i];
                    if (row < n_rows) {
                        d_x[row * H + k] = dxv;
                        xprime_out[row * H + k] = xp;
                        d_q_out[row * H + k] = dq;
                    }
                    srow[i * H + k] = dq;  // only this lane touches srow[.][k]
                }
            }
        }
        __syncwarp();
        // ---- d_h += d_q * W_ig
        {
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const int k = lane + 32 * u;
                if (k >= H) continue;
                float a[kRW];
#pragma unroll
                for (int i = 0; i < kRW; ++i) a[i] = 0.f;
                if (ingate) {
                    for (int c = 0; c < H; ++c) {
                        const float wv = Wig_t[k * (H + 1) + c];
#pragma unroll
                        for (int i = 0; i < kRW; ++i) a[i] = fmaf(wv, srow[i * H + c], a[i]);
                    }
                }
#pragma unroll
                for (int i = 0; i < kRW; ++i) {
                    const int64_t row = row0 + i;
                    if (row < n_rows) d_h[row * H + k] = dh_direct[i][u] + a[i];
                }
            }
        }
        __syncwarp();
    }
}

template <class Cell, int NU, int kRW>
__global__ void __launch_bounds__(kCellWarps * 32)
cell_bwd_kernel(const float* __restrict__ x, const float* __restrict__ h,
                const float* __restrict__ gy, const float* __restrict__ w_ih,
                const float* __restrict__ w_hh, const float* __restrict__ b_ih,
                const float* __restrict__ b_hh, const float* __restrict__ w_ig,
                const float* __restrict__ b_ig, float* __restrict__ d_x, float* __restrict__ d_h,
                float* __restrict__ d_gi_out, float* __restrict__ d_gh_out,
                float* __restrict__ d_q_out, float* __restrict__ xprime_out,
                float* __restrict__ dpre_out, int64_t n_rows, int H, int flags, CellState cs) {
    SPG_PDL_ENTRY();
    extern __shared__ float sm[];
    cell_load_weights<Cell>(sm, w_ih, w_hh, w_ig, H, flags & SPG_GRU_INGATE);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* scratch = sm + cell_weight_floats<Cell>(H) + warp * cell_scratch_floats<Cell>(H, kRW);
    const int64_t warps_total = (int64_t)gridDim.x * kCellWarps;
    for (int64_t row0 = ((int64_t)blockIdx.x * kCellWarps + warp) * kRW; row0 < n_rows;
         row0 += warps_total * kRW)
        cell_rows_backward<Cell, NU, kRW>(sm, scratch, H, flags, x, h, gy, b_ih, b_hh, b_ig, d_x,
                                          d_h, d_gi_out, d_gh_out, d_q_out, xprime_out, dpre_out,
                                          cs, row0, n_rows, lane);
}


// ------------------------------------------------------------------ fused recurrence
// The R x {ECC, cell} loop of RNNGraphConvModule (ref: learning/modules.py:160-180) as ONE
// persistent kernel each way, for the training-batch regime (a few thousand superpoints) where
// 2R..3R separate launches are pure latency.  A warp owns a node for the whole recurrence:
//   forward   r:  inp_i = ECC(h_r)_i  ->  h_{r+1,i} = cell(inp_i, h_{r,i})   | grid barrier
//   backward  r:  (d_inp_i, d_h_i) = cell'(g_i)  | grid barrier |  g_i = d_h_i + ECC'(d_inp)_i (+cat)
// so only the neighbour exchange crosses the barrier; the cell weights are loaded into shared
// memory once per CTA instead of once per step.  The LSTM's cell state is node-local: the warp
// that owns a node reads and writes its c (forward) and dL/dc (backward) rows without any
// exchange.  Vector filters, H = 32, fp32, no idxe.
constexpr int kRecH = kC;  // the ECC rows of ecc_rows.cuh

// All CTAs are co-resident (the launchers cap the grid with the occupancy API); `counter` counts
// arrivals monotonically and is zeroed by the launcher.
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
        } while (v < target);
        __threadfence();
    }
    __syncthreads();
}

template <class Cell>
__global__ void __launch_bounds__(kCellWarps * 32)
rnn_vv_fwd_kernel(float* hs, float* inps, const float4* __restrict__ w,
                  const int* __restrict__ rowptr, const int* __restrict__ idxn,
                  const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                  const float* __restrict__ b_ih, const float* __restrict__ b_hh,
                  const float* __restrict__ w_ig, const float* __restrict__ b_ig, int n, int R,
                  int flags, unsigned* barrier, float* cs) {
    SPG_PDL_ENTRY();
    extern __shared__ float sm[];
    cell_load_weights<Cell>(sm, w_ih, w_hh, w_ig, kRecH, flags & SPG_GRU_INGATE);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* scratch = sm + cell_weight_floats<Cell>(kRecH) + warp * cell_scratch_floats<Cell>(kRecH, 1);
    const int gwarp = blockIdx.x * kCellWarps + warp, nwarps = gridDim.x * kCellWarps;
    for (int r = 0; r < R; ++r) {
        float* hcur = hs + (size_t)r * n * kRecH;
        float* hnext = hcur + (size_t)n * kRecH;
        float* inp = inps + (size_t)r * n * kRecH;
        const CellState cst = Cell::fwd_state(cs, r, (size_t)n * kRecH);
        for (int node = gwarp; node < n; node += nwarps) {
            const float4 acc = ecc_vv_row_fwd<LdCg, LdNc>(hcur, w, idxn, rowptr[node],
                                                          rowptr[node + 1], lane);
            // Stored from slot 0 in this form on purpose: written as `lane < kG`, ptxas gives this
            // kernel 8 fewer registers and the cell rows' schedule suffers (fused forward 5-11%
            // slower at 10^5 nodes on an H100 80GB HBM3, 700 W).
            if ((lane >> 3) == 0)
                *reinterpret_cast<float4*>(inp + (int64_t)node * kRecH + (lane & 7) * 4) = acc;
            __syncwarp();
            float st[1][4];
            cell_rows_forward<Cell, 1>(sm, scratch, kRecH, flags, inp, hcur, b_ih, b_hh, b_ig, node,
                                       n, lane, st);
            Cell::template emit<1>(scratch, kRecH, flags, b_ih, b_hh, hnext, cst, node, n, lane, st);
        }
        if (r + 1 < R) grid_barrier(barrier, (unsigned)(r + 1) * gridDim.x);
    }
}

template <class Cell>
__global__ void __launch_bounds__(kCellWarps * 32)
rnn_vv_bwd_kernel(const float* __restrict__ hs, const float* __restrict__ inps,
                  const float4* __restrict__ w, const float* __restrict__ gtop,
                  const float* __restrict__ gcat, const int* __restrict__ tgt_rowptr,
                  const int* __restrict__ src_rowptr, const int* __restrict__ src_perm,
                  const int* __restrict__ edge_tgt, const float* __restrict__ w_ih,
                  const float* __restrict__ w_hh, const float* __restrict__ b_ih,
                  const float* __restrict__ b_hh, const float* __restrict__ w_ig,
                  const float* __restrict__ b_ig, float* ginp, float* dh, float* gh,
                  float* __restrict__ d_gi, float* __restrict__ d_gh, float* __restrict__ d_q,
                  float* __restrict__ xp, float* dpre, int n, int R, int flags,
                  unsigned* barrier, const float* __restrict__ cs, float* dc) {
    SPG_PDL_ENTRY();
    extern __shared__ float sm[];
    cell_load_weights<Cell>(sm, w_ih, w_hh, w_ig, kRecH, flags & SPG_GRU_INGATE);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* scratch = sm + cell_weight_floats<Cell>(kRecH) + warp * cell_scratch_floats<Cell>(kRecH, 1);
    const int gwarp = blockIdx.x * kCellWarps + warp, nwarps = gridDim.x * kCellWarps;
    const size_t plane = (size_t)n * kRecH;
    for (int r = R - 1; r >= 0; --r) {
        const float* gy = (r == R - 1) ? gtop : gh;   // gh rows are produced by the same warp
        float* ginp_r = ginp + r * plane;
        const CellState cst = Cell::bwd_state(cs, dc, r, R, plane);
        for (int node = gwarp; node < n; node += nwarps)
            cell_rows_backward<Cell, 1, 1>(sm, scratch, kRecH, flags, inps + r * plane,
                                           hs + r * plane, gy, b_ih, b_hh, b_ig, ginp_r, dh,
                                           d_gi + Cell::kGates * r * plane,
                                           d_gh + Cell::kGates * r * plane, d_q + r * plane,
                                           xp + r * plane, dpre + Cell::kDpreCols * r * plane,
                                           cst, node, n, lane);
        grid_barrier(barrier, (unsigned)(R - r) * gridDim.x);
        for (int node = gwarp; node < n; node += nwarps) {
            float4 acc = ecc_vv_row_bwd_x<LdCg, LdNc>(w, ginp_r, tgt_rowptr, src_perm, edge_tgt,
                                                      src_rowptr[node], src_rowptr[node + 1], lane);
            if (lane < kG) {  // slot 0: sub = lane
                const int64_t o = (int64_t)node * kG + lane;
                acc = add4(acc, reinterpret_cast<const float4*>(dh)[o]);
                if (gcat) acc = add4(acc, __ldg(reinterpret_cast<const float4*>(gcat + r * plane) + o));
                reinterpret_cast<float4*>(gh)[o] = acc;
            }
            __syncwarp();
        }
    }
}

static inline int rnn_grid(const void* kernel, size_t smem, int n) {
    int per_sm = 0, sms = 0, dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCellWarps * 32, smem) !=
        cudaSuccess)
        return -1;
    if (per_sm > 2) per_sm = 2;
    int64_t blocks = ceil_div64(n, kCellWarps);
    const int64_t cap = (int64_t)per_sm * sms;
    if (blocks > cap) blocks = cap;
    return (int)blocks;   // 0 if the kernel does not fit at all
}

constexpr size_t kMaxSmem = 227 * 1024;  // opt-in shared memory per block on sm_90

template <class Cell>
static inline size_t cell_smem_bytes(int H, int rw) {
    return sizeof(float) *
           ((size_t)cell_weight_floats<Cell>(H) + (size_t)kCellWarps * cell_scratch_floats<Cell>(H, rw));
}

// rows per warp: 4 amortises the shared-memory weight reads when there are enough rows to fill
// the GPU; small graphs (the S3DIS training batches) use 1 so that every row gets its own warp.
// When 4 rows do not fit next to the weights, Cell::kFewerRowsIfFull says whether to take 1.
// 0: the chosen tiling does not fit.
template <class Cell>
static inline int cell_rows_per_warp(int64_t n_rows, int H) {
    int rw = n_rows >= (int64_t)kNumSMs * kCellWarps * 4 * 2 ? 4 : 1;
    if (rw == 4 && Cell::kFewerRowsIfFull && cell_smem_bytes<Cell>(H, 4) > kMaxSmem) rw = 1;
    return cell_smem_bytes<Cell>(H, rw) <= kMaxSmem ? rw : 0;
}

template <class Cell, int RW>
static int cell_fwd_launch(int kid, const float* x, const float* h, const float* w_ih,
                           const float* w_hh, const float* b_ih, const float* b_hh,
                           const float* w_ig, const float* b_ig, float* hy, CellState cs,
                           int64_t n_rows, int H, int flags, cudaStream_t stream) {
    const size_t smem = cell_smem_bytes<Cell>(H, RW);
    int64_t blocks = ceil_div64(n_rows, (int64_t)kCellWarps * RW);
    if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
    cudaError_t e = cudaFuncSetAttribute(cell_fwd_kernel<Cell, RW>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(kid, stream, (cell_fwd_kernel<Cell, RW>), (unsigned)blocks, kCellWarps * 32, smem,
               x, h, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, hy, n_rows, H, flags, cs);
    return launch_status();
}

template <class Cell>
static int cell_fwd(int kid, const float* x, const float* h, const float* w_ih, const float* w_hh,
                    const float* b_ih, const float* b_hh, const float* w_ig, const float* b_ig,
                    float* hy, CellState cs, int64_t n_rows, int H, int flags,
                    cudaStream_t stream) {
    if (H > 128) return SPG_E_UNSUPPORTED;
    const int rw = cell_rows_per_warp<Cell>(n_rows, H);
    if (rw == 4)
        return cell_fwd_launch<Cell, 4>(kid, x, h, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, hy, cs,
                                        n_rows, H, flags, stream);
    if (rw == 1)
        return cell_fwd_launch<Cell, 1>(kid, x, h, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, hy, cs,
                                        n_rows, H, flags, stream);
    return SPG_E_UNSUPPORTED;
}

template <class Cell, int NU, int RW>
static int cell_bwd_launch(int kid, const float* x, const float* h, const float* gy,
                           const float* w_ih, const float* w_hh, const float* b_ih,
                           const float* b_hh, const float* w_ig, const float* b_ig, float* d_x,
                           float* d_h, float* d_gi, float* d_gh, float* d_q, float* xprime,
                           float* dpre, CellState cs, int64_t n_rows, int H, int flags,
                           cudaStream_t stream) {
    const size_t smem = cell_smem_bytes<Cell>(H, RW);
    int64_t blocks = ceil_div64(n_rows, (int64_t)kCellWarps * RW);
    if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
    cudaError_t e = cudaFuncSetAttribute(cell_bwd_kernel<Cell, NU, RW>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    SPG_LAUNCH(kid, stream, (cell_bwd_kernel<Cell, NU, RW>), (unsigned)blocks, kCellWarps * 32,
               smem, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x, d_h, d_gi, d_gh, d_q,
               xprime, dpre, n_rows, H, flags, cs);
    return launch_status();
}

template <class Cell, int NU>
static int cell_bwd_rw(int rw, int kid, const float* x, const float* h, const float* gy,
                       const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                       const float* w_ig, const float* b_ig, float* d_x, float* d_h, float* d_gi,
                       float* d_gh, float* d_q, float* xprime, float* dpre, CellState cs,
                       int64_t n_rows, int H, int flags, cudaStream_t stream) {
    if (rw == 4)
        return cell_bwd_launch<Cell, NU, 4>(kid, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x,
                                            d_h, d_gi, d_gh, d_q, xprime, dpre, cs, n_rows, H,
                                            flags, stream);
    return cell_bwd_launch<Cell, NU, 1>(kid, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x,
                                        d_h, d_gi, d_gh, d_q, xprime, dpre, cs, n_rows, H, flags,
                                        stream);
}

template <class Cell>
static int cell_bwd(int kid, const float* x, const float* h, const float* gy, const float* w_ih,
                    const float* w_hh, const float* b_ih, const float* b_hh, const float* w_ig,
                    const float* b_ig, float* d_x, float* d_h, float* d_gi, float* d_gh,
                    float* d_q, float* xprime, float* dpre, CellState cs, int64_t n_rows, int H,
                    int flags, cudaStream_t stream) {
    if (H > 128) return SPG_E_UNSUPPORTED;
    const int rw = cell_rows_per_warp<Cell>(n_rows, H);
    if (rw == 0) return SPG_E_UNSUPPORTED;
    if (H <= 32)
        return cell_bwd_rw<Cell, 1>(rw, kid, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x,
                                    d_h, d_gi, d_gh, d_q, xprime, dpre, cs, n_rows, H, flags, stream);
    if (H <= 64)
        return cell_bwd_rw<Cell, 2>(rw, kid, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x,
                                    d_h, d_gi, d_gh, d_q, xprime, dpre, cs, n_rows, H, flags, stream);
    return cell_bwd_rw<Cell, 4>(rw, kid, x, h, gy, w_ih, w_hh, b_ih, b_hh, w_ig, b_ig, d_x, d_h,
                                d_gi, d_gh, d_q, xprime, dpre, cs, n_rows, H, flags, stream);
}

// cooperative launch: the driver guarantees that all CTAs are co-resident (the grid barrier
// spins on them) or fails the launch; other streams' kernels cannot starve the grid
static int rnn_cooperative_launch(int kid, const void* kernel, int n, void** kargs, size_t smem,
                                  void* barrier_ws, cudaStream_t stream) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    const int blocks = rnn_grid(kernel, smem, n);
    if (blocks <= 0) return SPG_E_UNSUPPORTED;
    e = cudaMemsetAsync(barrier_ws, 0, sizeof(unsigned), stream);
    if (e != cudaSuccess) return (int)e;
    {
        ::spg::LaunchScope _scope(kid, stream);
        e = cudaLaunchCooperativeKernel(kernel, dim3((unsigned)blocks), dim3(kCellWarps * 32), kargs,
                                        smem, stream);
    }
    if (e != cudaSuccess) return (int)e;
    return launch_status();
}

template <class Cell>
static int rnn_vv_fwd(int kid, float* hs, float* cs, float* inps, const float* w,
                      const int32_t* tgt_rowptr, const int32_t* idxn, const float* weight_ih,
                      const float* weight_hh, const float* bias_ih, const float* bias_hh,
                      const float* ig_weight, const float* ig_bias, int64_t n_nodes,
                      int n_repeats, int flags, void* barrier_ws, cudaStream_t stream) {
    const float4* w4 = reinterpret_cast<const float4*>(w);
    int n_i = (int)n_nodes;
    unsigned* bar = reinterpret_cast<unsigned*>(barrier_ws);
    void* kargs[] = {&hs, &inps, &w4, &tgt_rowptr, &idxn, &weight_ih, &weight_hh, &bias_ih, &bias_hh,
                     &ig_weight, &ig_bias, &n_i, &n_repeats, &flags, &bar, &cs};
    return rnn_cooperative_launch(kid, (const void*)rnn_vv_fwd_kernel<Cell>, n_i, kargs,
                                  cell_smem_bytes<Cell>(kRecH, 1), barrier_ws, stream);
}

template <class Cell>
static int rnn_vv_bwd(int kid, const float* hs, const float* cs, const float* inps, const float* w,
                      const float* grad_top, const float* grad_cat, const int32_t* tgt_rowptr,
                      const int32_t* src_rowptr, const int32_t* src_perm, const int32_t* edge_tgt,
                      const float* weight_ih, const float* weight_hh, const float* bias_ih,
                      const float* bias_hh, const float* ig_weight, const float* ig_bias,
                      float* grad_inp, float* d_h_ws, float* d_c_ws, float* grad_h0, float* d_gi,
                      float* d_gh, float* d_q, float* xprime, float* dpre, int64_t n_nodes,
                      int n_repeats, int flags, void* barrier_ws, cudaStream_t stream) {
    const float4* w4 = reinterpret_cast<const float4*>(w);
    int n_i = (int)n_nodes;
    unsigned* bar = reinterpret_cast<unsigned*>(barrier_ws);
    void* kargs[] = {&hs, &inps, &w4, &grad_top, &grad_cat, &tgt_rowptr, &src_rowptr, &src_perm,
                     &edge_tgt, &weight_ih, &weight_hh, &bias_ih, &bias_hh, &ig_weight, &ig_bias,
                     &grad_inp, &d_h_ws, &grad_h0, &d_gi, &d_gh, &d_q, &xprime, &dpre, &n_i,
                     &n_repeats, &flags, &bar, &cs, &d_c_ws};
    return rnn_cooperative_launch(kid, (const void*)rnn_vv_bwd_kernel<Cell>, n_i, kargs,
                                  cell_smem_bytes<Cell>(kRecH, 1), barrier_ws, stream);
}

static int cell_args_ok(const float* bias_ih, const float* bias_hh, const float* ig_weight,
                        const float* ig_bias, int flags) {
    if ((flags & SPG_GRU_BIAS) && (!bias_ih || !bias_hh)) return 0;
    if ((flags & SPG_GRU_INGATE) && (!ig_weight || !ig_bias)) return 0;
    return 1;
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_gru_fwd(const float* x, const float* h, const float* weight_ih, const float* weight_hh,
                const float* bias_ih, const float* bias_hh, const float* ig_weight,
                const float* ig_bias, float* hy, int64_t n_rows, int hidden, int flags,
                spg_stream_t stream) {
    if (n_rows < 0 || hidden <= 0) return SPG_E_BADARG;
    if (n_rows == 0) return SPG_OK;
    if (!x || !h || !weight_ih || !weight_hh || !hy) return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return cell_fwd<GruCell>(K_GRU_FWD, x, h, weight_ih, weight_hh, bias_ih, bias_hh, ig_weight,
                             ig_bias, hy, CellState{}, n_rows, hidden, flags,
                             (cudaStream_t)stream);
}

int spg_gru_bwd(const float* x, const float* h, const float* grad_hy, const float* weight_ih,
                const float* weight_hh, const float* bias_ih, const float* bias_hh,
                const float* ig_weight, const float* ig_bias, float* d_x, float* d_h,
                float* d_gi, float* d_gh, float* d_q, float* xprime, float* dpre,
                int64_t n_rows, int hidden, int flags, spg_stream_t stream) {
    if (n_rows < 0 || hidden <= 0) return SPG_E_BADARG;
    if (n_rows == 0) return SPG_OK;
    if (!x || !h || !grad_hy || !weight_ih || !weight_hh || !d_x || !d_h || !d_gi || !d_gh ||
        !d_q || !xprime || !dpre)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return cell_bwd<GruCell>(K_GRU_BWD, x, h, grad_hy, weight_ih, weight_hh, bias_ih, bias_hh,
                             ig_weight, ig_bias, d_x, d_h, d_gi, d_gh, d_q, xprime, dpre,
                             CellState{}, n_rows, hidden, flags, (cudaStream_t)stream);
}

int spg_lstm_fwd(const float* x, const float* h, const float* c, const float* weight_ih,
                 const float* weight_hh, const float* bias_ih, const float* bias_hh,
                 const float* ig_weight, const float* ig_bias, float* hy, float* cy,
                 int64_t n_rows, int hidden, int flags, spg_stream_t stream) {
    if (n_rows < 0 || hidden <= 0) return SPG_E_BADARG;
    if (n_rows == 0) return SPG_OK;
    if (!x || !h || !c || !weight_ih || !weight_hh || !hy || !cy) return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return cell_fwd<LstmCell>(K_LSTM_FWD, x, h, weight_ih, weight_hh, bias_ih, bias_hh, ig_weight,
                              ig_bias, hy, CellState{c, cy, nullptr}, n_rows, hidden, flags,
                              (cudaStream_t)stream);
}

int spg_lstm_bwd(const float* x, const float* h, const float* c, const float* grad_hy,
                 const float* grad_cy, const float* weight_ih, const float* weight_hh,
                 const float* bias_ih, const float* bias_hh, const float* ig_weight,
                 const float* ig_bias, float* d_x, float* d_h, float* d_c, float* d_gi,
                 float* d_gh, float* d_q, float* xprime, int64_t n_rows, int hidden, int flags,
                 spg_stream_t stream) {
    if (n_rows < 0 || hidden <= 0) return SPG_E_BADARG;
    if (n_rows == 0) return SPG_OK;
    if (!x || !h || !c || !grad_hy || !weight_ih || !weight_hh || !d_x || !d_h || !d_c || !d_gi ||
        !d_gh || !d_q || !xprime)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return cell_bwd<LstmCell>(K_LSTM_BWD, x, h, grad_hy, weight_ih, weight_hh, bias_ih, bias_hh,
                              ig_weight, ig_bias, d_x, d_h, d_gi, d_gh, d_q, xprime, nullptr,
                              CellState{c, d_c, grad_cy}, n_rows, hidden, flags,
                              (cudaStream_t)stream);
}

int spg_rnn_vv_supported(int64_t n_nodes, int hidden) {
    // any number of nodes: the kernels walk the nodes grid-strided inside every step
    return hidden == kRecH && n_nodes > 0 && n_nodes < ((int64_t)1 << 31) / (4 * kRecH);
}

int spg_rnn_vv_fwd(float* hs, float* inps, const float* w, const int32_t* tgt_rowptr,
                   const int32_t* idxn, const float* weight_ih, const float* weight_hh,
                   const float* bias_ih, const float* bias_hh, const float* ig_weight,
                   const float* ig_bias, int64_t n_nodes, int hidden, int n_repeats, int flags,
                   void* barrier_ws, spg_stream_t stream) {
    if (n_nodes < 0 || n_repeats < 0) return SPG_E_BADARG;
    if (n_nodes == 0 || n_repeats == 0) return SPG_OK;
    if (!spg_rnn_vv_supported(n_nodes, hidden)) return SPG_E_UNSUPPORTED;
    if (!hs || !inps || !w || !tgt_rowptr || !idxn || !weight_ih || !weight_hh || !barrier_ws)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return rnn_vv_fwd<GruCell>(K_RNN_FWD, hs, nullptr, inps, w, tgt_rowptr, idxn, weight_ih,
                               weight_hh, bias_ih, bias_hh, ig_weight, ig_bias, n_nodes, n_repeats,
                               flags, barrier_ws, (cudaStream_t)stream);
}

int spg_rnn_vv_bwd(const float* hs, const float* inps, const float* w, const float* grad_top,
                   const float* grad_cat, const int32_t* tgt_rowptr, const int32_t* src_rowptr,
                   const int32_t* src_perm, const int32_t* edge_tgt, const float* weight_ih,
                   const float* weight_hh, const float* bias_ih, const float* bias_hh,
                   const float* ig_weight, const float* ig_bias, float* grad_inp, float* d_h_ws,
                   float* grad_h0, float* d_gi, float* d_gh, float* d_q, float* xprime,
                   float* dpre, int64_t n_nodes, int hidden, int n_repeats, int flags,
                   void* barrier_ws, spg_stream_t stream) {
    if (n_nodes < 0 || n_repeats < 0) return SPG_E_BADARG;
    if (n_nodes == 0 || n_repeats == 0) return SPG_OK;
    if (!spg_rnn_vv_supported(n_nodes, hidden)) return SPG_E_UNSUPPORTED;
    if (!hs || !inps || !w || !grad_top || !tgt_rowptr || !src_rowptr || !src_perm || !edge_tgt ||
        !weight_ih || !weight_hh || !grad_inp || !d_h_ws || !grad_h0 || !d_gi || !d_gh || !d_q ||
        !xprime || !dpre || !barrier_ws)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return rnn_vv_bwd<GruCell>(K_RNN_BWD, hs, nullptr, inps, w, grad_top, grad_cat, tgt_rowptr,
                               src_rowptr, src_perm, edge_tgt, weight_ih, weight_hh, bias_ih,
                               bias_hh, ig_weight, ig_bias, grad_inp, d_h_ws, nullptr, grad_h0,
                               d_gi, d_gh, d_q, xprime, dpre, n_nodes, n_repeats, flags,
                               barrier_ws, (cudaStream_t)stream);
}

int spg_rnn_vv_lstm_fwd(float* hs, float* cs, float* inps, const float* w,
                        const int32_t* tgt_rowptr, const int32_t* idxn, const float* weight_ih,
                        const float* weight_hh, const float* bias_ih, const float* bias_hh,
                        const float* ig_weight, const float* ig_bias, int64_t n_nodes, int hidden,
                        int n_repeats, int flags, void* barrier_ws, spg_stream_t stream) {
    if (n_nodes < 0 || n_repeats < 0) return SPG_E_BADARG;
    if (n_nodes == 0 || n_repeats == 0) return SPG_OK;
    if (!spg_rnn_vv_supported(n_nodes, hidden)) return SPG_E_UNSUPPORTED;
    if (!hs || !cs || !inps || !w || !tgt_rowptr || !idxn || !weight_ih || !weight_hh ||
        !barrier_ws)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return rnn_vv_fwd<LstmCell>(K_RNN_LSTM_FWD, hs, cs, inps, w, tgt_rowptr, idxn, weight_ih,
                                weight_hh, bias_ih, bias_hh, ig_weight, ig_bias, n_nodes,
                                n_repeats, flags, barrier_ws, (cudaStream_t)stream);
}

int spg_rnn_vv_lstm_bwd(const float* hs, const float* cs, const float* inps, const float* w,
                        const float* grad_top, const float* grad_cat, const int32_t* tgt_rowptr,
                        const int32_t* src_rowptr, const int32_t* src_perm,
                        const int32_t* edge_tgt, const float* weight_ih, const float* weight_hh,
                        const float* bias_ih, const float* bias_hh, const float* ig_weight,
                        const float* ig_bias, float* grad_inp, float* d_h_ws, float* d_c_ws,
                        float* grad_h0, float* d_gi, float* d_gh, float* d_q, float* xprime,
                        int64_t n_nodes, int hidden, int n_repeats, int flags, void* barrier_ws,
                        spg_stream_t stream) {
    if (n_nodes < 0 || n_repeats < 0) return SPG_E_BADARG;
    if (n_nodes == 0 || n_repeats == 0) return SPG_OK;
    if (!spg_rnn_vv_supported(n_nodes, hidden)) return SPG_E_UNSUPPORTED;
    if (!hs || !cs || !inps || !w || !grad_top || !tgt_rowptr || !src_rowptr || !src_perm ||
        !edge_tgt || !weight_ih || !weight_hh || !grad_inp || !d_h_ws || !d_c_ws || !grad_h0 ||
        !d_gi || !d_gh || !d_q || !xprime || !barrier_ws)
        return SPG_E_BADARG;
    if (!cell_args_ok(bias_ih, bias_hh, ig_weight, ig_bias, flags)) return SPG_E_BADARG;
    return rnn_vv_bwd<LstmCell>(K_RNN_LSTM_BWD, hs, cs, inps, w, grad_top, grad_cat, tgt_rowptr,
                                src_rowptr, src_perm, edge_tgt, weight_ih, weight_hh, bias_ih,
                                bias_hh, ig_weight, ig_bias, grad_inp, d_h_ws, d_c_ws, grad_h0,
                                d_gi, d_gh, d_q, xprime, nullptr, n_nodes, n_repeats, flags,
                                barrier_ws, (cudaStream_t)stream);
}

}  // extern "C"
