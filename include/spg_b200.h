/*
 * spg_b200.h — C-ABI of libspg_b200.so, the sm_90a (H100) implementation of the
 * superpoint-graph learning hot path of loicland/superpoint_graph.
 *
 * Every entry point is `extern "C"`, takes plain device pointers, sizes and the
 * CUDA stream to enqueue on (a `cudaStream_t` passed as `void*`), never
 * synchronises the host and never throws.  Return value: 0 on success,
 * a negative SPG_E_* code for an argument the kernels cannot serve, or a
 * positive `cudaError_t` if the launch failed (see spg_error_string()).
 *
 * All matrices are row-major and contiguous unless a leading dimension is
 * given.  `dtype`: 0 = float32, 1 = float64 (float64 is served by the generic
 * kernels only; it exists for gradcheck-style tests, reference
 * learning/ecc/test_GraphConvModule.py:25).
 *
 * A call whose scratch is sized by a `spg_*_workspace` query takes that scratch as one `workspace`
 * argument and no other: 256-byte aligned (else SPG_E_ALIGN) and at least the reported bytes (else
 * SPG_E_BADARG), both checked before any kernel is launched.  The reported size is exact, with no slack.
 *
 * Each function names the reference code it replaces as
 * `ref: <file>:<lines>` relative to the reference repository root.
 */
#ifndef SPG_B200_H_
#define SPG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* spg_stream_t; /* cudaStream_t */

#define SPG_OK 0
#define SPG_E_BADARG (-1)      /* null pointer / negative size / bad flag */
#define SPG_E_UNSUPPORTED (-2) /* shape or dtype not served by any kernel */
#define SPG_E_ALIGN (-3)       /* pointer or leading dimension misaligned */

#define SPG_F32 0
#define SPG_F64 1

/* ---------------------------------------------------------------- runtime */
int spg_version(void);
const char* spg_error_string(int code);
/* Programmatic dependent launch of every kernel of the library (default on; environment SPG_PDL=0 switches it
 * off): kernel n+1 of a stream is scheduled while kernel n runs and waits on the device (griddepcontrol.wait)
 * for n's results.  No reference counterpart: the reference launches its kernels in plain stream order. */
int spg_set_pdl(int enabled);
/* cudaMemsetAsync(ptr, 0, bytes) on the stream. */
int spg_zero(void* ptr, int64_t bytes, spg_stream_t stream);

/* Per-kernel launch accounting.  Counting is always on; timing (a pair of CUDA
 * events recorded around every launch on the launching stream) only while
 * enabled.  spg_prof_collect() synchronises the recorded events and folds them
 * into per-kernel totals.                                                    */
int spg_prof_enable(int on);
int spg_prof_reset(void);
int spg_prof_collect(void);
int spg_prof_num_kernels(void);
const char* spg_prof_kernel_name(int kernel_id);
int spg_prof_kernel_stats(int kernel_id, int64_t* launches, double* total_ms);
int64_t spg_prof_total_launches(void);

/* ------------------------------------------------- edge-conditioned conv  */
/* Graph structure arrays (all int32, device):
 *   tgt_rowptr[n_out+1]  exclusive scan of the in-degrees `degs`
 *                        (ref: learning/ecc/GraphConvInfo.py:56, cuda_kernels.py:123)
 *   idxn[n_edges]        source node of every edge, edges sorted by target
 *                        (ref: GraphConvInfo.py:50-52)
 *   idxe[n_edges]|NULL   row of `w` used by every edge (edge-feature compaction,
 *                        ref: GraphConvInfo.py:59-62); NULL = identity
 *   edge_tgt[n_edges]    target node of every edge
 *   src_rowptr[n_in+1], src_perm[n_edges]
 *                        CSR over SOURCE nodes: src_perm lists edge ids grouped by
 *                        source (stable), used for the atomic-free grad_input.   */

/* out[i,:] = (1/deg_i) * sum_{e in in(i)} op(x[idxn_e,:], w[e]) ; 0 if deg_i==0.
 * w_is_matrix=0: w [n_w_rows,c_in], op = elementwise product (needs c_in==c_out)
 * w_is_matrix=1: w [n_w_rows,c_in,c_out], op = vector-matrix product.
 * ref: learning/ecc/GraphConvModule.py:43-94 (GraphConvFunction.forward),
 *      learning/ecc/cuda_kernels.py:55-86,117-127 (conv_aggregate_fw).        */
int spg_ecc_fwd(const void* x, const void* w, const int32_t* tgt_rowptr, const int32_t* idxn,
                const int32_t* idxe, void* out, int64_t n_out, int64_t n_edges, int c_in,
                int c_out, int w_is_matrix, int dtype, spg_stream_t stream);

/* grad_w[e] (+)= sum_{r<n_iter} op'(x_r[idxn_e,:], g_r[tgt_e,:]/deg_tgt)
 * with x_r = xs + r*x_iter_stride elements, g_r = gs + r*g_iter_stride elements;
 * op' = elementwise product (vector filters) or outer product (matrix filters).
 * n_iter>1 folds the recurrent reuse of one filter bank (ref:
 * learning/modules.py:160,171-176) into one pass.  With idxe the rows are
 * accumulated atomically into grad_w, which the caller must have zeroed.
 * ref: GraphConvModule.py:108-133, cuda_kernels.py:88-114,129-139.             */
int spg_ecc_bwd_w(const void* xs, const void* gs, int64_t x_iter_stride, int64_t g_iter_stride,
                  int n_iter, const int32_t* tgt_rowptr, const int32_t* idxn,
                  const int32_t* idxe, const int32_t* edge_tgt, void* grad_w, int64_t n_out,
                  int64_t n_edges, int c_in, int c_out, int w_is_matrix, int accumulate,
                  int dtype, spg_stream_t stream);

/* grad_x[j,:] = add0[j,:] + add1[j,:] + sum_{e: idxn_e=j} op''(w[e], g[tgt_e,:]/deg_tgt)
 * (add0/add1 may be NULL).  ref: GraphConvModule.py:135-146.                    */
int spg_ecc_bwd_x(const void* w, const void* g, const int32_t* tgt_rowptr,
                  const int32_t* src_rowptr, const int32_t* src_perm, const int32_t* edge_tgt,
                  const int32_t* idxe, const void* add0, const void* add1, void* grad_x,
                  int64_t n_in, int64_t n_edges, int c_in, int c_out, int w_is_matrix,
                  int dtype, spg_stream_t stream);

/* ------------------------------------------------------------ ECC-CRF  */
/* The mean-field recurrence of ECC_CRFModule over a square graph (n nodes, n_in == n_out),
 * float32, matrix filters w [n_edges,C,C] with 1 <= C <= 32, no idxe.
 *   Q_0 = softmax(U);  Z_r = U - P_r,  P_r[t] = (1/deg_t) sum_{e in in(t)} Q_{r-1}[idxn_e] @ w[e];
 *   Q_r = softmax(Z_r) for r < R;  the module returns Z_R.
 * ref: learning/modules.py:185-202 (ECC_CRFModule.forward), graphnet.py:57-64.       */

/* out = softmax(x) over each row of x [n,C]  (g == NULL), or
 * out = x * (g - <g,x>) row by row, the softmax backward with x = softmax output (g != NULL).
 * ref: modules.py:196,201 (nnf.softmax on 2-D input, dim 1).                       */
int spg_crf_softmax(const float* x, const float* g, float* out, int64_t n, int C,
                    spg_stream_t stream);

/* One forward iteration: out[t] = softmax(Z_r[t]) if do_softmax else Z_r[t], with Z_r as above from
 * U [n,C] and q_prev = Q_{r-1} [n,C]; a warp per target, filters read once, no atomics.
 * ref: modules.py:197-201 (propagation, `input - Q`, softmax).                       */
int spg_crf_fwd_step(const float* u, const float* q_prev, const float* w, const int32_t* tgt_rowptr,
                     const int32_t* idxn, float* out, int64_t n, int64_t n_edges, int C,
                     int do_softmax, spg_stream_t stream);

/* One backward iteration over the SOURCE CSR (a warp per source row, no atomics), from
 * gp = dL/dP_r = -dL/dZ_r [n,C]:
 *   dQ[j]  = sum_{e: idxn_e = j} w[e] @ gp[tgt_e] / deg_tgt
 *   dZ[j]  = q_prev[j] * (dQ[j] - <dQ[j], q_prev[j]>)          (q_prev = Q_{r-1})
 *   du_out[j] = du_in[j] + dZ[j]    (du_out may alias du_in)
 *   gp_out[j] = -dZ[j]              (gp_out = dL/dP_{r-1}; NULL skips it)
 * ref: the autograd of modules.py:197-201 and GraphConvModule.py:135-146.            */
int spg_crf_bwd_step(const float* w, const float* gp, const float* q_prev,
                     const float* du_in, float* du_out, float* gp_out, const int32_t* tgt_rowptr,
                     const int32_t* src_rowptr, const int32_t* src_perm, const int32_t* edge_tgt,
                     int64_t n, int64_t n_edges, int C, spg_stream_t stream);


/* ----------------------------------------------------------- GRUCellEx    */
#define SPG_GRU_LAYERNORM 1
#define SPG_GRU_INGATE 2
#define SPG_GRU_BIAS 4
/* hy = GRUCellEx(x, h).  input_size == hidden_size == H (as built by
 * learning/graphnet.py:74).  weight_ih/weight_hh [3H,H], bias_* [3H],
 * ig_weight [H,H], ig_bias [H].  ref: learning/modules.py:205-251.             */
int spg_gru_fwd(const float* x, const float* h, const float* weight_ih, const float* weight_hh,
                const float* bias_ih, const float* bias_hh, const float* ig_weight,
                const float* ig_bias, float* hy, int64_t n_rows, int hidden, int flags,
                spg_stream_t stream);
/* Backward of the cell for one step.  Row-local gradients d_x, d_h are final; the
 * parameter gradients are left as per-row factors for one batched reduction over
 * all recurrent steps: d_gi, d_gh [n,3H] (grads of the pre-norm gate inputs),
 * d_q [n,H] (grad of the input-gate pre-activation), xprime [n,H] (gated input),
 * dpre [n,4H] = [d_pr,d_pz,d_pn,d_pn*r] (bias gradients' summands).             */
int spg_gru_bwd(const float* x, const float* h, const float* grad_hy, const float* weight_ih,
                const float* weight_hh, const float* bias_ih, const float* bias_hh,
                const float* ig_weight, const float* ig_bias, float* d_x, float* d_h,
                float* d_gi, float* d_gh, float* d_q, float* xprime, float* dpre,
                int64_t n_rows, int hidden, int flags, spg_stream_t stream);

/* ------------------------------------------- fused recurrence (R x {ECC, cell})
 * The whole loop of RNNGraphConvModule.forward (ref: learning/modules.py:160-180:
 * `for r: input = GraphConvFunction(hx, weights); hx = cell(input, hx)`) as ONE persistent
 * kernel per direction, for vector filters ([n_edges,H]), H == 32, no idxe, and batches
 * small enough that a warp per superpoint fills the GPU (spg_rnn_vv_supported).  A warp
 * owns a node through all steps; steps are separated by a grid-wide barrier
 * (barrier_ws: >= 4 bytes of device memory, zeroed by the call).
 *   hs   [R+1,n,H]  hs[0] = initial state on entry; hs[1..R] written
 *   inps [R,n,H]    ECC outputs of every step (kept for the backward)              */
int spg_rnn_vv_supported(int64_t n_nodes, int hidden);
int spg_rnn_vv_fwd(float* hs, float* inps, const float* w, const int32_t* tgt_rowptr,
                   const int32_t* idxn, const float* weight_ih, const float* weight_hh,
                   const float* bias_ih, const float* bias_hh, const float* ig_weight,
                   const float* ig_bias, int64_t n_nodes, int hidden, int n_repeats, int flags,
                   void* barrier_ws, spg_stream_t stream);
/* Backward of the loop: grad_top [n,H] is the gradient w.r.t. hs[R]; grad_cat (NULL or
 * [R+1,n,H]) the direct gradient of every hs[r] when all states were concatenated
 * (`cat_all`, ref: modules.py:166,178; grad_top is then grad_cat[R]).  Outputs: grad_inp
 * [R,n,H] (gradient of every ECC output, consumed by spg_ecc_bwd_w), grad_h0 [n,H], and the
 * per-row parameter-gradient factors of spg_gru_bwd stacked over the steps
 * (d_gi,d_gh [R,n,3H]; d_q,xprime [R,n,H]; dpre [R,n,4H]).  d_h_ws: [n,H] scratch.      */
int spg_rnn_vv_bwd(const float* hs, const float* inps, const float* w, const float* grad_top,
                   const float* grad_cat, const int32_t* tgt_rowptr, const int32_t* src_rowptr,
                   const int32_t* src_perm, const int32_t* edge_tgt, const float* weight_ih,
                   const float* weight_hh, const float* bias_ih, const float* bias_hh,
                   const float* ig_weight, const float* ig_bias, float* grad_inp, float* d_h_ws,
                   float* grad_h0, float* d_gi, float* d_gh, float* d_q, float* xprime,
                   float* dpre, int64_t n_nodes, int hidden, int n_repeats, int flags,
                   void* barrier_ws, spg_stream_t stream);

/* ----------------------------------------------------------- LSTMCellEx   */
/* (hy, cy) = LSTMCellEx(x, (h, c)).  input_size == hidden_size == H (as built by
 * learning/graphnet.py:74).  weight_ih/weight_hh [4H,H], bias_* [4H] (added inside the linears,
 * before the norm), ig_weight [H,H], ig_bias [H]; gates (i, f, g, o) in that order.  flags are the
 * SPG_GRU_LAYERNORM/INGATE/BIAS bits above: they mean the same for both cells.  H <= 73: the
 * weights ((2*4+1)*H*H floats) and one row per warp must fit in shared memory, else SPG_E_UNSUPPORTED.
 * ref: learning/modules.py:281-308 (LSTMCellEx.forward).                                          */
int spg_lstm_fwd(const float* x, const float* h, const float* c, const float* weight_ih,
                 const float* weight_hh, const float* bias_ih, const float* bias_hh,
                 const float* ig_weight, const float* ig_bias, float* hy, float* cy,
                 int64_t n_rows, int hidden, int flags, spg_stream_t stream);
/* Backward of the cell for one step, from grad_hy and grad_cy (NULL = 0; d_c may alias it).
 * d_x, d_h, d_c are final; the parameter gradients are left as per-row factors for one batched
 * reduction over all recurrent steps: d_gi, d_gh [n,4H] (grads of the pre-norm gate inputs,
 * biases included: the bias gradients are their column sums), d_q [n,H] (grad of the input-gate
 * pre-activation), xprime [n,H] (gated input).
 * ref: the autograd of learning/modules.py:281-308.                                              */
int spg_lstm_bwd(const float* x, const float* h, const float* c, const float* grad_hy,
                 const float* grad_cy, const float* weight_ih, const float* weight_hh,
                 const float* bias_ih, const float* bias_hh, const float* ig_weight,
                 const float* ig_bias, float* d_x, float* d_h, float* d_c, float* d_gi,
                 float* d_gh, float* d_q, float* xprime, int64_t n_rows, int hidden, int flags,
                 spg_stream_t stream);
/* The fused recurrence of spg_rnn_vv_fwd/bwd with LSTMCellEx as the cell (same conditions,
 * spg_rnn_vv_supported).  cs [R+1,n,H]: cs[0] = initial cell state on entry (RNNGraphConvModule
 * starts from zeros), cs[1..R] written.  The backward takes no gradient for any cs[r] (the cell
 * state never leaves the module), carries dL/dc in d_c_ws [n,H] (scratch) and leaves the factors
 * of spg_lstm_bwd stacked over the steps (d_gi,d_gh [R,n,4H]; d_q,xprime [R,n,H]).
 * ref: learning/modules.py:167-183 (the `_isLSTM` branch: cx = 0, (hx, cx) = cell(input, (hx, cx))). */
int spg_rnn_vv_lstm_fwd(float* hs, float* cs, float* inps, const float* w,
                        const int32_t* tgt_rowptr, const int32_t* idxn, const float* weight_ih,
                        const float* weight_hh, const float* bias_ih, const float* bias_hh,
                        const float* ig_weight, const float* ig_bias, int64_t n_nodes, int hidden,
                        int n_repeats, int flags, void* barrier_ws, spg_stream_t stream);
int spg_rnn_vv_lstm_bwd(const float* hs, const float* cs, const float* inps, const float* w,
                        const float* grad_top, const float* grad_cat, const int32_t* tgt_rowptr,
                        const int32_t* src_rowptr, const int32_t* src_perm,
                        const int32_t* edge_tgt, const float* weight_ih, const float* weight_hh,
                        const float* bias_ih, const float* bias_hh, const float* ig_weight,
                        const float* ig_bias, float* grad_inp, float* d_h_ws, float* d_c_ws,
                        float* grad_h0, float* d_gi, float* d_gh, float* d_q, float* xprime,
                        int64_t n_nodes, int hidden, int n_repeats, int flags, void* barrier_ws,
                        spg_stream_t stream);

/* ------------------------------------------------------------- dense      */
/* C[M,N] = opA(A) * opB(B) (+ bias[N]), fp32, FMA accumulation.
 *   a_kmajor=1: A is [M,K] (ld = lda, K contiguous); 0: A is [K,M] (M contiguous)
 *   b_kmajor=1: B is [N,K] (ld = ldb, K contiguous); 0: B is [K,N] (N contiguous)
 * Optional fused prologue (the "BN apply + ReLU of the producing layer"):
 *   a_scale/a_shift [K] (needs a_kmajor=1): A'[m,k] = f(A[m,k]*a_scale[k]+a_shift[k])
 *   b_scale/b_shift [N] (needs b_kmajor=0): B'[k,n] = f(B[k,n]*b_scale[n]+b_shift[n])
 *   f = ReLU if the matching *_relu flag is set (scale may be NULL = 1, shift NULL = 0).
 * split_k>1 reduces K in `split_k` slices through `workspace`
 * (>= split_k*M*N floats) and a deterministic second pass.
 * ref: the nn.Conv1d(k=1)/nn.Linear calls of learning/pointnet.py:29,41,51,85,100
 *      and learning/graphnet.py:27,32, and their autograd backward.            */
int spg_gemm(const float* A, int64_t lda, int a_kmajor, const float* B, int64_t ldb, int b_kmajor,
             const float* bias, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
             const float* a_scale, const float* a_shift, int a_relu, const float* b_scale,
             const float* b_shift, int b_relu, int split_k, float* workspace, float* stats_ws,
             spg_stream_t stream);
/* Fused batch statistics: if stats_ws != NULL (needs split_k == 1) spg_gemm also writes, per
 * 128-row tile and output column, (count, mean, M2) into stats_ws[spg_gemm_stats_tiles(M), N, 3];
 * spg_colstats_merge folds n_partials such triples per column into mean[C], biased var[C].   */
int64_t spg_gemm_stats_tiles(int64_t M);
int spg_colstats_merge(float* partials, int64_t n_partials, int C, float* mean, float* var,
                       spg_stream_t stream);
/* merge + spg_bn_fold in one pass (the last merge level folds): */
int spg_colstats_merge_fold(float* partials, int64_t n_partials, int C, float* mean, float* var,
                            const float* gamma, const float* beta, float eps, float* scale,
                            float* shift, float* running_mean, float* running_var,
                            int64_t* num_batches_tracked, float momentum, int64_t M,
                            spg_stream_t stream);
/* (the merge is two-level: `partials` needs room for ceil(n_partials/256) extra triples per column
 *  after the n_partials*C*3 floats; the same holds for stats_ws)                                */

/* wgmma tensor-core path of the same product for the large point-wise layers:
 *   C[M,N] = f(A)[M,K] * B[N,K]^T + bias in fp32-equivalent precision (3xTF32 split, fp32 register
 *   accumulation), lda/ldc % 4 == 0, 16-byte aligned pointers.
 * B is given as a pre-split, pre-swizzled image built by spg_tc_pack_weights from W (ld = ldw):
 *   transpose=0: B[n][k] = W[n][k] (forward, W = [N,K]); transpose=1: B[n][k] = W[k][n]
 *   (data gradient, W = [K,N]).  image needs spg_tc_weight_image_floats(N,K) floats; entries with
 *   k >= k_valid are zero (K padded to a multiple of 32, e.g. the 14 input features -> 32).
 * Returns SPG_E_UNSUPPORTED for other shapes (use spg_gemm).                                      */
int64_t spg_tc_weight_image_floats(int N, int K);
int spg_tc_pack_weights(const float* W, int64_t ldw, int transpose, int N, int K, int k_valid,
                        float* image, spg_stream_t stream);
/* image of diag(row_scale) * W (W = [N,K], ld ldw): eval-mode BatchNorm folded into the weights */
int spg_tc_pack_weights_scaled(const float* W, int64_t ldw, const float* row_scale, int N, int K, int k_valid,
                               float* image, spg_stream_t stream);
/* All weight images of a model in one launch: table (device, int64 [n_jobs,8]) rows are
 * {W, ldw, transpose, N, K, k_valid, image, first element index}; total = sum N*K.            */
int spg_tc_pack_weights_multi(const int64_t* table, int n_jobs, int64_t total, spg_stream_t stream);
int spg_tc_gemm_supported(int64_t M, int N, int K);
/* Plain form (affine+ReLU prologue, no fused reduction).  N % 32 == 0 (N <= 64) or N % 64 == 0,
 * N <= 256, K % 32 == 0, K <= 256.  The resident weight slice is loaded by TMA
 * (cp.async.bulk.tensor over a 2-D view of the image).                                           */
int spg_tc_gemm(const float* A, int64_t lda, const float* weight_image, const float* bias, float* C,
                int64_t ldc, int64_t M, int N, int K, const float* a_scale, const float* a_shift,
                int a_relu, spg_stream_t stream);
/* Full form: the BatchNorm bookkeeping of a training step fused on both sides of the product
 * (replaces nn.BatchNorm1d's statistics pass and autograd's BatchNorm/ReLU backward kernels around
 * the Conv1d(k=1) stacks of learning/pointnet.py:27-37,83-96).
 *   prologue  a2 == NULL : f(A) = relu?(A*a_scale + a_shift)                     (forward)
 *             a2 != NULL : A = dL/d(activation), a2 = raw layer output y [M,K] (ld lda2);
 *                          f = a_scale*(gz - s1/M - xhat*s2/M), gz = relu'(y*a_scale+a_shift)*A,
 *                          xhat = (y-a_mean)/sqrt(a_var+a_eps), a_s12 = s1[K] | s2[K];
 *                          dy_out (optional, ld lddy) receives f(A) for the weight-gradient kernel
 *   epilogue  0 none
 *             1 batch statistics of C: mean_out/var_out[N] (biased) and, if scale_out != NULL, the
 *               fold scale = gamma/sqrt(var+eps), shift = beta - mean*scale, running statistics
 *               (momentum, unbiased variance) and num_batches_tracked += 1
 *             2 BatchNorm-backward sums of the layer BELOW (C is its dL/d(activation), e_y its raw
 *               output [M,N]): e_s12 = sum_m gz | sum_m gz*xhat with that layer's e_scale/e_shift/
 *               e_mean/e_var/e_relu
 * partials_ws: spg_tc_gemm_max_partials() * N * 3 floats.  The reductions finish inside the kernel
 * (last CTA merges the per-CTA partials in a fixed order: deterministic).                          */
int spg_tc_gemm_max_partials(void);
int spg_tc_gemm_ex(const float* A, int64_t lda, const float* weight_image, const float* bias, float* C,
                   int64_t ldc, int64_t M, int N, int K,
                   const float* a_scale, const float* a_shift, int a_relu,
                   const float* a2, int64_t lda2, const float* a_mean, const float* a_var,
                   const float* a_s12, float a_eps, float* dy_out, int64_t lddy,
                   int epilogue, float* partials_ws,
                   float* mean_out, float* var_out, const float* gamma, const float* beta, float eps,
                   float* scale_out, float* shift_out, float* running_mean, float* running_var,
                   int64_t* num_batches_tracked, float momentum,
                   const float* e_y, int64_t e_ldy, const float* e_scale, const float* e_shift,
                   const float* e_mean, const float* e_var, float e_eps, int e_relu, float* e_s12,
                   spg_stream_t stream);

/* Weight gradient of a point-wise layer on the tensor cores (3xTF32, fp32-equivalent):
 *   dW[co,ci] = sum_m dY[m,co] * f(P)[m,ci],  f = affine(p_scale,p_shift)+ReLU of P's producer.
 * co in {64,128,256}, ci in {32,64,128}; every CTA reduces a slab of points into a partial held in
 * registers, workspace >= spg_tc_dw_ctas(M)*co*ci floats, partials are summed in a fixed order.
 * C[M,N] = sum_z partials[z,M,N] (+ bias) is also exported on its own (spg_splitk_reduce).       */
int spg_tc_dw_supported(int64_t M, int co, int ci);
int spg_tc_dw_ctas(int64_t M);
int spg_tc_dw(const float* dY, int64_t lddy, const float* P, int64_t ldp, const float* p_scale,
              const float* p_shift, int p_relu, float* dW, float* workspace, int64_t M, int co, int ci,
              spg_stream_t stream);
int spg_splitk_reduce(const float* partials, int split, int64_t M, int64_t N, const float* bias,
                      float* C, int64_t ldc, spg_stream_t stream);

/* Chunks of the per-column partials of spg_colsum and spg_act_bwd_reduce (workspace bound). */
int64_t spg_colstats_chunks(int64_t M);
/* BatchNorm fold of batch statistics mean[C], biased var[C]:
 * scale = gamma/sqrt(var+eps), shift = beta-mean*scale; if running_* non-NULL:
 * running = (1-momentum)*running + momentum*{mean, var*M/(M-1)}; if num_batches_tracked
 * (int64 scalar, device) is non-NULL it is incremented by one.  ref: nn.BatchNorm1d in training
 * mode (learning/pointnet.py:31,43,87,103; learning/graphnet.py:29).              */
int spg_bn_fold(const float* mean, const float* var, const float* gamma, const float* beta,
                float eps, float* scale, float* shift, float* running_mean, float* running_var,
                int64_t* num_batches_tracked, float momentum, int64_t M, int C,
                spg_stream_t stream);
/* out[m,c] = drop(f(Y[m,c]*scale[c]+shift[c])); scale/shift may be NULL; drop: see below. */
int spg_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* out, int64_t ldo, int64_t M, int C, float p, const int64_t* drop_slot,
                   spg_stream_t stream);
/* Column sums: out[c] = sum_m X[m,c]; workspace >= C*spg_colstats_chunks(M).      */
int spg_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* workspace,
               spg_stream_t stream);
/* Backward of a = drop(relu?(bn?(y))):
 *   pass 1 (spg_act_bwd_reduce, BN layers only): s12 = [s1 | s2] (2*C floats),
 *       s1[c] = sum_m g*mask, s2[c] = sum_m g*mask*xhat       (= d_beta, d_gamma)
 *       workspace >= 2*C*spg_colstats_chunks(M) floats
 *   pass 2 (spg_act_bwd_apply): dY = scale*(g*mask - s1/M - xhat*s2/M)   (BN)
 *                               dY = g*mask                             (no BN)
 *   g = drop'(G); mask = (y*scale+shift > 0) if relu else 1; xhat = (y-mean)*rstd; in-place OK;
 *   in apply, Y may be NULL without relu and BN.
 * drop: with drop_slot == NULL the identity (p ignored); otherwise training-mode dropout with the mask of
 * `drop_slot` (below): drop(a) = a*m/(1-p) and drop'(G) = G*m/(1-p), as a select, so that p >= 1 or an
 * infinite G gives 0.                                                                              */
int spg_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, float* s12, float* workspace,
                       int64_t M, int C, float p, const int64_t* drop_slot, spg_stream_t stream);
int spg_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                      const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, int has_bn, const float* s1,
                      const float* s2, float* dY, int64_t lddy, int64_t M, int C, float p,
                      const int64_t* drop_slot, spg_stream_t stream);

/* ------------------------------------------------------------ dropout     */
/* Training-mode nn.Dropout(p) directly after a layer's [BatchNorm][ReLU] (ref: learning/pointnet.py:
 * 109-110, learning/graphnet.py:54-55).  Element (m, c) of an [M, C] activation, i = m*C + c, is kept iff
 * word i&3 of Philox4x32-10(counter = (i>>2 low 32 bits, i>>34, ctr_lo, ctr_hi), key = (seed_lo,
 * seed_hi)) is >= floor(p * 2^32); kept elements are scaled by 1/(1-p); p >= 1 drops every element.  The
 * mask depends on (seed, ctr, i) only; it is its own stream, not the bits of the reference's nn.Dropout.
 * `slot` is an int64[2] (seed, ctr) in device memory.  The masked forward and backward are
 * spg_affine_act / spg_act_bwd_reduce / spg_act_bwd_apply with a drop_slot.                           */
/* slot = (state[0] ^ key_xor, state[1]); state[1] += 1.  state: the device's int64[2] (seed, counter);
 * key_xor folds a data-parallel rank into the key (0 on one GPU).                                     */
int spg_dropout_rng_next(int64_t* state, int64_t* slot, int64_t key_xor, spg_stream_t stream);
/* mask[m*C+c] = 1 if element (m, c) is kept, else 0 (uint8, [M, C] contiguous).                       */
int spg_dropout_mask(const int64_t* slot, float p, int64_t M, int C, uint8_t* mask, spg_stream_t stream);

/* ------------------------------------------------------------ PointNet    */
/* clouds [B,F,L] (the reference's NCL layout, learning/spg.py:162) -> rows [B*L, ld]
 * (point-major, channel contiguous, zero padded to ld).  If T [B,2,2] is given the
 * first two channels are replaced by (xy^T * T')^T with T' = T (+ I if add_eye: the STN's
 * "+ identity", ref: learning/pointnet.py:61,121-124).                                   */
int spg_cloud_rows(const float* clouds, const float* T, int add_eye, float* rows, int64_t ld,
                   int64_t B, int F, int L, spg_stream_t stream);
/* Segmented max-pool over point rows Y [rows, ldy] (ref: learning/pointnet.py:126, max_pool1d over each
 * superpoint's points).  The segments are described by (B, L, offsets):
 *   offsets NULL: B segments of fixed length L, segment b is rows [b*L, (b+1)*L) (the reference's
 *     layout: its loader resamples every superpoint to ptn_npts points, learning/spg.py:209-214);
 *   offsets int64 [B+1]: segment b is rows [offsets[b], offsets[b+1]) (ragged CSR superpoints, without
 *     that resampling); L is ignored; a segment holds fewer than 2^31 rows.
 * The row-wise backward entries also take row_seg int32 [rows] = segment of each row (required with
 * offsets, ignored without) and the total row count (B*L for fixed length).
 * pooled[b,c] = max over segment b of f(Y[r,c]*scale[c]+shift[c]), f = relu or identity; argmax[b,c] =
 * index WITHIN the segment of the first maximiser; an empty segment gives pooled 0 and argmax -1.
 * Writes into pooled with leading dimension ldp (so that the "global" features can sit in the same row,
 * ref: learning/pointnet.py:126-132).                                                                  */
int spg_segmax_fwd(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* pooled, int64_t ldp, int32_t* argmax, int64_t B, int L, const int64_t* offsets,
                   int C, spg_stream_t stream);
/* G[r,c] = g_pooled[b,c] if row r is the argmax of its segment b, else 0 (all rows of G written).      */
int spg_segmax_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, float* G,
                   int64_t ldG, int64_t B, int L, const int64_t* offsets, const int32_t* row_seg,
                   int64_t rows, int C, spg_stream_t stream);
/* Max-pool backward fused with the BatchNorm(+ReLU) backward of the layer Y that fed the pool:
 * s12 = [s1|s2] (= d_beta | d_gamma, 2*C floats, statistics over all rows) and dY[rows,C] are produced
 * straight from the pooled gradient and the argmax; the dense gradient of the pooled activation is never
 * materialised.  workspace >= 2*C*ceil(B/256) floats.  C % 4 == 0.                                     */
int spg_segmax_bn_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, const float* Y,
                      int64_t ldy, const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, float* s12, float* dY, int64_t lddy,
                      float* workspace, int64_t B, int L, const int64_t* offsets, const int32_t* row_seg,
                      int64_t rows, int C, spg_stream_t stream);
/* GroupNorm(groups, C) + [ReLU] + [training-mode dropout] over the segments (B, L, offsets) of point rows
 * Y [rows, ldy], segments as in spg_segmax_fwd (an FC layer's rows are B segments of L = 1).  The
 * statistics of (segment b, group g) run over the rows of b and the C/groups columns of g, biased variance:
 *   forward:  mean[b,g] = mean[b,g,0] + mean[b,g,1] ([B, groups, 2]: a float pair, so that a mean that is
 *             large against the spread keeps its precision), rstd[b,g] = 1/sqrt(var + eps) ([B, groups]);
 *             both 0 for an empty segment;
 *             out[r,c] = drop(f((Y[r,c] - mean)*rstd*gamma[c] + beta[c])), f = relu or identity
 *   backward: from G = dL/d(out): g = relu'(.)*drop'(G), gh = g*gamma, xhat = (Y - mean)*rstd,
 *             dY = rstd*(gh - mean(gh) - xhat*mean(gh*xhat)) (means over the segment's group),
 *             dbg = [d_beta | d_gamma] (2*C floats) = [sum g | sum g*xhat] over all rows;
 *             workspace >= 2*C*spg_group_norm_partials(B) floats
 * drop as in spg_affine_act (mask index r*C + c).  gamma and beta are required (affine GroupNorm); C <= 1024.
 * Deterministic: fixed-order sums, no atomics.
 * ref: learning/pointnet.py:32-35,44-47,88-91,104-107 (nn.GroupNorm(1, C) for norm='layer',
 * nn.GroupNorm(n_group, C) for norm='group').                                                          */
int64_t spg_group_norm_partials(int64_t B);
int spg_group_norm_fwd(const float* Y, int64_t ldy, const float* gamma, const float* beta, float eps, int relu,
                       float* out, int64_t ldo, float* mean, float* rstd, int64_t B, int L,
                       const int64_t* offsets, int C, int groups, float p, const int64_t* drop_slot,
                       spg_stream_t stream);
int spg_group_norm_bwd(const float* G, int64_t ldg, const float* Y, int64_t ldy, const float* mean,
                       const float* rstd, const float* gamma, const float* beta, int relu, float* dY,
                       int64_t lddy, float* dbg, float* workspace, int64_t B, int L, const int64_t* offsets,
                       int C, int groups, float p, const int64_t* drop_slot, spg_stream_t stream);
/* dT[b,i,j] = sum_l xy[b,i,l] * dXrows[b*L+l, j], i,j in {0,1}; clouds is the raw
 * [B,F,L] input, dXrows has leading dimension ld.                                    */
int spg_stn_apply_bwd(const float* clouds, const float* dXrows, int64_t ld, float* dT, int64_t B,
                      int F, int L, spg_stream_t stream);
/* Row gather / scatter between the [Nv,C] PointNet output and the zero-filled [N,C]
 * descriptors (ref: learning/pointnet.py:156-157): dst[idx[i],:] = src[i,:] and back. */
int spg_rows_scatter(const float* src, const int64_t* idx, float* dst, int64_t n_src, int C,
                     spg_stream_t stream);
int spg_rows_gather(const float* src, const int64_t* idx, float* dst, int64_t n_dst, int C,
                    spg_stream_t stream);

/* ---------------------------------------------------------------- step    */
/* Weighted cross entropy with ignore_index (mean reduction = sum w_y*nll / sum w_y),
 * ref: learning/main.py:205.  loss_out[0] = loss, d_logits [n,C] = dloss/dlogits.
 * class_weight may be NULL.  workspace: 16 bytes, 8-byte aligned (zeroed by the call).  */
int spg_ce_loss(const float* logits, const int64_t* target, const float* class_weight,
                int64_t ignore_index, float* loss_out, float* d_logits, float* workspace,
                int64_t n_rows, int C, spg_stream_t stream);
/* One fused pass over the flat parameter/gradient buffers (ref: learning/main.py:210-213):
 *   g = clamp(g*grad_scale, -clip, clip) (clip<=0: no clamp); g += wd*p; Adam(m,v,step).  */
int spg_clamp_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                   int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                   float grad_clip, float grad_scale, int64_t step, spg_stream_t stream);

/* Same update, step count kept in device memory (*step_counter is read as step-1 and incremented
 * by the call): nothing step-dependent is baked into launch parameters, so the whole training
 * step can be captured in a CUDA graph and replayed.                                          */
int spg_clamp_adam_dev(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                       float lr, float beta1, float beta2, float eps, float weight_decay,
                       float grad_clip, float grad_scale, int64_t* step_counter,
                       spg_stream_t stream);

/* ------------------------------------------- either side of the path (SURVEY 8(f))  */
/* Batch loader, per-superpoint part (ref: learning/spg.py:198-236 load_superpoint,
 * :238-260 augment_cloud, stacked as cloud.T by loader :146-166).  The parsed points of
 * the resident superpoints are one packed array points[rows, ldp] (columns as the
 * reference's parsed files: xyz 0-2, rgb 3-5, e 6, lpsv 7-10, XYZ 11-13, d 14).
 * For cloud i of n_clouds:
 *   rows   = points[sp_start[i] + sample_idx[i, j]], j < n_points   (sample_idx NULL: the
 *            first min(count, L) points as they are, the rest drawn on the device)
 *   xyz    = xyz - mean(xyz) (sequential fp32 column sums, as numpy); if normalize:
 *            diameter = max_k (max xyz_k - min xyz_k); xyz /= fp32(diameter + 1e-10)
 *   out[f] = column columns[f] (columns < 3: the centred xyz)
 *   out[0..2] = out[0..2] . xform[i]^T (double, rounded once) if xform != NULL
 *   out   += jitter[i, j, f]  if jitter != NULL; else clip(jitter_sigma*N(0,1), +-jitter_clip)
 *            from a counter-based generator keyed by `seed` if jitter_sigma > 0
 *   clouds[i, f, j] = out[j, f];  diameters[i] = diameter (0 if !normalize)
 * With host-provided sample_idx (and jitter) the result is bit-identical to the reference.  */
int spg_cloud_build(const float* points, int64_t ldp, const int64_t* sp_start,
                    const int32_t* sp_count, const int32_t* sample_idx, const int32_t* columns,
                    int n_attribs, int n_points, int normalize, const double* xform,
                    const float* jitter, float jitter_sigma, float jitter_clip, int64_t seed,
                    float* clouds, float* diameters, int64_t n_clouds, spg_stream_t stream);
/* Device-side builder of the graph views the ECC kernels read, from the collated (idxn, degs) pair of
 * ref: learning/ecc/GraphConvInfo.py:48-69 (set_batch leaves idxn = source node per edge with the edges
 * sorted by target, degs = in-degree per target; the reference uploads both, GraphConvInfo.py:71-77):
 *   idxn32 [E] = int32(idxn); tgt_rowptr [n_out+1] = exclusive scan of degs; edge_tgt [E] = target of each
 *   edge; src_perm [E] = the STABLE permutation sorting the edges by source (identical to numpy
 *   argsort(kind="stable")); src_rowptr [n_in+1] = first position of each source in that order.
 * status [1] (device int32) receives a bit mask: 1 = idxn out of [0,n_in), 2 = a degree out of range,
 * 4 = sum(degs) != E; the outputs are undefined when it is non-zero.  workspace: 256-byte aligned,
 * spg_graph_build_workspace() bytes.  All int64 inputs and int32 outputs are device pointers.           */
int spg_graph_build_workspace(int64_t n_out, int64_t n_in, int64_t n_edges, int64_t* bytes);
int spg_graph_build(const int64_t* idxn, const int64_t* degs, int64_t n_out, int64_t n_in, int64_t n_edges,
                    int32_t* idxn32, int32_t* tgt_rowptr, int32_t* edge_tgt, int32_t* src_rowptr,
                    int32_t* src_perm, int32_t* status, void* workspace, int64_t workspace_bytes,
                    spg_stream_t stream);
/* Evaluation bookkeeping (ref: learning/main.py:257-262,297-305 + metrics.py:16-18):
 * pred_i = first argmax of logits[i,:]; for nodes with label_mode[i] != -100:
 * confusion[:, pred_i] += label_vec[i,:], counters[0] += 1, counters[1] += (pred_i == label_mode[i]).
 * confusion [C,C] and counters [2] are int64 device arrays accumulated across calls (caller zeroes
 * them); pred_out [n] (may be NULL) receives every node's prediction.                        */
int spg_confusion_count(const float* logits, int64_t ld_logits, const int64_t* label_mode,
                        const int64_t* label_vec, int64_t ld_vec, int64_t* confusion,
                        int64_t* counters, int64_t* pred_out, int64_t n_nodes, int n_classes,
                        spg_stream_t stream);
/* The step's only collective fused with the optimizer (ref: learning/main.py:210-213 on the averaged
 * gradient; SURVEY.md 8(e)): one-shot all-reduce over NVLink peer memory + 1/world + element-wise clamp
 * + Adam in ONE kernel.  grad: this rank's flat gradient (local memory, n floats, 16-byte aligned);
 * peer_stage: DEVICE array of `world` pointers to the ranks' symmetric staging buffers of
 * spg_allreduce_stage_floats(n) floats (two halves, used alternately: no "done reading" handshake);
 * peer_flags: DEVICE array of `world` pointers to zero-initialised symmetric uint32 buffers of
 * spg_allreduce_flag_words(world) words; local_state: 2 zero-initialised uint32 words in local device
 * memory (launch epoch, block ticket); step_counter as in spg_clamp_adam_dev.  All ranks must call it once
 * per step, in the same order.  The sum runs in rank order: bit-identical on every rank.            */
int spg_allreduce_flag_words(int world);
int64_t spg_allreduce_stage_floats(int64_t n);
int spg_allreduce_clamp_adam(const float* grad, float* const* peer_stage, uint32_t* const* peer_flags, int rank,
                             int world, float* param, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                             float beta1, float beta2, float eps, float weight_decay, float grad_clip,
                             float grad_scale, int64_t* step_counter, uint32_t* local_state, spg_stream_t stream);
/* Eval-mode PointNet trunk, fully fused (ref: learning/pointnet.py:55-61,120-127 under model.eval()):
 * for every superpoint b (n_points must be 128 = one tensor-core M tile, n_features <= 16):
 *   x = clouds[b] ([F, 128], NCL as the reference stacks them, learning/spg.py:162)
 *   if T: (x0, x1) <- (x0, x1) (T[b] (+ I))                                   (pointnet.py:123)
 *         (T needs n_features >= 2: T with a single feature is SPG_E_BADARG)
 *   for l < n_layers: x <- relu(W_l x + b_l)     W_l [widths[l], K_l], BatchNorm already folded in
 *   pooled[b, :widths[n_layers-1]] = max over the 128 points
 * Activations stay in shared memory; the input tile and the weight stream arrive by TMA;
 * products are 3xTF32 on wgmma (fp32-equivalent).  weight_image = for each layer the
 * spg_tc_pack_weights_scaled image ([K_l/32][hi|lo][N_l][32 floats]; K_0 = 32, k_valid = F) back to
 * back (spg_pointnet_fused_image_rows(...) * 32 floats); bias = the folded biases back to back;
 * widths: HOST int32 array, every width in {32,64,128,256}, inner widths <= 128, at most 6 layers.   */
int spg_pointnet_fused_supported(int n_features, int n_points, int n_layers, const int32_t* widths);
int64_t spg_pointnet_fused_image_rows(int n_features, int n_layers, const int32_t* widths);
int spg_pointnet_fused_eval(const float* clouds, int64_t n_clouds, int n_features, int n_points, const float* T,
                            int add_eye, const float* weight_image, const float* bias, int n_layers,
                            const int32_t* widths, float* pooled, int64_t ldp, spg_stream_t stream);
/* bf16 arithmetic for the same trunk (BASELINE configs[3]): bf16 operands, fp32 accumulation in registers
 * (wgmma bf16, one MMA per product), activations between layers as bf16 on chip; inputs
 * fp32 [B,F,128], pooled output fp32.  weight_image: per layer [K_l/64][N_l][64] bf16 from
 * spg_tc_pack_weights_bf16 (K_0 = 64 with k_valid = F; a layer that follows a 32-wide one has K = 64 with
 * k_valid = 32).  Agreement with the fp32 path is bounded by bf16 rounding (~1e-2), not 1e-4.          */
int64_t spg_pointnet_fused_bf16_image_rows(int n_features, int n_layers, const int32_t* widths);
int spg_tc_pack_weights_bf16(const float* W, int64_t ldw, const float* row_scale, int N, int K, int k_valid,
                             void* image, spg_stream_t stream);
int spg_pointnet_fused_eval_bf16(const float* clouds, int64_t n_clouds, int n_features, int n_points, const float* T,
                                 int add_eye, const void* weight_image, const float* bias, int n_layers,
                                 const int32_t* widths, float* pooled, int64_t ldp, spg_stream_t stream);
/* clouds_grad[b,f,l] = rows_grad[b*L+l, f]: the input gradient of a PointNet without an internal transformer
 * back in the reference's [B,F,L] layout (autograd of learning/pointnet.py:126 w.r.t. its input; needed by
 * LocalCloudEmbedder, whose external STN is trained through it, pointnet.py:189-207).                    */
int spg_rows_to_clouds(const float* rows, int64_t ld, float* clouds, int64_t B, int F, int L,
                       spg_stream_t stream);
/* Ragged superpoints (north_star: CSR offset array instead of the reference's resample-to-ptn_npts,
 * learning/spg.py:209-214): point rows [P, ld] of all superpoints back to back, offsets int64 [B+1]; the
 * max-pool is spg_segmax_* with offsets.
 *   spg_rows_xy_transform(+_bwd): columns 0,1 of every row times its segment's 2x2 T (+I)
 *     (learning/pointnet.py:123), row_seg int32 [P] = segment of each row; backward: dT [B,4].        */
int spg_rows_xy_transform(const float* rows_in, const float* T, int add_eye, const int32_t* row_seg,
                          float* rows_out, int64_t P, int64_t ld, spg_stream_t stream);
int spg_rows_xy_transform_bwd(const float* rows_in, int64_t ld, const float* d_rows_out, int64_t ld_d,
                              const int64_t* offsets, float* dT, int64_t B, spg_stream_t stream);
/* Label up-sampling, the step after the path (ref: partition/provider.py:630-635,676-682):
 * spg_labels_to_points: labels_full[n_ver] (uint8, zero-initialised here) gets labels_red[c] at every
 *   member point of component c; comp_ptr int64 [n_components+1] is the CSR over point_ids.
 * spg_nn1_interpolate: exact 1-nearest-neighbour transfer (squared Euclidean distance in float64, ties
 *   to the lowest index) from the n_ref pruned points to the n_query points; writes the neighbour's
 *   label (int64) and/or its index (int32).                                                       */
int spg_labels_to_points(const int64_t* labels_red, const int64_t* comp_ptr, const int64_t* point_ids,
                         int64_t n_components, uint8_t* labels_full, int64_t n_ver, spg_stream_t stream);
int spg_nn1_interpolate(const float* xyz_ref, int64_t n_ref, const float* xyz_query, int64_t n_query,
                        const int64_t* labels_ref, int64_t* labels_out, int32_t* nn_index_out,
                        spg_stream_t stream);

/* ------------------------------------------- learned partition (supervized_partition/losses.py)
 * Edge arrays src/tgt are int64 [E] device arrays; is_transition is uint8 [E] (0 = intra, 1 = inter);
 * pred_in_component int64 [V].  Endpoints outside [0, V) are skipped (never read).  No float atomics:
 * every float output is bit-reproducible.
 * spg_lp_workspace: bytes of the scratch (`workspace`, 256-byte aligned) of spg_lp_incidence, spg_lp_xpart
 * and spg_lp_seal for up to n_ver vertices, n_edges edges and n_comp components; a call whose own counts
 * need more than workspace_bytes returns SPG_E_BADARG.                                                  */
int spg_lp_workspace(int64_t n_ver, int64_t n_edges, int64_t n_comp, int64_t* bytes);
/* Per-vertex incidence CSR of the edge endpoints: entry j < E is the source side of edge j, j >= E the
 * target side of edge j - E; rowptr [V+1], entry [2E] sorted by vertex, stably (by j within a vertex).
 * No reference counterpart: the gather CSR of the deterministic backward of compute_dist
 * (ref: supervized_partition/losses.py:31-42 under autograd).                                         */
int spg_lp_incidence(const int64_t* src, const int64_t* tgt, int64_t n_ver, int64_t n_edges, int32_t* rowptr,
                     int32_t* entry, void* workspace, int64_t workspace_bytes, spg_stream_t stream);
/* diff[e] from embeddings emb [V, D] (dist_type 0 = euclidian: |x_s - x_t|^2, 1 = intrinsic:
 * (acos(0.999 x_s.x_t) - acos(0.999)) / (acos(-0.999) - acos(0.999)) * 3.141592, 2 = scalar: x_s.x_t - 1),
 * fp64 inside; coef [E] (intrinsic, scalar; may be NULL for euclidian) = d diff / d (x_s.x_t).
 * Backward: gemb [V, D] = dL/demb from gdiff [E], gathered through the incidence CSR.
 * ref: supervized_partition/losses.py:31-42                                                              */
int spg_lp_dist_fwd(const float* emb, int64_t n_ver, int D, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                    int dist_type, float* diff, float* coef, spg_stream_t stream);
int spg_lp_dist_bwd(const float* emb, int64_t n_ver, int D, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                    int dist_type, const float* coef, const float* gdiff, const int32_t* rowptr, const int32_t* entry,
                    float* gemb, spg_stream_t stream);
/* compute_loss: loss [2] = (sum over is_transition == 0 of the intra term, sum over is_transition == 1 of
 * the inter term), fp64 sums over spg_lp_loss_partials() fixed blocks (partials: 2 doubles per block),
 * merged in a fixed order.  intra: 0 = tv w*sqrt(d+1e-10), 1 = laplacian w*d, 2 = TVH
 * 0.2*w*(sqrt(1+d/0.04)-1); inter: 0 = zhang clamp(w*(beta - sqrt(d+1e-10)), min=0) (beta = 1.0471975512 for
 * dist_type 1, else 1), 1 = TVminus w*sqrt(d+1e-10), -1 = none (loss[1] = 0).
 * Backward: gdiff [E] from gloss [2] (device).  ref: supervized_partition/losses.py:24-29,44-64          */
int64_t spg_lp_loss_partials(void);
int spg_lp_loss_fwd(const float* diff, const float* weights, const uint8_t* is_transition, int64_t n_edges,
                    int intra, int inter, int dist_type, double* partials, float* loss, spg_stream_t stream);
int spg_lp_loss_bwd(const float* diff, const float* weights, const uint8_t* is_transition, int64_t n_edges,
                    int intra, int inter, int dist_type, const float* gloss, float* gdiff, spg_stream_t stream);
/* crosspartition weights: connected components of the edges with is_transition == 0 and
 * pred_in_component[s] == pred_in_component[t] (components numbered by their smallest vertex:
 * in_component_x [V], comp_size [V] (first n_comp used), n_comp [1]); every transition edge between
 * components (c1, c2) gets 1 + min(|c1|, |c2|) / #(transition edges between c1 and c2) * transition_factor
 * (fp64, rounded once), every other edge 1.
 * ref: supervized_partition/losses.py:130-158 (+ partition/ply_c/connected_components.cpp:17-110, cutoff 0) */
int spg_lp_xpart(const int64_t* src, const int64_t* tgt, const uint8_t* is_transition,
                 const int64_t* pred_in_component, int64_t n_ver, int64_t n_edges, double transition_factor,
                 float* weights, int32_t* in_component_x, int32_t* comp_size, int32_t* n_comp, void* workspace,
                 int64_t workspace_bytes, spg_stream_t stream);
/* SEAL weights: w[c] = |c| - (frequency of the most common object id in c) for the n_comp predicted
 * components (objects: int64 [V], 0 <= id < 2^32); transition edges get 1 + max(w[c_s], w[c_t]) *
 * transition_factor (fp64, rounded once), others 1; w_per_component [n_comp] (may be NULL).
 * ref: supervized_partition/losses.py:119-128,168-173                                                    */
int spg_lp_seal(const int64_t* src, const int64_t* tgt, const uint8_t* is_transition, const int64_t* pred_in_component,
                const int64_t* objects, int64_t n_ver, int64_t n_edges, int64_t n_comp, double transition_factor,
                float* weights, int32_t* w_per_component, void* workspace, int64_t workspace_bytes,
                spg_stream_t stream);
/* weights[e] = is_transition[e] != 0 ? w_transition : w_other ('none', 'proportional';
 * ref: supervized_partition/losses.py:96-101)                                                            */
int spg_lp_fill_weights(const uint8_t* is_transition, int64_t n_edges, float w_other, float w_transition,
                        float* weights, spg_stream_t stream);
/* counts [2] (int64, device) = (#(truth != 0 and pred != 0), #(truth != 0)); pred may be NULL (counts[0] = 0).
 * For 0/1 masks these are the numerator and denominator of compute_boundary_recall(truth, pred) and, with
 * the arguments swapped, of compute_boundary_precision.  ref: learning/metrics.py:87-92                  */
int spg_lp_count(const uint8_t* truth, const uint8_t* pred, int64_t n, int64_t* counts, spg_stream_t stream);
/* cut pursuit's edge weights (double [E]): threshold > 0: diff > 1 ? (float)threshold : 1; threshold < 0:
 * expf(diff * (float)threshold) / exp(threshold); 0: 1.  ref: supervized_partition/losses.py:68-72        */
int spg_lp_edge_weight(const float* diff, int64_t n_edges, double threshold, double* edge_weight,
                       spg_stream_t stream);
/* relax_edge_binary in place on relaxed [E] (uint8 0/1), `tolerance` rounds of: mark the endpoints of the
 * set edges (vertex_mark uint8 [V]); set edge 0 if some edge's source is unmarked and edge 1 if some edge's
 * source is marked (losses.py:184 indexes with the mark values); set every edge whose target is marked.
 * hit: int32 scratch; status [1] = 1 if edge 1 was needed but E == 1 (numpy raises IndexError).
 * ref: supervized_partition/losses.py:175-186                                                            */
int spg_lp_relax(uint8_t* relaxed, const int64_t* src, const int64_t* tgt, int64_t n_ver, int64_t n_edges,
                 int tolerance, uint8_t* vertex_mark, int32_t* hit, int32_t* status, spg_stream_t stream);
/* pred [V] (int64, zeroed here) = for the members (point_ids[comp_ptr[c]:comp_ptr[c+1]]) of every component c
 * the first argmax over k of the int64 sum of labels[v, 1 + k], k < n_classes (labels int64 [V, ld_labels]).
 * ref: partition/provider.py:689-695                                                                     */
int spg_lp_perfect_prediction(const int64_t* comp_ptr, const int64_t* point_ids, int64_t n_comp,
                              const int64_t* labels, int64_t ld_labels, int n_classes, int64_t n_ver, int64_t* pred,
                              spg_stream_t stream);

/* ---------------------------------------------------------------- learned-partition batch builder
 * graph_loader + graph_collate of the learned-embedding branch, one call per file of the batch, each writing
 * that file's slice of the collated outputs.  ref: supervized_partition/graph_processing.py:347-472,534-546.
 *
 * lp_augment: rgb_out [n, 3] = rgb / 255; xyz_out [n, 3] = xyz, or with rot (device float [9]: the float32
 * rotation M row-major) ((p - ref) M) + ref with ref = (x, y, 0) of vertex ref_index and p = xyz with the z
 * of vertex ref_index set to 0 (the reference's ref_point is a view of xyz).  Then jitter: xyz_out += noise and,
 * with rgb_jitter, rgb_out = clip(rgb_out + noise, -1, 1); the noise is noise_xyz / noise_rgb [n, 3] (host
 * draws, already clipped) or, with device_noise, clip(sigma N(0, 1), -clip, clip) from Philox4x32-10 keyed by
 * seed, counter (vertex, file_pos, 0 for xyz / 1 for rgb).  No jitter when both are absent, and then
 * rgb_jitter is ignored (rgb is jittered only with xyz).
 * ref: graph_processing.py:353,534-546                                                                    */
int spg_lp_augment(const float* xyz, const float* rgb, int64_t n_ver, const float* rot, int64_t ref_index,
                   const float* noise_xyz, const float* noise_rgb, int device_noise, int rgb_jitter, float sigma,
                   float clip, int64_t seed, int64_t file_pos, float* xyz_out, float* rgb_out, spg_stream_t stream);
/* lp_subgraph_select: with a vertex mask [n] (uint8), new_index [n + 1] = exclusive scan of the mask (the new
 * id of every kept vertex, the kept count last), selected [count] = the kept vertices in increasing order,
 * edge_pos [E + 1] = exclusive scan of the edge mask mask[src] * mask[tgt] (the kept edge count last).
 * object_max [1] = max over the kept vertices (every vertex without a mask) of objects, as the uint32
 * id ^ 0x80000000.  Workspace from spg_lp_subgraph_workspace, 256-byte aligned.
 * ref: graph_processing.py:371-385, partition/ply_c/random_subgraph.cpp:91-95                            */
int spg_lp_subgraph_workspace(int64_t n_ver, int64_t n_edges, int64_t* bytes);
int spg_lp_subgraph_select(const uint8_t* mask, const int32_t* objects, int64_t n_ver, const int32_t* src,
                           const int32_t* tgt, int64_t n_edges, int32_t* new_index, int32_t* selected,
                           int32_t* edge_pos, uint32_t* object_max, void* workspace, int64_t workspace_bytes,
                           spg_stream_t stream);
/* lp_subgraph_edges: the kept edges in their order (all edges when new_index is NULL), renumbered through
 * new_index and shifted by vertex_offset (graph_collate :464-465), with their is_transition.
 * ref: graph_processing.py:378-381,457-465                                                               */
int spg_lp_subgraph_edges(const int32_t* src, const int32_t* tgt, const uint8_t* is_transition, int64_t n_edges,
                          const int32_t* new_index, const int32_t* edge_pos, int64_t vertex_offset, int64_t* src_out,
                          int64_t* tgt_out, uint8_t* is_transition_out, spg_stream_t stream);
/* lp_object_offsets: offsets [B] = running sum of the object maxima of the earlier files (max, not max + 1,
 * as graph_collate); a file with counts[b] == 0 kept vertices adds 0.  ref: graph_processing.py:447,467   */
int spg_lp_object_offsets(const uint32_t* object_max, const int64_t* counts, int64_t n_files, int64_t* offsets,
                          spg_stream_t stream);
/* lp_local_clouds: for every kept vertex i (v = selected[i], or i when NULL) with its k first neighbours
 * u_j = local_geometry[v, j] (original ids): diameter = sqrt((var_x + var_y) + var_z) of xyz[u_j] (numpy's
 * sequential fp32 mean and variance), clouds [n_sel, 3 + 3 use_rgb, k] = (xyz[u_j] - xyz[v]) / (diameter +
 * 1e-10) and rgb[u_j]; clouds_global [n_sel, ld_global] = [diameter | elevation (flag 1) | rgb[v] (2) |
 * xyn[v] (4) | xyz[v, :2] (8)]; xyz_out [n_sel, 3], labels_out [n_sel, n_label_cols] (int64),
 * objects_out [n_sel] = objects[v] + object_offset[0].  rgb_scale: rgb is the resident 0..255 array.
 * k <= 256.  ref: graph_processing.py:387-411,430                                                         */
int spg_lp_local_clouds(const float* xyz, const float* rgb, int rgb_scale, const int32_t* local_geometry,
                        int64_t ld_geometry, int k, const int32_t* selected, int64_t n_sel, const float* elevation,
                        const float* xyn, const int32_t* labels, int64_t n_label_cols, const int32_t* objects,
                        const int64_t* object_offset, int use_rgb, int global_flags, float* clouds,
                        float* clouds_global, int64_t ld_global, float* xyz_out, int64_t* labels_out,
                        int64_t* objects_out, spg_stream_t stream);

/* ---------------------------------------------------------------- k-NN graphs and geometric features
 * compute_graph_nn / compute_graph_nn_2 / compute_geof of the partition pipelines (ref: partition/graphs.py:11-70,
 * partition/ply_c/ply_c.cpp:384-462), xyz float32 [n, 3] on the device, n < 2^31 - 1.
 *
 * spg_knn_bounds: words [8] (device, uint32) = the order-preserving keys of the finite coordinates' minimum
 * (words 0-2) and maximum (3-5) per axis, status (6) = 1 if some coordinate is not finite.
 * spg_knn_grid: a grid of cubic cells of size `cell` from origin (ox, oy, oz), dim_* cells per axis (each
 * < 2^21, coordinates outside are clamped into the edge cells): the stable sort of the points by cell and the
 * occupied-cell table, into `workspace` (spg_knn_workspace bytes, 256-byte aligned); n_cells [1] (device) = the
 * number of occupied cells.  The grid only sets the work of the query, never its result.
 * spg_knn_query (same grid arguments and workspace): for every vertex i its k <= spg_knn_max_k() nearest other
 * vertices ranked by d2 = (dx dx + dy dy) + dz dz in float64 (dx = double(x_i) - double(x_j)), ties by the smaller
 * index; source, target [n k1] (int64) = i, the first k1 of them; distances [n k1] = float32(sqrt(d2));
 * target2 [n k] (may be NULL) = all k.  Needs n >= k + 1.
 * spg_geof: geof [n, 4] (float32, 16-byte aligned) = linearity, planarity, scattering, verticality of vertex i
 * and its k neighbours target[i k .. i k + k) (int64): fp64 mean and covariance / (k + 1), symmetric fp64
 * eigen-solve, eigenvalues sorted descending and clamped at 0, ply_c.cpp:436-446 in fp64 (NaN in all four where
 * the largest eigenvalue is 0); status [1] (device, uint32) = 2 and the row NaN where an id is outside [0, n). */
int spg_knn_max_k(void);
int spg_knn_workspace(int64_t n, int64_t* bytes);
int spg_knn_bounds(const float* xyz, int64_t n, uint32_t* words, spg_stream_t stream);
int spg_knn_grid(const float* xyz, int64_t n, double ox, double oy, double oz, double cell, int64_t dim_x,
                 int64_t dim_y, int64_t dim_z, void* workspace, int64_t workspace_bytes, int32_t* n_cells,
                 spg_stream_t stream);
int spg_knn_query(int64_t n, int k, int k1, double ox, double oy, double oz, double cell, int64_t dim_x,
                  int64_t dim_y, int64_t dim_z, const void* workspace, int64_t workspace_bytes, int64_t* source,
                  int64_t* target, float* distances, int64_t* target2, spg_stream_t stream);
int spg_geof(const float* xyz, int64_t n, const int64_t* target, int k, float* geof, uint32_t* status,
             spg_stream_t stream);

/* ---------------------------------------------------------------- superpoint graph
 * compute_sp_graph of the partition pipelines (ref: partition/graphs.py:75-210), xyz float32 [n, 3] and
 * in_component int64 [n] on the device, n < 2^31 - 1.
 *
 * spg_sp_scan: words [2] (device, int64) = max(in_component) + 1 (n_com) and a status (1: a non-finite
 * coordinate, 4: a negative id).
 * spg_sp_points (workspace: spg_sp_points_workspace bytes, 256-byte aligned; 1 <= n_com <= n): the points sorted
 * by (component, x, y, z) (-0 == +0), the unique rows of every component (ref: graphs.py:155 np.unique(axis=0));
 * centroids [n_com, 3] = numpy's mean of them (sequential fp32 sum in sorted order / u), the unique row itself
 * when u == 1; length, surface, volume [n_com] (float32) = 0 (u == 1), numpy's fp32 sqrt(sum(var)), 0, 0
 * (u == 2), ev0, sqrt(ev0 ev1 + 1e-10), sqrt(ev0 ev1 ev2 + 1e-10) of the fp64 covariance (ddof 1) in fp64
 * (u >= 3); point_count [n_com] (int64); sp_labels [n_com, n_label_cols] (int64) = label_mode 1: the histogram of
 * labels [n] over 0..n_labels (n_label_cols = n_labels + 1; other values not counted), 2: the sum of the rows of
 * labels [n, n_label_cols]; 0: none (labels and sp_labels may be NULL).  status [1] (device, uint32) = 8 where a
 * component below n_com holds no point.  ref: graphs.py:146-181
 * spg_sp_edges_count (workspace: spg_sp_edges_workspace(n_tets, 0) bytes): simplices [n_tets, 4] (int64 when
 * ids64, else int32); tet_offsets [n_tets + 1] (device, int32) = the exclusive scan of the directed vertex pairs of
 * every tetrahedron whose endpoints lie in different components, tet_offsets[n_tets] = n_cand, their total; status
 * [1] = 2 where an id is outside [0, n).  n_tets <= (2^31 - 2) / 12.  ref: graphs.py:86-106
 * spg_sp_edges_build (workspace: spg_sp_edges_workspace(n_tets, n_cand) bytes): the pairs deduplicated (ref:
 * graphs.py:108), those with float32 sqrt((dx dx + dy dy) + dz dz) < float32(d_max) kept when d_max > 0 (:110-112),
 * grouped by the exact 64-bit (source component, target component) key, ascending (:114-124); n_sedg [1] (device,
 * int64) = the number of superedges.
 * spg_sp_edges_features (the build's workspace, n_sedg read back): source, target [n_sedg] (int64);
 * delta_mean, delta_std (ddof 0) [n_sedg, 3] and delta_norm [n_sedg] of delta = xyz[u] - xyz[v] over the pairs, in
 * fp64 rounded once (one pair: its float32 delta, 0, its float32 norm); delta_centroid [n_sedg, 3] = fp32
 * centroid difference; length / surface / volume ratios = fp32 a / (b + 1e-6f); point_count_ratio =
 * float32(double(cs) / (double(ct) + 1e-6)).  ref: graphs.py:183-209                                         */
int spg_sp_scan(const float* xyz, const int64_t* in_component, int64_t n, int64_t* words, spg_stream_t stream);
int spg_sp_points_workspace(int64_t n, int64_t* bytes);
int spg_sp_points(const float* xyz, const int64_t* in_component, int64_t n, int64_t n_com, const int64_t* labels,
                  int label_mode, int64_t n_label_cols, int n_labels, void* workspace, int64_t workspace_bytes,
                  float* centroids, float* length, float* surface, float* volume, int64_t* point_count,
                  int64_t* sp_labels, uint32_t* status, spg_stream_t stream);
int spg_sp_edges_workspace(int64_t n_tets, int64_t n_cand, int64_t* bytes);
int spg_sp_edges_count(const int64_t* in_component, int64_t n, const void* simplices, int ids64, int64_t n_tets,
                       int32_t* tet_offsets, void* workspace, int64_t workspace_bytes, uint32_t* status,
                       spg_stream_t stream);
int spg_sp_edges_build(const float* xyz, const int64_t* in_component, int64_t n, const void* simplices, int ids64,
                       int64_t n_tets, const int32_t* tet_offsets, int64_t n_cand, double d_max, void* workspace,
                       int64_t workspace_bytes, int64_t* n_sedg, spg_stream_t stream);
int spg_sp_edges_features(const float* xyz, int64_t n_tets, int64_t n_cand, const void* workspace,
                          int64_t workspace_bytes, int64_t n_sedg, const float* centroids, const float* length,
                          const float* surface, const float* volume, const int64_t* point_count, int64_t* source,
                          int64_t* target, float* delta_mean, float* delta_std, float* delta_norm,
                          float* delta_centroid, float* length_ratio, float* surface_ratio, float* volume_ratio,
                          float* point_count_ratio, spg_stream_t stream);

/* ---------------------------------------------------------------- voxel pruning
 * prune of the partition pipelines (ref: partition/ply_c/ply_c.cpp:149-380; called at partition/partition.py:124,
 * supervized_partition/graph_processing.py:124,142 and, chunk by chunk, partition/provider.py:250-303), xyz float32
 * [n, 3] on the device, 1 <= n < 2^31 - 1.  chunk_rows = 0: one cloud; > 0: every chunk of chunk_rows consecutive
 * points is pruned on its own (its own minimum) and the voxels are stacked in chunk order.  One workspace of
 * spg_prune_workspace(n, chunk_rows) bytes (256-byte aligned) serves the three calls, in order.
 *
 * spg_prune_bounds: words [4] (device, int64) = status (1: a non-finite coordinate, 2: a bin of 2^32 or more, 4: a
 * label outside [0, n_labels], 8: an object outside [0, n_objects]) and the largest bin of x, y and z over the
 * chunks.  A bin is (uint32) floor((x - x_min) / voxel_size) in fp32, x_min the chunk's minimum.  labels and objects
 * (int64 [n]) are read only where the reference reads them: labels when n_labels > 0, objects when n_labels > 0 and
 * n_objects > 0.  ref: ply_c.cpp:305-331
 * spg_prune_voxels (max_bin_* from the bounds): the points stably sorted by (chunk, bin x, bin y, bin z), packed into
 * the fewest bits that hold them (two sorts beyond 64 bits); the voxels numbered in order of first touch in point
 * order (the reference's insertion order); n_voxels [1] (device, int64) = m.  ref: ply_c.cpp:326-336
 * spg_prune_reduce (m read back): xyz_out [m, 3] = the fp32 sum of the voxel's points in point order from 0.f /
 * (float) count; rgb_out [m, 3] (uint8) = (uint8)((float) uint32 sum / (float) count); labels_out [m, n_labels + 1]
 * and objects_out [m, n_objects + 1] (int64) = the histograms, zero where the reference counts nothing.
 * ref: ply_c.cpp:338-379                                                                                   */
int spg_prune_workspace(int64_t n, int64_t chunk_rows, int64_t* bytes);
int spg_prune_bounds(const float* xyz, int64_t n, int64_t chunk_rows, float voxel_size, const int64_t* labels,
                     int n_labels, const int64_t* objects, int n_objects, void* workspace, int64_t workspace_bytes,
                     int64_t* words, spg_stream_t stream);
int spg_prune_voxels(const float* xyz, int64_t n, int64_t chunk_rows, float voxel_size, int64_t max_bin_x,
                     int64_t max_bin_y, int64_t max_bin_z, void* workspace, int64_t workspace_bytes,
                     int64_t* n_voxels, spg_stream_t stream);
int spg_prune_reduce(const float* xyz, const uint8_t* rgb, const int64_t* labels, int n_labels,
                     const int64_t* objects, int n_objects, int64_t n, int64_t chunk_rows, const void* workspace,
                     int64_t workspace_bytes, int64_t n_voxels, float* xyz_out, uint8_t* rgb_out,
                     int64_t* labels_out, int64_t* objects_out, spg_stream_t stream);

/* ---------------------------------------------------------------- cut pursuit
 * libcp.cutpursuit of both partition pipelines (ref: partition/cut-pursuit/src/cutpursuit.cpp:77-105, speed 4;
 * spatial 0: CutPursuit_L2, 1: CutPursuit_SPG), one stage per call; spg_cut_pursuit.py runs the main loop.
 * n vertices, n_edges listed edges (each one an arc pair, duplicates kept), dim in [1, 32], 2 n_edges < 2^31 - 1.
 * One workspace of spg_cp_workspace(n, n_edges, dim) bytes (256-byte aligned) holds the whole state; every call
 * takes the same (n, n_edges, dim, workspace).  spg_cp_regions writes the byte offsets in the workspace of: obs,
 * comp (int32 [n]), root (int32), sat (uint8), label (uint8), colour (uint8: 0 source tree, 1 free, 4 sink tree),
 * active (uint8 [n_edges]), value, c0, c1 (float64 [n, dim]), cs, ct (float32 [n]), ecap (float32 [n_edges]),
 * members, offsets (int32), words (int64), dwords (float64), partner (int32 [n]), res (int64 [2 n_edges]: the
 * residual fixed-point capacities of the arcs), excess, rt (int64 [n]: excess and residual sink capacity), arc_off
 * (int32 [n + 1]), arc_dst, arc_rev, arc_edge (int32 [2 n_edges]: head, reverse arc and listed edge of every arc),
 * nw (float32 [n]: the vertex weights) and cw (float64 [n]: the component weights, sum of nw, as of the last value
 * computation).
 *
 * spg_cp_setup: out[0] (host) = status (1: a non-finite observation, 2: a non-finite edge weight, 4: an edge id
 *   outside [0, n)); when 0, the arc CSR, one component (root 0, its mean as value), no active edge, every vertex
 *   weight 1 (libcp.cutpursuit, cutpursuit.cpp:91).
 * spg_cp_node_weights (after spg_cp_setup; libcp.cutpursuit2, cutpursuit.cpp:107-128): copies node_weight [n]
 *   (device) as the vertex weights; out[0] (host) = status (8: a negative or non-finite weight); when 0, the one
 *   component's value = sum w x / sum w and weight = sum w (all weights 0: NaN value).  Every later stage weighs
 *   its sums, centres, terminal capacities, merge gains and energy by them (CutPursuit_SPG.h).
 * spg_cp_members: members / offsets = the vertices grouped by component, ascending.
 * spg_cp_kmeans: labels = 0, then 2-means per unsaturated component of >= 2 vertices (members current).
 * spg_cp_centers: c0 / c1 of every unsaturated component; L2 saturates a component with an empty side.
 * spg_cp_capacities: cs / ct / ecap, the reference's fp32 capacities (unary: the SPG step's weight).
 * spg_cp_maxflow: colour and labels from the minimal cuts; out[0] = push-relabel rounds.
 * spg_cp_activate: L2 saturation, edge activation; out[0] = vertices in saturated components.
 * spg_cp_split: the connected components of the non-active graph; out[0] = the new component count.
 * spg_cp_merge: one merge pass (is_cutoff: merge(true)); out[0] = merges, out[1] = the new component count.
 * spg_cp_energy: out[0..2] (host) = fidelity, active edge weight, fidelity + reg_strength * weight.
 * spg_cp_output: in_component [n], offsets [n_comp + 1], members [n] (device, int64).                      */
int spg_cp_workspace(int64_t n, int64_t n_edges, int dim, int64_t* bytes);
int spg_cp_regions(int64_t n, int64_t n_edges, int dim, int64_t* offsets);
int spg_cp_setup(const float* obs, const int64_t* source, const int64_t* target, const float* edge_weight,
                 int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t* out,
                 spg_stream_t stream);
int spg_cp_node_weights(const float* node_weight, int64_t n, int64_t n_edges, int dim, void* workspace,
                        int64_t workspace_bytes, int64_t* out, spg_stream_t stream);
int spg_cp_members(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                   spg_stream_t stream);
int spg_cp_kmeans(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                  int64_t iteration, int64_t seed, spg_stream_t stream);
int spg_cp_centers(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                   int spatial, spg_stream_t stream);
int spg_cp_capacities(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes,
                      float reg_strength, float unary, int spatial, spg_stream_t stream);
int spg_cp_maxflow(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t* out,
                   spg_stream_t stream);
int spg_cp_activate(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                    int spatial, int64_t* out, spg_stream_t stream);
int spg_cp_split(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                 int64_t* out, spg_stream_t stream);
int spg_cp_merge(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                 double reg_strength, double cutoff, int is_cutoff, int64_t* out, spg_stream_t stream);
int spg_cp_energy(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes,
                  double reg_strength, double* out, spg_stream_t stream);
int spg_cp_output(int64_t n, int64_t n_edges, int dim, void* workspace, int64_t workspace_bytes, int64_t n_comp,
                  int64_t* in_component, int64_t* offsets, int64_t* members, spg_stream_t stream);

/* ---------------------------------------------------------------- Delaunay triangulation
 * The exact 3D Delaunay triangulation of a float32 cloud (the one compute_sp_graph takes as simplices; ref:
 * partition/graphs.py:82, scipy.spatial.Delaunay), one stage per call; spg_delaunay.py runs the rounds.  n points
 * (< 2^31 - 1), a store of cap tetrahedra (8 <= cap <= 2^29).  One workspace of spg_dt_workspace(n, cap) bytes
 * (256-byte aligned) holds the whole state; every call takes the same (n, cap, workspace).
 *
 * spg_dt_setup: out[0] (host) = status (1: a non-finite coordinate), out[1] = the unique points (exact duplicates,
 *   -0 equal to +0, keep their smallest index); the points ranked lexicographically and ordered by a Morton key.
 * spg_dt_init: out[0] = status (2: fewer than 4 affinely independent points, 4: a walk did not end); the first
 *   tetrahedron, its four infinite neighbours, every point located.
 * spg_dt_cavities (big_point -1, or the one nominee whose cavity outgrew its buffer): nominate, grow the cavities,
 *   claim, check; out[0..7] (host) = nominees, winners, new tetrahedra, overflowing nominees, the smallest of
 *   them, free slots, store top, largest cavity so far.
 * spg_dt_commit: out[0] (host) = 1 when the winners need more slots than the store holds (nothing is written);
 *   else the winners' cavities are retriangulated, the displaced points relocated, out[1] = status (4: a walk did
 *   not end, 8: a cavity that is not a ball).
 * spg_dt_grow: copies the state into a workspace of spg_dt_workspace(n, new_cap) bytes.
 * spg_dt_output: with simplices NULL, count (host) = the finite tetrahedra; else simplices [count, 4] (device,
 *   int32) = them in input ids, each rotated by an even permutation to (smallest, second smallest, ...), rows
 *   sorted.  The adjacency is consumed: output is the last call on a workspace.                            */
int spg_dt_workspace(int64_t n, int64_t cap, int64_t* bytes);
int spg_dt_setup(const float* xyz, int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                 spg_stream_t stream);
int spg_dt_init(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                spg_stream_t stream);
int spg_dt_cavities(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t big_point,
                    int64_t* out, spg_stream_t stream);
int spg_dt_commit(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* out,
                  spg_stream_t stream);
int spg_dt_grow(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t new_cap,
                void* new_workspace, int64_t new_workspace_bytes, spg_stream_t stream);
int spg_dt_output(int64_t n, int64_t cap, void* workspace, int64_t workspace_bytes, int64_t* count, int* simplices,
                  spg_stream_t stream);

/* ---------------------------------------------------------------- learned partition's graph structure
 * The structure graph_processing.py builds before write_structure (ref: supervized_partition/graph_processing.py:
 * 144-193), on the device.  status words (device, uint32) are zeroed by the call that fills them; 2: an id outside
 * [0, n).
 *
 * spg_st_vor_count: the Voronoi candidates of compute_graph_nn_2(voronoi > 0) (ref: partition/graphs.py:44-49):
 *   candidate c = p n_tets + r is (simplices[r][a_p], simplices[r][b_p]) for the column pairs (a_p, b_p) = (0,1),
 *   (0,2), (0,3), (1,2), (1,3), (2,3) (simplices [n_tets, 4], int64 when ids64 else int32, n_tets <= 2^29); it is
 *   kept when d2 = (dx dx + dy dy) + dz dz, rounded op by op in float32, is < voronoi (the float32 of the caller's
 *   threshold).  block_counts [spg_st_vor_blocks(n_tets) + 1] (device, int64) = the kept candidates of every chunk,
 *   and their total in the last entry.
 * spg_st_vor_build (workspace: spg_st_vor_workspace(n, n_tets, n k_nn1, n_kept) bytes, 256-byte aligned; n_kept
 *   read back from the count): distances [n_kept] = d2 of the kept candidates in candidate order (graphs.py:64);
 *   source, target [n_kept + n k_nn1] (device, int64) = the union of the kept candidates and the k-NN edges
 *   (i, knn_target[i k_nn1 + j]) deduplicated and sorted by (target, source) (np.unique of source + n target,
 *   graphs.py:53-62); n_edges [1] (device, int64) = the number of edges written.
 * spg_st_cc (workspace: spg_st_cc_workspace(n_ver) bytes): libply_c's connected_comp with cutoff 0 (ref:
 *   partition/ply_c/connected_components.cpp:17-40): the components of the edges whose active byte, read as a
 *   signed char, is > 0; in_component [n_ver] numbered by smallest vertex (boost's numbering), offsets
 *   [n_ver + 1] (first n_comp + 1 used) and members [n_ver] (ascending within a component), n_comp [1] (device,
 *   all int64).
 * spg_st_argmax: out [n] (int64) = add + the first column of maximum value of a[i, col0:cols) (np.argmax);
 *   zero_empty: 0 where a[i, col0:] sums to 0; weight [n] (float32, may be NULL) = 0 there, else 1
 *   (graph_processing.py:126,152-154,161-162,168).
 * spg_st_transitions: is_transition [n_edges] (uint8) = lab[s] != lab[t] (mode 0; :149,165,169),
 *   hs != ht * (hs != 0) * (ht != 0) (mode 1, numpy's precedence of :155-156) or lab[s] == lab[t] (mode 2).
 * spg_st_select (workspace: spg_st_select_workspace(n) bytes): index = the ascending i with (flags[i] != 0) ==
 *   want, count [1] (device, int64) = their number.
 * spg_st_gather_rows: out[j] = the row_bytes bytes of row index[j] of src [n_rows].
 * spg_st_points: with bounds = spg_knn_bounds' words of xyz: elevation [n] = z - min z in float32 (plane 0,
 *   :186) or float32(z - (x c0 + y c1 + b)) in fp64 (plane 1, :184); xyn [n, 2] = (xy - min) / (max - min +
 *   1e-8f) in float32 (:189-190); low [n] (uint8) = z - min z < 0.5f (:182); geof [n, 4]: column 3 doubled in
 *   place (:177).  Every output may be NULL.                                                               */
int64_t spg_st_vor_blocks(int64_t n_tets);
int spg_st_vor_workspace(int64_t n, int64_t n_tets, int64_t n_knn, int64_t n_kept, int64_t* bytes);
int spg_st_vor_count(const float* xyz, int64_t n, const void* simplices, int ids64, int64_t n_tets, float voronoi,
                     int64_t* block_counts, uint32_t* status, spg_stream_t stream);
int spg_st_vor_build(const float* xyz, int64_t n, const void* simplices, int ids64, int64_t n_tets, float voronoi,
                     const int64_t* block_counts, const int64_t* knn_target, int64_t k_nn1, int64_t n_kept,
                     void* workspace, int64_t workspace_bytes, float* distances, int64_t* source, int64_t* target,
                     int64_t* n_edges, uint32_t* status, spg_stream_t stream);
int spg_st_cc_workspace(int64_t n_ver, int64_t* bytes);
int spg_st_cc(const int64_t* src, const int64_t* tgt, const uint8_t* active, int64_t n_ver, int64_t n_edges,
              void* workspace, int64_t workspace_bytes, int64_t* in_component, int64_t* offsets, int64_t* members,
              int64_t* n_comp, uint32_t* status, spg_stream_t stream);
int spg_st_argmax(const int64_t* a, int64_t n, int64_t cols, int64_t col0, int64_t add, int zero_empty,
                  int64_t* out, float* weight, spg_stream_t stream);
int spg_st_transitions(const int64_t* lab, int64_t n, const int64_t* src, const int64_t* tgt, int64_t n_edges,
                       int mode, uint8_t* is_transition, uint32_t* status, spg_stream_t stream);
int spg_st_select_workspace(int64_t n, int64_t* bytes);
int spg_st_select(const uint8_t* flags, int64_t n, int want, void* workspace, int64_t workspace_bytes, int64_t* index,
                  int64_t* count, spg_stream_t stream);
int spg_st_gather_rows(const void* src, int64_t n_rows, int64_t row_bytes, const int64_t* index, int64_t m, void* out,
                       uint32_t* status, spg_stream_t stream);
int spg_st_points(const float* xyz, int64_t n, const uint32_t* bounds, int plane, double c0, double c1, double b,
                  float* elevation, float* xyn, uint8_t* low, float* geof, spg_stream_t stream);

/* ---------------------------------------------------------------- superpoint graph batch builder
 * loader's sub-graph selection + eccpc_collate / GraphConvInfo.set_batch, one graph of the batch per call.
 * ref: learning/spg.py:114-143,178-193, learning/ecc/GraphConvInfo.py:33-69
 *
 * batch_select: src / tgt [E] (int32, the file's edge order); the undirected adjacency is the spg_graph_build
 * views of the file's stably target-sorted edges (tgt_rowptr [n + 1], in_src = its idxn [E], src_rowptr
 * [n + 1], src_perm [E], edge_tgt [E]); sizes [n] (int64) the vertex attribute s.  perm [n] (new id of every
 * vertex, NULL: identity).  centres [n_centres] (new ids; NULL: every vertex kept) start a BFS of depth `order`
 * ignoring edge directions.  cut > 0 keeps the prefix, in increasing new id, of the kept vertices whose running
 * count of s >= minpts is <= cut (k_big_enough).  Outputs: new_index [n] = sub-graph id of every vertex or -1,
 * edge_pos [E + 1] = exclusive scan of the kept-edge flags, out [2 + n] = (kept vertices, kept edges, the kept
 * original ids in sub-graph order).  Workspace from spg_batch_select_workspace, 256-byte aligned.          */
int spg_batch_select_workspace(int64_t n_ver, int64_t n_edges, int64_t* bytes);
int spg_batch_select(const int32_t* src, const int32_t* tgt, int64_t n_ver, int64_t n_edges,
                     const int32_t* tgt_rowptr, const int32_t* in_src, const int32_t* src_rowptr,
                     const int32_t* src_perm, const int32_t* edge_tgt, const int64_t* sizes, const int32_t* perm,
                     const int32_t* centres, int64_t n_centres, int order, int64_t minpts, int64_t cut,
                     int32_t* new_index, int32_t* edge_pos, int32_t* out, void* workspace, int64_t workspace_bytes,
                     spg_stream_t stream);
/* batch_edges: the graph's slice of the collated batch.  The kept edges in file order, stably sorted by new
 * target; idxn_out / tgt_out [kE] = vertex_offset + new (source, target), degs_out [n_kept] = in-degrees,
 * feats_out [kE, n_feats] = edge_feats rows, targets_out [n_kept, n_target_cols] = targets rows of kept
 * (the original ids, batch_select's out + 2).  Workspace from spg_batch_edges_workspace.
 * ref: learning/spg.py:183-185, learning/ecc/GraphConvInfo.py:48-69                                       */
int spg_batch_edges_workspace(int64_t n_kept, int64_t n_kept_edges, int64_t* bytes);
int spg_batch_edges(const int32_t* src, const int32_t* tgt, int64_t n_edges, const int32_t* new_index,
                    const int32_t* edge_pos, const int32_t* kept, int64_t n_kept, int64_t n_kept_edges,
                    int64_t vertex_offset, const float* edge_feats, int64_t n_feats, const int64_t* targets,
                    int64_t n_target_cols, int64_t* idxn_out, int64_t* tgt_out, int64_t* degs_out,
                    float* feats_out, int64_t* targets_out, void* workspace, int64_t workspace_bytes,
                    spg_stream_t stream);

/* ---------------------------------------------------------------- the batch's draws on the device
 * The random choices of loader (ref: learning/spg.py:117 random.sample, :135-137 random.shuffle, :209-214 the
 * resample, :240-257 augment_cloud) with the reference's distributions, drawn from Philox4x32-10 keyed by `seed`.
 * Counter layout: the 64-bit draw k of stream (a, b, purpose) is Philox(c0 = k >> 1, c1 = a, c2 = b, c3 = purpose)
 * words (2(k & 1), 2(k & 1) + 1) as (low, high); purposes 1 permutation, 2 centres, 3 resample, 4 augmentation,
 * 5 jitter.  Graph draws: (a, b) = (0, graph_pos), draw v for vertex (new id) v.  Training clouds: (a, b) =
 * (superpoint id, graph_pos); resample draw j for output point j, augmentation draws 0 scale, 1 angle, 2 and 3 the
 * mirrors, jitter element j F + f draws 2k and 2k + 1.  Evaluation clouds: (a, b) = the low and high words of
 * id + test_seed_offset, purpose 3 | 0x100.  u53(x) = (x >> 11) 2^-53; an index below n is the high word of x n.
 *
 * batch_draw: perm [n] (permute) = the rank of each vertex in a stable sort of its permutation key (a uniform
 * permutation; perm[i] = new id of vertex i), centres [n_centres] = the new ids of the n_centres smallest centre
 * keys (a uniform subset independent of perm).  Workspace from spg_batch_draw_workspace.
 * ref: learning/spg.py:117,135-137                                                                          */
int spg_batch_draw_workspace(int64_t n_ver, int64_t* bytes);
int spg_batch_draw(int64_t n_ver, int64_t seed, int64_t graph_pos, int permute, int64_t n_centres, int32_t* perm,
                   int32_t* centres, void* workspace, int64_t workspace_bytes, spg_stream_t stream);
/* batch_cloud_flags: one graph's slice [n_ver] of the batch's cloud table, from batch_select's out `selected`.
 * Position i < selected[0] holds kept vertex id = selected[2 + i]: count = sp_count[id] (-1 for an id the store
 * lacks, and for id >= n_ids), first_row = sp_first_row[id], flags = -2 missing, -1 count < minpts, else 0;
 * valid = (selected[1] > 0 and flags == 0); key = graph_pos << 32 | id.  Other positions: flags -1, valid 0.
 * batch_clouds: the stable compaction of the valid positions of the whole batch into start_out / count_out /
 * key_out (the first sum(valid) entries).  Workspace from spg_batch_clouds_workspace.
 * ref: learning/spg.py:146-152 (ptn_minpts), s3dis_dataset.py:151-158 (one dataset per superpoint)          */
int spg_batch_cloud_flags(const int32_t* selected, int64_t n_ver, int64_t graph_pos, const int64_t* sp_first_row,
                          const int32_t* sp_count, int64_t n_ids, int64_t minpts, int32_t* flags, int32_t* valid,
                          int64_t* first_row, int32_t* count, int64_t* key, spg_stream_t stream);
int spg_batch_clouds_workspace(int64_t n, int64_t* bytes);
int spg_batch_clouds(const int32_t* valid, const int64_t* first_row, const int32_t* count, const int64_t* key,
                     int64_t n, void* workspace, int64_t workspace_bytes, int64_t* start_out, int32_t* count_out,
                     int64_t* key_out, spg_stream_t stream);
/* batch_cloud_draw: the inputs of spg_cloud_build for n_clouds clouds of key / count (batch_clouds' outputs).
 * sample_idx [n, L]: identity when count == L, the original points first when count < L, else uniform in
 * [0, count).  xform [n, 9] (NULL: none; evaluation passes NULL): s = 1/scale + (scale - 1/scale) u when
 * scale > 1, the rotation about z by 2 pi u when rotate == 1, each mirror when u < mirror_prob / 2, composed in
 * float64 in augment_matrix's order.  jitter [n, L, F] (NULL: none): float32(clip(0.01 g, +-0.05)) with g the
 * float64 Box-Muller normal of (1 - u53, u53).  train == 0 keys the resample by id + test_seed_offset.
 * ref: learning/spg.py:207-214,240-257                                                                     */
int spg_batch_cloud_draw(const int64_t* key, const int32_t* count, int64_t n_clouds, int n_points, int n_attribs,
                         int64_t seed, int train, int64_t test_seed_offset, double scale, int rotate,
                         double mirror_prob, int32_t* sample_idx, double* xform, float* jitter, spg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SPG_B200_H_ */
