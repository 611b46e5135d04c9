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
 *  after the n_partials*C*3 floats; the same holds for the workspaces of spg_colstats / stats_ws) */

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

/* Per-column batch statistics of Y[M,C] (ld = ldy): mean[C], biased var[C];
 * workspace >= 3*C*spg_colstats_chunks(M) floats.  ref: nn.BatchNorm1d in training
 * mode (learning/pointnet.py:31,43,87,103; learning/graphnet.py:29).            */
int64_t spg_colstats_chunks(int64_t M);
int spg_colstats(const float* Y, int64_t ldy, int64_t M, int C, float* mean, float* var,
                 float* workspace, spg_stream_t stream);
/* scale = gamma/sqrt(var+eps), shift = beta-mean*scale; if running_* non-NULL:
 * running = (1-momentum)*running + momentum*{mean, var*M/(M-1)}; if num_batches_tracked
 * (int64 scalar, device) is non-NULL it is incremented by one.                    */
int spg_bn_fold(const float* mean, const float* var, const float* gamma, const float* beta,
                float eps, float* scale, float* shift, float* running_mean, float* running_var,
                int64_t* num_batches_tracked, float momentum, int64_t M, int C,
                spg_stream_t stream);
/* out[m,c] = f(Y[m,c]*scale[c]+shift[c]); scale/shift may be NULL.               */
int spg_affine_act(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* out, int64_t ldo, int64_t M, int C, spg_stream_t stream);
/* Column sums: out[c] = sum_m X[m,c]; workspace >= C*spg_colstats_chunks(M).      */
int spg_colsum(const float* X, int64_t ldx, int64_t M, int C, float* out, float* workspace,
               spg_stream_t stream);
/* Backward of a = relu?(bn?(y)):
 *   pass 1 (spg_act_bwd_reduce, BN layers only):
 *       s1[c] = sum_m G*mask, s2[c] = sum_m G*mask*xhat       (= d_beta, d_gamma)
 *   pass 2 (spg_act_bwd_apply): dY = scale*(G*mask - s1/M - xhat*s2/M)   (BN)
 *                               dY = G*mask                             (no BN)
 *   mask = (y*scale+shift > 0) if relu else 1; xhat = (y-mean)*rstd; in-place OK. */
int spg_act_bwd_reduce(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                       const float* scale, const float* shift, const float* mean,
                       const float* var, float eps, int relu, float* s1, float* s2,
                       float* workspace, int64_t M, int C, spg_stream_t stream);
int spg_act_bwd_apply(const float* G, int64_t ldg, const float* Y, int64_t ldy,
                      const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, int has_bn, const float* s1,
                      const float* s2, float* dY, int64_t lddy, int64_t M, int C,
                      spg_stream_t stream);

/* ------------------------------------------------------------ PointNet    */
/* clouds [B,F,L] (the reference's NCL layout, learning/spg.py:162) -> rows [B*L, ld]
 * (point-major, channel contiguous, zero padded to ld).  If T [B,2,2] is given the
 * first two channels are replaced by (xy^T * T')^T with T' = T (+ I if add_eye: the STN's
 * "+ identity", ref: learning/pointnet.py:61,121-124).                                   */
int spg_cloud_rows(const float* clouds, const float* T, int add_eye, float* rows, int64_t ld,
                   int64_t B, int F, int L, spg_stream_t stream);
/* pooled[b,c] = max_l f(Y[b*L+l,c]*scale[c]+shift[c]); argmax[b,c] = first maximiser.
 * Writes into pooled with leading dimension ldp (so that the "global" features can sit
 * in the same row, ref: learning/pointnet.py:126-132).                              */
int spg_segmax_fwd(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                   float* pooled, int64_t ldp, int32_t* argmax, int64_t B, int L, int C,
                   spg_stream_t stream);
/* G[b*L+l,c] = (l==argmax[b,c]) ? g_pooled[b,c] : 0 (G fully written).              */
int spg_segmax_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, float* G,
                   int64_t ldG, int64_t B, int L, int C, spg_stream_t stream);
/* Max-pool backward fused with the BatchNorm(+ReLU) backward of the layer Y that fed the pool:
 * s12 = [s1|s2] (= d_beta | d_gamma, 2*C floats) and dY[B*L,C] are produced straight from the pooled
 * gradient and the argmax; the dense gradient of the pooled activation is never materialised.
 * workspace >= 2*C*ceil(B/256) floats.  C % 4 == 0.                                            */
int spg_segmax_bn_bwd(const float* g_pooled, int64_t ldg, const int32_t* argmax, const float* Y,
                      int64_t ldy, const float* scale, const float* shift, const float* mean,
                      const float* var, float eps, int relu, float* s12, float* dY, int64_t lddy,
                      float* workspace, int64_t B, int L, int C, spg_stream_t stream);
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
 * learning/spg.py:209-214): point rows [P, ld] of all superpoints back to back, offsets int64 [B+1].
 *   spg_segmax_csr_fwd: pooled[b,c] = max over the segment's rows of relu?(Y*scale+shift); argmax_row
 *     int64 [B,C] = GLOBAL row of the first maximum (-1 and pooled 0 for an empty segment)
 *   spg_segmax_csr_bwd: G[P,C] (zeroed here) receives g_pooled[b,c] at row argmax_row[b,c]
 *   spg_rows_xy_transform(+_bwd): columns 0,1 of every row times its segment's 2x2 T (+I)
 *     (learning/pointnet.py:123), row_seg int32 [P] = segment of each row; backward: dT [B,4].        */
int spg_segmax_csr_fwd(const float* Y, int64_t ldy, const float* scale, const float* shift, int relu,
                       const int64_t* offsets, float* pooled, int64_t ldp, int64_t* argmax_row, int64_t B,
                       int C, spg_stream_t stream);
int spg_segmax_csr_bwd(const float* g_pooled, int64_t ldg, const int64_t* argmax_row, float* G, int64_t ldG,
                       int64_t B, int C, int64_t P, spg_stream_t stream);
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

#ifdef __cplusplus
}
#endif
#endif /* SPG_B200_H_ */
