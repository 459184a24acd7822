// kernels.cuh -- device helpers + launcher declarations shared by rgcn_kernels.cu / api.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "graph.h"

#define RGCN_WARPS_PER_BLOCK 8
#define RGCN_THREADS (RGCN_WARPS_PER_BLOCK * 32)

extern int64_t g_rgcn_launches;  // counted on the host at every kernel launch of this library

struct AggLaunch {
  const WorkItem* items;
  int n_items;
  const int32_t* nbr;   // gather row per message
  const int32_t* relw;  // weight id per message
  const float* norm;    // per message
  const float* X;       // gathered feature matrix, row-major, leading dimension ldx
  int ldx;
  int d;                // feature width
  const int32_t* split_nitems;
  float* scratch;  // [n_split, d]  zeroed
  int* counters;   // [n_split * n_slabs] zeroed
};

// Block-diagonal aggregation (forward, and backward-w.r.t.-H with the transposed table):
//   out[row,:] = act( out[row,:] (*mask/keep) + sum_m norm_m * Wt[relw_m] (.) X[nbr_m,:] )
// Wt layout: [n_relw][s][d] with Wt[w][j][b*s+i] = coefficient multiplying x[b*s+j] in y[b*s+i].
int launch_block_agg(const AggLaunch& a, int s, const float* Wt, float* out, const uint8_t* mask,
                     float inv_keep, int relu, cudaStream_t st);

// Weight-id major variant of the above (weights in registers, vector reductions into `out`, which
// must already hold the self-loop term).  Supported block sizes: block_rel_supported().
bool block_rel_supported(int d, int s);
bool block_rel_fuse_dw_supported(int d, int s);
// dWt != nullptr (backward pass, X = G, rows = sources, Hrow = layer input): additionally accumulates
// the block weight gradient in the j-major layout (dWt zeroed by the caller) in the same walk.
int launch_block_rel(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                     const float* r_norm, const float* X, int ldx, int d, int s, const float* Wt,
                     float* out, const float* Hrow, int ldh, float* dWt, cudaStream_t st);

// Same contract as launch_block_rel with the gathered rows staged through shared memory by TMA bulk copies
// (block_staged.cu); block sizes 4, 8, 16.
bool block_stg_supported(int d, int s);
int launch_block_stg(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                     const float* r_norm, const float* X, int ldx, int d, int s, const float* Wt, float* out,
                     const float* Hrow, int ldh, float* dWt, cudaStream_t st);

// Block-diagonal weight gradient, weight-id major:
//   dWt[w][j][b*s+i] += sum_{m: relw_m = w} norm_m * G[dst_m, b*s+i] * H[src_m, b*s+j]
int launch_block_dw(const WorkItem* items, int n_items, const int32_t* r_dst, const int32_t* r_src,
                    const float* r_norm, const float* H, int ldh, const float* G, int ldg, int d,
                    int s, float* dWt, cudaStream_t st);

// Re-layout of the reference weight tables [R,B,s,s] (W.x orientation) into the kernel tables.
//   transpose = 0:  Wt[w][j][b*s+i] = W[w][b][i][j]      (forward)
//   transpose = 1:  Wt[w][i][b*s+j] = W[w][b][i][j]      (backward w.r.t. H: y = W^T g)
int launch_block_relayout(const float* Wf, const float* Wb, int R, int B, int s, int transpose,
                          float* Wt, cudaStream_t st);
// inverse of transpose=0 layout: dW[w][b][i][j] = dWt[w][j][b*s+i]
int launch_block_unlayout(const float* dWt, int R, int B, int s, float* dWf, float* dWb,
                          int accumulate, int table_t, cudaStream_t st);

// Basis aggregation: Agg[row][dir][...] = sum_m norm_m * C[relw_m, b] * X[nbr_m, k]
//   layout 0 (interleaved): index k*B + b      (matches V.reshape(d_in*B, d_out) rows)
//   layout 1 (planar):      index b*d + k      (matches V.reshape(d_in, B*d_out) columns)
// dir = relw >= n_relw/2.  Row stride of Agg is 2*d*B, direction stride d*B.
int launch_basis_agg(const AggLaunch& a, const float* C, int B, int n_relw, int layout, float* Agg,
                     cudaStream_t st);

// One-hot basis layer backward (source major, X = G): the planar basis aggregation written straight into the two
// [V_src][B][d] weight-gradient tables, dW_dir[u][b][:] = sum_{m: src_m = u, dir} norm_m C[relw_m,b] G[dst_m,:],
// fused with dC[w][b] += sum_{m: relw_m = w} norm_m < W_dir[src_m][b][:], G[dst_m,:] > (dC zeroed by the caller).
// Rows without messages in a direction are written as zeros; split rows must be zeroed first.
int launch_basis_agg_dc(const AggLaunch& a, const float* C, int B, int n_relw, const float* W0, const float* W1,
                        float* dW0, float* dW1, float* dC, cudaStream_t st);

// basis_onehot.cu -- one-hot basis layer forward (push over the source-major view; `out` holds the self-loop term):
//   out[dst_m,:] += norm_m * sum_b C[relw_m,b] W_dir[src_m][b][:]     (W_dir = Wf for relw < n_relw/2, else Wb)
int launch_basis_onehot_push(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                             const float* norm, const float* Wf, const float* Wb, const float* C, int B, int d,
                             int n_relw, float* out, cudaStream_t st);

// basis_diagcoef.cu -- basis layer with per-channel sigmoid coefficients (gcn_basis_times_diag.py).  sig is the
// [n_relw][B][d] table sigmoid([Cf; Cb]); P the [V_src][2][B][d] transformed rows H [V_f | V_b].
int launch_diagcoef_sigmoid(const float* Cf, const float* Cb, int64_t n_half, float* sig, cudaStream_t st);
//   out[dst_m,:] += norm_m * sum_b sig[relw_m,b,:] (.) P[src_m][dir][b][:]      (destination-major view)
int launch_diagcoef_fwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                        const float* P, const float* sig, int B, int d, int n_relw, float* out, cudaStream_t st);
// out = act(out + bias), bias [d]
int launch_diagcoef_bias_act(float* out, const float* bias, int64_t rows, int d, int relu, cudaStream_t st);
// db = column sums of G [rows, d] (db is overwritten)
int launch_diagcoef_colsum(const float* G, int64_t rows, int d, float* db, cudaStream_t st);
//   dP[u][dir][b][:] = sum_{m: src_m = u, dir} norm_m sig[relw_m,b,:] (.) G[dst_m,:]   (source-major view; rows
//   without messages in a direction are written as zeros, split rows must be zeroed first)
int launch_diagcoef_dp(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* G, const float* sig, int B, int d, int n_relw, float* dP, cudaStream_t st);
//   dC_dir[w][b][:] += sig (1 - sig) (.) sum_{m: relw_m = w} norm_m P[src_m][dir][b][:] (.) G[dst_m,:]
//   (weight-id-major view with rows = sources; dCf / dCb zeroed by the caller)
int launch_diagcoef_dc(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                       const float* r_norm, const float* P, const float* G, const float* sig, int B, int d, int n_relw,
                       float* dCf, float* dCb, cudaStream_t st);

// gcn_diag.cu -- diagonal R-GCN layer (gcn_diag.py); D_dir tables [R][d], weight id w reads Df[w] (w < n_relw/2)
// or Db[w - n_relw/2].  Forward, destination-major view, `out` holding H W_self (unmasked):
//   out[row] = act( dropout(out[row]) + sum_{m into row} norm_m D[relw_m] (.) H[src_m] + bias )
// (split rows: scratch [n_split, d] and counters [n_split * slabs] zeroed by the caller)
int launch_diaggcn_fwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* H, const float* Df, const float* Db, int d, int n_relw, const float* bias,
                       const uint8_t* mask, float inv_keep, int relu, const int32_t* split_nitems, float* scratch,
                       int* counters, float* out, cudaStream_t st);
// Backward, source-major view (rows = sources u):  dH[u] += sum_{m from u} norm_m D[relw_m] (.) G[dst_m];
// dD[w] += sum_{m: relw_m = w} norm_m H[src_m] (.) G[dst_m] (dDf / dDb zeroed by the caller); if sumsq2 != null,
// sumsq2[dir] += sum_m norm_m^2 |H[src_m] (.) G[dst_m]|^2 over the messages of each direction.
int launch_diaggcn_bwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* G, const float* H, const float* Df, const float* Db, int d, int n_relw, float* dH,
                       float* dDf, float* dDb, float* sumsq2, cudaStream_t st);

// compgcn.cu -- CompGCN layer (Name=compgcn); Z [2R][d] (weight id w reads Z[w]), phi = h (.) z (op 0, mult) or
// h - z (op 1, sub).  Forward, destination-major view: Cat [V_dst, 3d] =
//   [ mask / keep (.) A_f | mask / keep (.) A_b | phi(H[row], z_loop) ] / 3,   A_dir[row] = sum_m norm_m phi(H[src_m], Z[w_m])
// (mask [V_dst, 2d] or null; split rows of Cat zeroed by the caller).
int launch_compgcn_fwd(int op, const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                       const float* norm, const float* H, const float* Z, const float* zloop, int d, int n_relw,
                       const uint8_t* mask, float inv_keep, float* Cat, cudaStream_t st);
// Backward, source-major view (rows = sources u), dCat = dL/dCat:  per (u, w) run S = sum_m norm_m dCat'_slab(w)[dst_m]
// (dCat' = dCat with the mask / keep and the 1/3 of the forward), dH[u] = sum of the runs' phi_h^T S plus, for
// u < V_dst, the loop term; dZ[w] and dz_loop accumulate the phi_z^T S terms (zeroed by the caller; split rows of dH
// zeroed by the caller).
int launch_compgcn_bwd(int op, const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                       const float* norm, const float* dCat, const float* H, const float* Z, const float* zloop, int d,
                       int n_relw, int V_dst, const uint8_t* mask, float inv_keep, float* dH, float* dZ,
                       float* dzloop, cudaStream_t st);

// Basis coefficient gradient (destination major):
//   dC[w][b] += sum_{m into row, relw_m = w} norm_m * < H[src_m,:], dAgg[row][dir][:, b] >
int launch_basis_dc(const AggLaunch& a, const float* dAgg, int B, int n_relw, float* dC,
                    cudaStream_t st);

// slice_norm.cu: squared norms of the un-aggregated IndexedSlices gradients (tf.clip_by_global_norm semantics)
int launch_block_sqnorm(const float* X, int64_t rows, int ld, int B, int s, float* XB, cudaStream_t st);
// out2[0] += sum over forward-table messages, out2[1] += backward-table messages of norm^2 * <GB[dst], HB[src]>
int launch_block_slice_sumsq(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                             const float* r_norm, const float* GB, const float* HB, int B, int half, float* out2,
                             cudaStream_t st);

// Elementwise helpers
// G = dOut * (out > 0 if relu);  dS = G * mask * inv_keep (only if mask != null, else dS untouched)
int launch_grad_prologue(const float* dOut, const float* out, const uint8_t* mask, float inv_keep,
                         int relu, int64_t n, float* G, float* dS, cudaStream_t st);
// x = x * mask * inv_keep (if mask) ; x = relu(x) (if relu)
int launch_mask_relu(float* x, const uint8_t* mask, float inv_keep, int relu, int64_t n,
                     cudaStream_t st);
// dst[rows[i], :] += src[i, :], rows unique within the call
int launch_rows_add(float* dst, const int64_t* rows, const float* src, int64_t n, int d, cudaStream_t st);
int launch_rows_gather(float* dst, const float* src, const int64_t* rows, int64_t n, int d, int max_ctas,
                       cudaStream_t st);
// zero rows listed in `rows` of a [*, width] matrix
int launch_zero_rows(float* A, int64_t width, const int32_t* rows, int n_rows, cudaStream_t st);

// fp32-accurate tensor-core GEMM (gemm_tf32x3.cu): C[M,N] (+)= A[M,K] * Bt[N,K]^T with Bt pre-split
int launch_gemm_split_b(const float* B, int64_t ldb, int N, int K, int transposed, float* hi, float* lo,
                        cudaStream_t st);
int launch_gemm_tf32x3(const float* A, int64_t lda, const float* Bt_hi, const float* Bt_lo, int64_t ldb,
                       float* C, int64_t ldc, int M, int N, int K, int accumulate, cudaStream_t st);
// C = act(A Bt^T + bias), act = ReLU if relu, the identity otherwise; bias [N]
int launch_gemm_bias_act_tf32x3(const float* A, int64_t lda, const float* Bt_hi, const float* Bt_lo, int64_t ldb,
                                const float* bias, int relu, float* C, int64_t ldc, int M, int N, int K,
                                cudaStream_t st);

int launch_gemm_rank_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const float* gold_sig, const int32_t* gold_col, const uint32_t* known,
                            int words, int32_t* raw_cnt, int32_t* known_cnt, cudaStream_t st);

// Scoring GEMM with the top-k epilogue: for every row of Q and every 128-column tile of Bt, the tile's best k
// eligible (energy, column) pairs -- energy descending, smaller column first on ties; excl bit set or column >= N:
// not eligible -- in order in cand [M, ceil(N / 128), k] as (energy bits, column), the tail padded (-inf, -1).
int launch_gemm_topk_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const uint32_t* excl, int words, int k, uint2* cand, cudaStream_t st);
// topk.cu -- merge of those candidates: ids [n, k] / energies [n, k] of every row's best k, in the same order, the
// tail past the row's eligible columns padded (-1, -inf)
int launch_topk_merge(const uint2* cand, int64_t n, int per_row, int k, int32_t* ids, float* energies,
                      cudaStream_t st);

// In-place truncation split of `count` floats (count % 4 == 0): a becomes the TF32 hi part, lo the remainder's --
// the split the scoring GEMM's producer applies to the query rows
int launch_split_trunc(float* a, float* lo, int64_t count, cudaStream_t st);
// Ensemble ranking GEMM (R-GCN+): per member X the query rows q_X [M, K_X] (truncation split) against the entity
// codes c_X [N, K_X] (round-to-nearest split); c = w s_A + (1 - w) s_B in float64 of the two float32 sigmoid scores,
// G the same of the gold sigmoids; raw_cnt / known_cnt += the counts of c >= G (the gold column always counts).
int launch_gemm_ensemble_rank_tf32x3(const float* qa_hi, const float* qa_lo, const float* ca_hi, const float* ca_lo,
                                     const float* gold_sig_a, int Ka, const float* qb_hi, const float* qb_lo,
                                     const float* cb_hi, const float* cb_lo, const float* gold_sig_b, int Kb, int M,
                                     int N, double w, double omw, const int32_t* gold_col, const uint32_t* known,
                                     int words, int32_t* raw_cnt, int32_t* known_cnt, cudaStream_t st);
// Ensemble top-k candidate: u = w sigma(-E_A) + (1 - w) sigma(-E_B) in double and the column; id -1 = none (u +inf)
struct EnsCand {
  double u;
  int32_t id;
  int32_t pad;
};
// candidates per row and 64-column tile of the ensemble top-k GEMM: a tile has no more than 64 columns to offer
inline int ensemble_topk_per_tile(int k) { return k < 64 ? k : 64; }
// Ensemble top-k GEMM: operands as launch_gemm_ensemble_rank_tf32x3; for every row and every 64-column tile the best
// ensemble_topk_per_tile(k) eligible (u, column) pairs -- u ascending, smaller column first on ties; excl bit set or
// column >= N: not eligible -- in order in cand [M, ceil(N / 64), ensemble_topk_per_tile(k)], the tail (+inf, -1).
int launch_gemm_ensemble_topk_tf32x3(const float* qa_hi, const float* qa_lo, const float* ca_hi, const float* ca_lo,
                                     int Ka, const float* qb_hi, const float* qb_lo, const float* cb_hi,
                                     const float* cb_lo, int Kb, int M, int N, double w, double omw,
                                     const uint32_t* excl, int words, int k, EnsCand* cand, cudaStream_t st);
// topk.cu -- merge of those candidates: ids [n, k], u [n, k] and c = 1 - u [n, k] (double) of every row's best k in
// the same order, the tail past the row's eligible columns padded (-1, +inf, 0)
int launch_ensemble_topk_merge(const EnsCand* cand, int64_t n, int per_row, int k, int32_t* ids, double* u,
                               double* scores, cudaStream_t st);

// max_splits > 0 caps the split-K count; max_splits = 1 makes C bitwise repeatable (one CTA adds each tile's parts
// in order), at the cost of fewer CTAs when the output has few tiles
int launch_gemm_tn_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc,
                          int M, int N, int K, int accumulate, cudaStream_t st, int max_splits = 0);

// 1-N training (onen.cu and the EPI = 5 scoring GEMM).  Loss parts the GEMM writes for M queries and N entities:
int64_t gemm_onen_loss_parts(int64_t M, int N);
// For query m and entity n, z = <Q[m], codes[n]>, y' = pos / neg as bit n of labels row m is set / clear:
// loss_part gets the sums of max(z,0) - z y' + log1p(exp(-|z|)); Gt[n * ldgt + m] = (sigmoid(z) - y') scale g_scale[0]
// (g_scale null: 1; Gt null: loss only)
int launch_gemm_onen_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const uint32_t* labels, float pos, float neg, float scale,
                            const float* g_scale, float* Gt, int64_t ldgt, float* loss_part, cudaStream_t st);
// label rows: bits [n, words] of the queries X[t] = (anchor, r, anchor) of one side from the training CSR (keys sorted,
// key = (2 r + side) V + anchor; entities of key i at offsets[i] .. offsets[i+1])
int launch_onen_labels(const int64_t* keys, const int64_t* offsets, const int32_t* entities, int64_t n_keys,
                       const int32_t* X, int64_t n, int side, int V, int words, uint32_t* bits, cudaStream_t st);
// reg parts: onen_reg_parts(n) sums of |codes[anchor]|^2 + |rel[r]|^2 over the queries
int64_t onen_reg_parts(int64_t n);
int launch_onen_reg(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* reg_part,
                    cudaStream_t st);
// loss[0] = inv_nv * (sum of the loss parts), loss[1] = inv_nd * (sum of the reg parts), each summed in a fixed order
int launch_onen_loss_reduce(const float* loss_part, int64_t n_loss, const float* reg_part, int64_t n_reg,
                            double inv_nv, double inv_nd, float* loss, cudaStream_t st);
// dst = g_scale[0] src, count % 4 == 0 floats
int launch_onen_scale(const float* src, const float* g_scale, int64_t count, float* dst, cudaStream_t st);
// anchor and relation gradients of the queries of one side: from dQ [n, d] and the L2 term c = g_scale[1] 2 / (n_all d)
// (g_scale null: 1), red.global.add into dcodes[anchor] and drel[r]; complex = 0 DistMult, 1 ComplEx; dQ null (DistMult
// kernel, either decoder): the L2 term only
int launch_onen_query_bwd(int complex, const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                          int side, const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                          cudaStream_t st);

// Highway gate GEMM with the blend epilogue: gate = sigmoid(c2 W + bias), out = c2 + gate (c1 - c2); W given
// pre-split as Bt = W^T [d, d]; all [M, d] matrices contiguous
int launch_gemm_highway_tf32x3(const float* c2, const float* Bt_hi, const float* Bt_lo, const float* bias,
                               const float* c1, float* out, float* gate, int M, int d, cudaStream_t st);
// highway.cu -- highway backward prologue: dc1 = g dY, dc2 = (1 - g) dY, dz = dY (c1 - c2) g (1 - g),
// db = column sums of dz (db is overwritten)
int launch_highway_prologue(const float* c1, const float* c2, const float* g, const float* dY, int64_t V, int d,
                            float* dc1, float* dz, float* dc2, float* db, cudaStream_t st);

// Variational head (extras/variational_encoding.py).  W_int [d, 2w] interleaves the columns of W_mu and W_sigma
// [d, w]; its pre-split is made from the two tables: transposed = 1 gives Bt = W_int^T [2w, d], 0 gives W_int [d, 2w].
int launch_gemm_split_b_interleave(const float* Wmu, const float* Wsig, int d, int w, int transposed, float* hi,
                                   float* lo, cudaStream_t st);
// KL parts written by launch_gemm_variational_tf32x3 for M rows
int64_t gemm_variational_kl_parts(int64_t M, int w);
// P = H W_int + (b_mu, b_sigma) interleaved [M, 2w], z = mu + exp(l) eps [M, w], KL parts of 1 + 2l - mu^2 - exp(2l)
int launch_gemm_variational_tf32x3(const float* H, const float* Bt_hi, const float* Bt_lo, const float* b_mu,
                                   const float* b_sigma, const float* eps, float* P, float* z, float* kl_part, int M,
                                   int d, int w, cudaStream_t st);
// variational.cu -- embedding variant forward (mu = Wmu, l = Wsig, [V, w]): z and var_emb_kl_parts(V, w) parts
int64_t var_emb_kl_parts(int64_t V, int w);
int launch_var_emb_forward(const float* Wmu, const float* Wsig, const float* eps, int64_t V, int w, float* z,
                           float* kl_part, cudaStream_t st);
// kl[0] = -0.0005 * sum of the n parts, summed in a fixed order
int launch_var_kl_reduce(const float* kl_part, int64_t n, float* kl, cudaStream_t st);
// embedding variant backward: dWmu = dz + 0.001 g mu, dWsig = dz exp(l) eps + 0.001 g (exp(2l) - 1), g = g_kl[0]
int launch_var_emb_backward(const float* Wmu, const float* Wsig, const float* eps, const float* dz, const float* g_kl,
                            int64_t V, int w, float* dWmu, float* dWsig, cudaStream_t st);
// gcn variant backward prologue: dP [V, 2w] interleaved from P [V, 2w], eps, dz [V, w], g = g_kl[0]; col_part
// [var_colsum_parts(V), 2w] the per-row-block column sums of dP
int64_t var_colsum_parts(int64_t V);
int launch_var_prologue(const float* P, const float* eps, const float* dz, const float* g_kl, int64_t V, int w,
                        float* dP, float* col_part, cudaStream_t st);
// db_mu[j] / db_sigma[j] = sum over the parts of col_part[:, 2j] / [:, 2j + 1], in part order
int launch_var_colsum_finish(const float* col_part, int64_t parts, int w, float* db_mu, float* db_sigma,
                             cudaStream_t st);
// dW_mu[:, j] = dW_int[:, 2j], dW_sigma[:, j] = dW_int[:, 2j + 1]  (dW_int [d, 2w])
int launch_var_deinterleave(const float* dWint, int d, int w, float* dWmu, float* dWsig, cudaStream_t st);

// DistMult
// queries + gold scores of the fused scorer/ranker: side 0 (subjects corrupted): Q[t] = rel[r] * codes[o], gold = s;
// side 1 (objects corrupted): Q[t] = codes[s] * rel[r], gold = o.  gold_sig[t] = sigmoid(<Q[t], codes[gold]>)
// (gold_sig == nullptr: Q only; the gold column of X is then not read)
int launch_distmult_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                                 float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);
// relation queries (h, ?, t): Q[t] = codes[h] * codes[t], gold = r, gold_sig[t] = sigmoid(<Q[t], rel[r]>)
// (gold_sig == nullptr: Q only; the relation column of X is then not read)
int launch_distmult_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                                     float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);
int launch_distmult_rank_finalize(const int32_t* raw_cnt, const int32_t* known_cnt, int64_t n, int32_t* raw_rank,
                                  int32_t* filtered_rank, cudaStream_t st);
int launch_distmult_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N,
                            const float* Y, float* energies, float* loss_out, cudaStream_t st);
int launch_distmult_backward(const float* codes, const float* rel, int d, const int32_t* X,
                             int64_t N, const float* Y, const float* energies, float g_loss,
                             float g_reg, const float* g_scale_dev, const float* g_energy,
                             float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st);

// ComplEx (complex.cu): same contracts as the DistMult launchers above, rows split as [real | imaginary]
int launch_complex_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           float* energies, float* loss_out, cudaStream_t st);
int launch_complex_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                            const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                            const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq,
                            cudaStream_t st);
// side 0: Q[t] = [rr e2r + ri e2i, rr e2i - ri e2r], gold = s;  side 1: Q[t] = [e1r rr - e1i ri, e1i rr + e1r ri],
// gold = o.  gold_sig[t] = sigmoid(<Q[t], codes[gold]>)
int launch_complex_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                                float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);
// relation queries (h, ?, t): Q[t] = [hr tr + hi ti, hr ti - hi tr], gold = r, gold_sig[t] = sigmoid(<Q[t], rel[r]>)
// (gold_sig == nullptr: Q only; the relation column of X is then not read)
int launch_complex_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                                    float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);

// self_adversarial.cu -- self-adversarial objective over N = n (K + 1) triples in the sampler's layout (decoder: one of
// the SELFADV_* kinds; gamma is read by RotatE and TransE only): energies [N], the energy-gradient coefficients coef [N],
// loss_out[0] the loss, loss_out[1] the decoder's L2 term of its NegativeSampling forward; parts: 2n floats of scratch
// for the per-group loss and norm parts
enum { SELFADV_DISTMULT = 0, SELFADV_COMPLEX = 1, SELFADV_ROTATE = 2, SELFADV_TRANSE = 3, SELFADV_QUATE = 4,
       SELFADV_HOLE = 5 };
int launch_self_adversarial_forward(int decoder, const float* codes, const float* rel, int d, const int32_t* X,
                                    int64_t N, int K, float alpha, float gamma, float* energies, float* coef,
                                    float* loss_out, float* parts, cudaStream_t st);

// rotate.cu -- RotatE (DESIGN.md section 1).  Scorer and backward: the contracts of the ComplEx launchers with the
// margin gamma; rows [re | im], the phases in the first d / 2 columns of the relation row.
int launch_rotate_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          float gamma, float* energies, float* loss_out, cudaStream_t st);
int launch_rotate_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                           const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st);
// all-entity ranking by distance: query rows Q [n, d] ([re | im]; side 1: codes[s] e^{i theta}, side 0:
// codes[o] e^{-i theta}), gold_D[t] the gold's distance and gold_col[t] its id; then raw_cnt / known_cnt (zeroed by the
// caller) += the counts of D_v <= gold_D (the gold always counts) over all V entities
int launch_rotate_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                               float* Q, float* gold_D, int32_t* gold_col, cudaStream_t st);
int launch_rotate_rank(const float* Q, const float* codes, int V, int d, int64_t n, const float* gold_D,
                       const int32_t* gold_col, const uint32_t* known, int32_t* raw_cnt, int32_t* known_cnt,
                       cudaStream_t st);

// transe.cu -- TransE (DESIGN.md section 1).  Scorer and backward: the contracts of the RotatE launchers; rows are
// plain real vectors of d % 4 == 0 columns, all d columns of the relation row are used.
int launch_transe_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          float gamma, float* energies, float* loss_out, cudaStream_t st);
int launch_transe_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                           const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st);
// query rows Q [n, d] of X: mode 1 (objects corrupted) codes[s] + rel[r], gold o; mode 0 (subjects corrupted)
// codes[o] - rel[r], gold s; mode TRANSE_RELATIONS codes[o] - codes[s], gold r (the candidates are rel).  With gold_D,
// also gold_D[t] = the gold's distance and gold_col[t] its id (gold_D == nullptr: Q only; the gold is not read).
enum { TRANSE_RELATIONS = 2 };
int launch_transe_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int mode,
                          float* Q, float* gold_D, int32_t* gold_col, cudaStream_t st);
// ranks against the first V rows of `table`: raw_cnt / known_cnt (zeroed by the caller) += the counts of
// D_v <= gold_D (the gold always counts), known [n, ceil(V/32)] or nullptr
int launch_transe_rank(const float* Q, const float* table, int V, int d, int64_t n, const float* gold_D,
                       const int32_t* gold_col, const uint32_t* known, int32_t* raw_cnt, int32_t* known_cnt,
                       cudaStream_t st);
// top-k against the first V rows of `table`: ids [n, k] / energies [n, k] = gamma - D of every row's k smallest D, the
// smaller id first on ties, never a column whose bit is set in excl [n, ceil(V/32)] (or nullptr); the tail (-1, -inf).
// cand: n * transe_topk_tiles(V) * k candidates of scratch.
inline int transe_topk_tiles(int V) { return (V + 127) / 128; }
int launch_transe_topk(const float* Q, const float* table, int V, int d, int64_t n, const uint32_t* excl, int k,
                       float gamma, uint2* cand, int32_t* ids, float* energies, cudaStream_t st);

// quate.cu -- QuatE (DESIGN.md section 1).  Scorer and backward: the contracts of the DistMult launchers; quaternion k
// of a row is the float4 at column 4k (d % 4 == 0), the relation quaternions are normalised before use.
int launch_quate_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                         float* energies, float* loss_out, cudaStream_t st);
int launch_quate_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                          const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st);
// entity query rows in launch_distmult_rank_prepare's contract: side 1 Q = h (x) rh, side 0 Q = t (x) conj(rh)
int launch_quate_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                              float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);
// rh [R, d] = the normalised quaternions of rel[0:R]: the candidates of the relation queries
int launch_quate_normalize(const float* rel, int R, int d, float* rh, cudaStream_t st);
// pair query rows in launch_distmult_relation_prepare's contract: Q = conj(h) (x) t, the gold scored against the
// normalised rel[r]
int launch_quate_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* Q,
                                  float* gold_sig, int32_t* gold_col, cudaStream_t st);
// 1-N query backward in launch_onen_query_bwd's contract (dQ is never null)
int launch_quate_query_bwd(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                           const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                           cudaStream_t st);

// hole.cu -- HolE (DESIGN.md section 1) on rows in the real Fourier basis x~ = x U.  U [d, d] (d % 4 == 0) into a
// device buffer:
int launch_hole_basis(int d, float* U, cudaStream_t st);
// Scorer and backward over transformed rows: the contracts of the DistMult launchers.
int launch_hole_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                        float* energies, float* loss_out, cudaStream_t st);
int launch_hole_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                         const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                         const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st);
// entity query rows in launch_distmult_rank_prepare's contract: side 1 Q = w (h r), side 0 Q = w conj(r) t
int launch_hole_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                             float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st);
// pair query rows in launch_distmult_relation_prepare's contract: Q = w conj(h) t
int launch_hole_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* Q,
                                 float* gold_sig, int32_t* gold_col, cudaStream_t st);
// 1-N query backward in launch_onen_query_bwd's contract (dQ is never null)
int launch_hole_query_bwd(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                          const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                          cudaStream_t st);

// conve.cu -- the ConvE query network (DESIGN.md section 1): d = h w, image 2h x w, C filters 3x3, F = C (2h-2)(w-2)
// feature columns stored with leading dimension Fp (F rounded up to 4).  Masks are uint8 keep-masks or null.
// Feature rows Feat [n, Fp] of the queries X[t] (anchor in column acol, relation row rel[X[t][1]])
int launch_conve_conv_fwd(const float* codes, const float* rel, int d, int h, int C, const int32_t* X, int acol,
                          int64_t n, const float* filt, const float* cbias, const uint8_t* in_mask, float inv_in,
                          const uint8_t* feat_mask, float inv_feat, int Fp, float* Feat, cudaStream_t st);
// Q = relu((Q + b) hid_mask / keep) in place, Q [n, d]
int launch_conve_fc_act(float* Q, int64_t n, int d, const float* b, const uint8_t* hid_mask, float inv_hid,
                        cudaStream_t st);
// dZ [m, d] and dZt [d, ldt] (columns m..ldt-1 zero) = dQ [Q > 0] hid_mask / keep
int launch_conve_dz(const float* Q, const float* dQ, int64_t m, int d, const uint8_t* hid_mask, float inv_hid,
                    float* dZ, float* dZt, int64_t ldt, cudaStream_t st);
// db (+)= the row sums of dZt [d, m] (leading dimension ldt), each in a fixed order
int launch_conve_rowsum(const float* dZt, int d, int64_t m, int64_t ldt, float* db, int accumulate, cudaStream_t st);
// convolution backward: conve_conv_parts(m) filter / bias gradient parts [parts, 10 C] into part, the image gradient
// red.add into dcodes[anchor = X[t][0]] and drel[X[t][1]]
int64_t conve_conv_parts(int64_t m);
int64_t conve_smem_bytes(int d, int h, int w, int C);
int launch_conve_conv_bwd(const float* codes, const float* rel, int d, int h, int C, const int32_t* X, int64_t m,
                          const float* filt, const uint8_t* in_mask, float inv_in, const float* Feat, const float* dF,
                          float inv_feat, int Fp, float* part, float* dcodes, float* drel, cudaStream_t st);
// dfilt [C, 9] / dbias [C] (+)= the sum of the parts in part order
int launch_conve_filter_reduce(const float* part, int parts, int C, float* dfilt, float* dbias, int accumulate,
                               cudaStream_t st);
// pre-split of W [F, d] zero-padded to Fp rows: transposed = 1 -> [d, Fp], 0 -> [Fp, d]
int launch_conve_split_w(const float* W, int F, int d, int Fp, int transposed, float* hi, float* lo, cudaStream_t st);
// dW [F, d] = dWt [d, Fp]^T (first F columns)
int launch_conve_transpose(const float* dWt, int F, int d, int Fp, float* dW, cudaStream_t st);
// gold_sig[t] = sigmoid(<Q[t], codes[gold]>), gold = X[t][0] (side 0) or X[t][2] (side 1)
int launch_conve_gold(const float* Q, const float* codes, int d, const int32_t* X, int64_t n, int side,
                      float* gold_sig, int32_t* gold_col, cudaStream_t st);
// dst = g_scale[0] src, any count
int launch_conve_scale(const float* src, const float* g_scale, int64_t count, float* dst, cudaStream_t st);
