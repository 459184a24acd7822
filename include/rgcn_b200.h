/*
 * rgcn_b200.h -- C-ABI of librgcn_b200.so: the H100-native (sm_90a) R-GCN relational
 * message-passing hot path (block-diagonal + basis decomposition, forward and backward) and the
 * DistMult triple scorer.
 *
 * The reference (MichSchli/RelationPrediction) is pure Python/TensorFlow-1 and has no FFI; its
 * "operator interface" for this path is the set of plugin hooks that build a TF graph.  Each entry
 * point below cites the reference hook(s) (file:line under the reference's code/ directory) whose *executed*
 * TF ops it replaces.  INTEGRATION.md shows the ctypes binding a reference maintainer would add.
 *
 * Conventions
 *   - every function returns int: 0 = ok, negative = error (RGCN_ERR_*); rgcn_last_error() gives text.
 *   - no exceptions cross the boundary; no torch types; plain pointers + explicit sizes.
 *   - the caller owns every tensor (device pointers unless the name ends in _host); the library
 *     owns only the opaque graph handle.  `stream` is a cudaStream_t passed as void*.
 *   - all feature / weight tensors are dense row-major fp32; all indices are int32.
 *   - all calls are asynchronous with respect to the host (work is enqueued on `stream`).
 *   - a "message" is one (source row -> destination row, relation-weight id) item.  A triple
 *     (s, r, o) yields two messages: forward  s->o with weight id r       (W_forward[r])
 *                                    backward o->s with weight id r + R   (W_backward[r])
 *     (reference: extras/graph_representations.py:21-27, message_gcn.py:28-42).
 */
#ifndef RGCN_B200_H
#define RGCN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RGCN_OK 0
#define RGCN_ERR_INVALID (-1)   /* bad argument (shape, null pointer, index out of range)      */
#define RGCN_ERR_CUDA (-2)      /* CUDA runtime / cuBLAS failure; text in rgcn_last_error()    */
#define RGCN_ERR_NOMEM (-3)     /* host or device allocation failed                            */
#define RGCN_ERR_WORKSPACE (-4) /* caller workspace too small (see *_workspace_bytes)          */
#define RGCN_ERR_NODEVICE (-5)  /* device entry point called on a host-only graph / no GPU     */

/* normalisation modes for rgcn_graph_create (extras/graph_representations.py:84-93,124-133) */
#define RGCN_NORM_CANONICAL 0 /* 1 / (#messages of that direction into the destination)        */
#define RGCN_NORM_EXPLICIT 1  /* caller supplies norm_f[E], norm_b[E] (e.g. tf_unsorted_compat) */
#define RGCN_NORM_NONE 2      /* all ones ('none' branch, :70-82)                               */

typedef struct rgcn_graph rgcn_graph_t; /* opaque */

int rgcn_version(void);
const char* rgcn_last_error(void);
/* number of CUDA kernels this library has launched in this process (bench.py "gpu_launches") */
int64_t rgcn_launch_count(void);

/* Library options.  "block_algo": 0 = destination-major aggregation (deterministic summation order,
 * epilogue fused), 1 = weight-id-major aggregation with the gathered rows in registers (block weights in
 * registers, vector reductions in L2; fp32 summation order not reproducible run to run), 3 = the same walk with the
 * gathered rows staged through shared memory by TMA bulk copies / cp.async (block sizes 4, 8, 16; fastest),
 * -1 = auto (default): 3 where the block size allows, else 1, else 0.
 * The environment variable RGCN_BLOCK_ALGO overrides the option.
 * "graph_views": which sorted views GPU-prepared graphs created AFTER the call get: 1 = the two CSR views
 * (deterministic block mode, basis layers), 2 = the two weight-id-major views (default block kernels),
 * 3 = all four (default).  A 200 M-message graph saves ~5 GB and half its preparation time with 2; entry
 * points return RGCN_ERR_INVALID when the view they walk is absent. */
int rgcn_set_option(const char* name, int64_t value);

/* Dense fp32-accurate GEMM on the Hopper tensor cores (wgmma, 3xTF32 split, register accumulators):
 *   C[M,N] = (accumulate ? C : 0) + A[M,K] * op(B),   op(B) = B[K,N] (b_is_nk = 0) or B[N,K]^T (b_is_nk = 1)
 * all row-major fp32 device pointers; K, N and the leading dimensions must be multiples of 4.
 * workspace: 2*N*K floats (the hi/lo split of B).  This is the kernel the layer entry points use for
 * the self-loop terms (gcn_basis.py:70-71 / gcn_basis_concat.py:65-66). */
int rgcn_gemm_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, int b_is_nk, float* C,
                     int64_t ldc, int32_t M, int32_t N, int32_t K, int accumulate, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* C[M,N] = (accumulate ? C : 0) + A^T B with A [K,M], B [K,N] row-major (the V-long reductions of
 * the backward pass: dW_self = H^T dS).  Same tensor-core path, both operands MN-major, split-K with
 * vector reductions into C (fp32 summation order across splits not reproducible run to run).
 * M, N and the leading dimensions must be multiples of 4. */
int rgcn_gemm_tn_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc,
                        int32_t M, int32_t N, int32_t K, int accumulate, void* stream);

/* Host-side neighbourhood-expansion edge sampler (next row N2; train.py:161-198): writes sample_size
 * DISTINCT edge ids.  Same stochastic process as the reference (vertex ~ unpicked-degree x seen, then a
 * uniform unpicked incident edge), O(log V) per draw instead of O(V); its own random stream (seed). */
int rgcn_sample_edge_neighborhood(const int32_t* triples_host, int64_t E, int32_t V, int64_t sample_size,
                                  uint64_t seed, int32_t* out_edges_host);

/* The same sampler with the per-dataset incidence structure built once: create a handle for the training
 * triples, then draw any number of samples from it.  Draws are thread-compatible (the handle is read-only, every
 * draw owns its scratch copies), so host threads can prepare samples concurrently.  A draw with the same seed
 * returns exactly what rgcn_sample_edge_neighborhood returns. */
typedef struct rgcn_sampler rgcn_sampler_t;
int rgcn_sampler_create(const int32_t* triples_host, int64_t E, int32_t V, rgcn_sampler_t** out);
int rgcn_sampler_draw(const rgcn_sampler_t* sampler, int64_t sample_size, uint64_t seed, int32_t* out_edges_host);
/* One whole training sample of train.py:140-198 in one call (so that the host threads preparing samples hold no
 * interpreter lock): batch = rgcn_sampler_draw(batch) edges; graph_split_host [split,3] = `split` of them uniformly
 * without replacement (np.random.choice(ids, split, replace=False)); X_host [(neg_rate+1)*batch, 3] / Y_host = the batch
 * followed by neg_rate corrupted copies with labels 1 / 0 (common/auxilliaries.py NegativeSampler.transform: fair coin
 * object-or-subject, uniform replacement entity).  Same stochastic process, own random stream. */
int rgcn_sampler_draw_batch(const rgcn_sampler_t* sampler, int32_t batch, int32_t split, int32_t neg_rate, uint64_t seed,
                            int32_t* graph_split_host, int32_t* X_host, float* Y_host);
void rgcn_sampler_destroy(rgcn_sampler_t* sampler);

/* Next row N1: global-norm clipping + Adam with TensorFlow-1.x semantics
 * (optimization/tensorflow_backend/algorithms.py:65-68 and :36-42).  Call rgcn_sumsq_accumulate on every
 * gradient tensor into one zeroed device float, then rgcn_adam_update on every (param, grad, m, v) with that
 * scalar: scale = max_norm * min(1/sqrt(sumsq), 1/max_norm) (skipped when sumsq_dev is NULL or max_norm <= 0);
 * lr_t = lr*sqrt(1-beta2^step)/(1-beta1^step); p -= lr_t * m / (sqrt(v) + eps).  step is 1-based. */
int rgcn_sumsq_accumulate(const float* g, int64_t n, float* acc_dev, void* stream);
int rgcn_adam_update(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1,
                     float beta2, float eps, int64_t step, const float* sumsq_dev, float max_norm,
                     void* stream);

/* Optional per-kernel timing (bench.py roofline): when enabled, every layer entry point records a
 * CUDA event on its stream after each internal stage.  rgcn_profile_read() synchronises, writes
 * the stage durations (ms) and their '\n'-separated names, clears the log and returns the count. */
int rgcn_profile_enable(int enable);
int rgcn_profile_read(float* ms_out, int max_entries, char* names_out, int names_cap);

/* ------------------------------------------------------------------------------------------------
 * Graph preparation.  Replaces Representation/MessageGraph
 * (extras/graph_representations.py:21-27 index vectors, :84-93 / :124-133 normalised incidence).
 *
 * triples_host : int32 [E,3], columns (subject, relation, object), host memory.
 * V            : number of entities (rows of H); R: number of relations.
 * device       : CUDA device ordinal, or -1 to build the host-side structure only (CPU tests).
 * Builds, deterministically (stable counting sorts; message id of triple k is k forward, E+k
 * backward): destination-CSR sorted by (dst, weight-id), source-CSR sorted by (src, weight-id),
 * two weight-id-major lists sorted by (supertile(dst), weight-id, dst) and (supertile(src),
 * weight-id, src), per-message norm, and warp work lists.
 * ---------------------------------------------------------------------------------------------- */
int rgcn_graph_create(const int32_t* triples_host, int64_t E, int32_t V, int32_t R, int norm_mode,
                      const float* norm_f_host, const float* norm_b_host, int device, void* stream,
                      rgcn_graph_t** out);

/* Generic message-list constructor used by the 1-D node-sharded path (SURVEY.md 8e): rank-local
 * destinations [0,V_dst), sources index an extended row space [0,V_src) (local rows then halo
 * rows).  All arrays host, length M.  relw in [0, n_relw). */
int rgcn_graph_create_messages(const int32_t* dst_host, const int32_t* src_host,
                               const int32_t* relw_host, const float* norm_host, int64_t M,
                               int32_t V_dst, int32_t V_src, int32_t n_relw, int device,
                               void* stream, rgcn_graph_t** out);

/* The same two constructors for index arrays that ALREADY live on `device` (int32 / float device pointers,
 * same shapes and meaning as the _host arguments above): the node-sharded path partitions the edge list on
 * the GPU and bench.py generates its synthetic graphs there, so a 100 M-edge list never visits the host.
 * GPU preparation only (device must be >= 0); the arrays are read on `stream` and may be freed by the caller
 * as soon as the call returns.  Replaces the same reference code as rgcn_graph_create
 * (extras/graph_representations.py:21-27, :84-93, :124-133). */
int rgcn_graph_create_device(const int32_t* triples_dev, int64_t E, int32_t V, int32_t R, int norm_mode,
                             const float* norm_f_dev, const float* norm_b_dev, int device, void* stream,
                             rgcn_graph_t** out);
int rgcn_graph_create_messages_device(const int32_t* dst_dev, const int32_t* src_dev,
                                      const int32_t* relw_dev, const float* norm_dev, int64_t M,
                                      int32_t V_dst, int32_t V_src, int32_t n_relw, int device,
                                      void* stream, rgcn_graph_t** out);

/* Opt-in stream-ordered destroy: GPU-prepared graphs return their arrays with cudaFreeAsync on `stream` (no
 * device synchronisation); every kernel that used the graph must be ordered before `stream`'s tail.  Host-prepared
 * graphs take the synchronous path of rgcn_graph_destroy. */
int rgcn_graph_destroy_async(rgcn_graph_t* graph, void* stream);
int rgcn_graph_destroy(rgcn_graph_t* g);

/* info[0]=M messages, [1]=V_dst, [2]=V_src, [3]=n_relw, [4]=#dst work items, [5]=#src work items,
 * [6]=#relw work items, [7]=#split dst rows, [8]=#split src rows, [9]=#(dst,relw) groups,
 * [10]=device, [11]=bytes resident on device, [12]=item_max, [13]=supertile rows, [14]=#supertiles,
 * [15]=#relw work items of the source-keyed view. */
int rgcn_graph_info(const rgcn_graph_t* g, int64_t info[16]);

/* Export of the prepared structure to host memory, for bit-exact index tests. */
enum {
  RGCN_X_DST_ROWPTR = 0, /* int32 [V_dst+1] */
  RGCN_X_DST_SRC = 1,    /* int32 [M]  source row of each message, destination-major order */
  RGCN_X_DST_RELW = 2,   /* int32 [M]  */
  RGCN_X_DST_NORM = 3,   /* float [M]  */
  RGCN_X_DST_MID = 4,    /* int32 [M]  original message id (k or E+k)                      */
  RGCN_X_SRC_ROWPTR = 5, /* int32 [V_src+1] */
  RGCN_X_SRC_DST = 6,
  RGCN_X_SRC_RELW = 7,
  RGCN_X_SRC_NORM = 8,
  RGCN_X_SRC_MID = 9,
  RGCN_X_REL_PTR = 10, /* int32 [n_super*n_relw+1]: weight-id major view keyed (supertile(dst), relw, dst) */
  RGCN_X_REL_DST = 11,
  RGCN_X_REL_SRC = 12,
  RGCN_X_REL_NORM = 13,
  RGCN_X_REL_MID = 14,
  RGCN_X_MSG_NORM = 15, /* float [M] norm in original message order */
  RGCN_X_REL2_PTR = 16, /* second weight-id major view keyed (supertile(src), relw, src) */
  RGCN_X_REL2_SRC = 17,
  RGCN_X_REL2_DST = 18,
  RGCN_X_REL2_NORM = 19,
  RGCN_X_REL2_MID = 20
};
int64_t rgcn_graph_export_bytes(const rgcn_graph_t* g, int which);
int rgcn_graph_export(const rgcn_graph_t* g, int which, void* dst_host, int64_t nbytes);

/* ------------------------------------------------------------------------------------------------
 * Block-diagonal R-GCN layer ("ConcatGcn", encoders/message_gcns/gcn_basis_concat.py:35-83 +
 * message_gcn.py:49-79).
 *
 *   out[v,:] = act( sum_{messages m into v} norm_m * blockdiag(W[relw_m]) . H[src_m,:]
 *                   + dropout(H[v,:] @ W_self) )
 *
 * H      : [V_src, d]   (rows [0,V_dst) are the local nodes: the self-loop uses those)
 * Wf, Wb : [R, B, s, s], s = d / B, "W . x" orientation (gcn_basis_concat.py:46-47):
 *          y[b*s+i] = sum_j W[r,b,i,j] * x[b*s+j].      n_relw of the graph must equal 2R.
 * Wself  : [d, d]
 * drop_mask : uint8 [V_dst, d] keep-mask (1 = keep) or NULL; survivors are scaled by 1/keep
 *          (tf.nn.dropout semantics, message_gcn.py:64; self-loop only).
 * relu   : 1 for hidden layers, 0 for the last layer (common/model_builder.py:275).
 * out    : [V_dst, d].
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_block_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward);

int rgcn_block_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                       const float* Wf, const float* Wb, const float* Wself,
                       const uint8_t* drop_mask, float keep, int relu, float* out, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* Backward of the above (what tf.gradients, optimization/abstract.py:117-118, derives):
 *   G = dOut * (out > 0 if relu);  dS = G * mask / keep
 *   dH      [V_src, d]  (overwritten)   dWf, dWb [R,B,s,s] (overwritten)   dWself [d,d] (overwritten)
 * `out` is the forward result (needed for the ReLU mask only when relu != 0). */
int rgcn_block_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                        const float* Wf, const float* Wb, const float* Wself,
                        const uint8_t* drop_mask, float keep, int relu, const float* out,
                        const float* dOut, float* dH, float* dWf, float* dWb, float* dWself,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* Messages-only parts of the block layer, for graphs whose sources live in a separate row space
 * (the halo rows of the node-sharded path: V_src may be smaller than V_dst):
 *   aggregate          : out[dst,:] += sum_m norm_m * blockdiag(W[relw_m]) . X[src_m,:]      (no self loop)
 *   aggregate_backward : dX [V_src,d] (overwritten) = sum_m norm_m W^T G[dst_m];
 *                        dWf, dWb (overwritten, or += when accumulate_dW) = block outer products.
 * Same per-message arithmetic as gcn_basis_concat.py:35-52 + the SpMMs of :69-75. */
int64_t rgcn_block_aggregate_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward);
int rgcn_block_aggregate(const rgcn_graph_t* g, int32_t d, int32_t B, const float* X, const float* Wf,
                         const float* Wb, float* out, void* workspace, int64_t workspace_bytes,
                         void* stream);
int rgcn_block_aggregate_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* X,
                                  const float* Wf, const float* Wb, const float* G, float* dX,
                                  float* dWf, float* dWb, int accumulate_dW, void* workspace,
                                  int64_t workspace_bytes, void* stream);

/* dst[rows[i], :] += src[i, :] for i < n, rows (int64, device) UNIQUE within the call -- no atomics.  The
 * node-sharded path returns halo gradients grouped by peer; a local row gets at most one contribution per peer,
 * so each peer segment is one call (replaces an atomic index_add over 16 GB per rank at 8 GPUs). */
int rgcn_rows_add(float* dst, const int64_t* rows, const float* src, int64_t n, int32_t d, void* stream);

/* G[i] = out[i] > 0 ? dOut[i] : 0 for i < n (n % 4 == 0): the ReLU gradient of message_gcn.py:64-66 as its own pass.
 * rgcn_block_backward applies it internally; the node-sharded layers need G before their first backward kernel
 * (the halo-source messages run first so that their gradients can travel while the local work runs). */
int rgcn_relu_backward(const float* dOut, const float* out, float* G, int64_t n, void* stream);

/* dst[i, :] = src[rows[i], :] for i < n (rows int64, device).  The halo PUSH of the node-sharded path: `dst` may be
 * (and in that path is) a PEER GPU's buffer mapped into this process (CUDA symmetric / IPC memory), so the rows a
 * peer needs go from H straight over NVLink into the buffer its aggregation kernel reads -- no packed send buffer,
 * no all-to-all (the reference has no multi-device path at all: model.py builds one tf.Session graph).
 * max_ctas > 0 bounds the grid so the push shares the GPU with the layer's local work; 0 = library default. */
int rgcn_rows_gather(float* dst, const float* src, const int64_t* rows, int64_t n, int32_t d, int32_t max_ctas,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Basis-decomposition R-GCN layer ("BasisGcn", encoders/message_gcns/gcn_basis.py:39-88).
 *
 *   m_f[k] = sum_b Cf[r_k,b] * (H[s_k,:] @ Vf[:,b,:])   (and likewise backward with Vb, Cb)
 *   out    = act( A_f m_f + A_b m_b + dropout(H @ W_self) )
 *
 * computed re-associated (aggregate-then-transform): Agg_dir[v,k,b] = sum_m norm_m C[relw_m,b] H[src_m,k]
 * followed by dense GEMMs with Vf/Vb viewed as [d_in*B, d_out].
 * Vf, Vb : [d_in, B, d_out] (gcn_basis.py:18);  Cf, Cb : [R, B] (gcn_basis.py:17).  d_in == d_out == d.
 * `saved` (float [V_dst, 2*d*B]) receives Agg_f | Agg_b and must be handed unchanged to backward.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_basis_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward);

int rgcn_basis_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                       const float* Vf, const float* Vb, const float* Cf, const float* Cb,
                       const float* Wself, const uint8_t* drop_mask, float keep, int relu,
                       float* out, float* saved, void* workspace, int64_t workspace_bytes,
                       void* stream);

int rgcn_basis_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                        const float* Vf, const float* Vb, const float* Cf, const float* Cb,
                        const float* Wself, const uint8_t* drop_mask, float keep, int relu,
                        const float* out, const float* saved, const float* dOut, float* dH,
                        float* dVf, float* dVb, float* dCf, float* dCb, float* dWself,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * One-hot (featureless) basis layer: layer 0 of the gcn_basis encoder with UseInputTransform=No
 * (model_builder.py:140-168, :277-283: Representation -> BasisGcn(onehot_input=True)).  With one-hot input
 * dot_or_lookup is an embedding lookup (shared_functions.py:5-9, gcn_basis.py:15-71, message_gcn.py:28-79):
 *
 *   out[v] = act( sum_dir sum_{m -> v} norm_m sum_b C_dir[r_m,b] W_dir[u_m,b,:]  +  dropout(W_self[v]) )
 *
 * Wf, Wb : [V_src, B, d] (vertex_feature_dimension = EntityCount);  Cf, Cb : [R, B];  Wself : [V_dst, d].
 * Backward:  G = dOut * relu'(out),  dW_dir[u,b,:] = sum_{m from u} norm_m C_dir[r_m,b] G[v_m,:],
 *            dC_dir[r,b] = sum_{m: r_m = r} norm_m < W_dir[u_m,b,:], G[v_m,:] >,  dWself = G * mask / keep.
 * The layer has no input, hence no input gradient.  Every dW row is written (rows without messages are zero).
 * Both calls walk the source-major CSR view: a graph prepared with graph_views = 2 is rejected (RGCN_ERR_INVALID).
 * Argument rules as rgcn_basis_*: d % 4 == 0, B >= 1, keep > 0, drop_mask uint8 [V_dst, d] or NULL.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_basis_onehot_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward);

int rgcn_basis_onehot_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* Wf, const float* Wb,
                              const float* Cf, const float* Cb, const float* Wself, const uint8_t* drop_mask,
                              float keep, int relu, float* out, void* workspace, int64_t workspace_bytes,
                              void* stream);

int rgcn_basis_onehot_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* Wf, const float* Wb,
                               const float* Cf, const float* Cb, const uint8_t* drop_mask, float keep, int relu,
                               const float* out, const float* dOut, float* dWf, float* dWb, float* dCf,
                               float* dCb, float* dWself, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes, "BasisGcnTimesDiag",
 * encoders/message_gcns/gcn_basis_times_diag.py with message_gcn.py:49-79), feature input:
 *
 *   P_dir  = H @ V_dir.reshape(d, B*d)                                   ([V_src, B, d] per direction)
 *   m      = sum_b sigmoid(C_dir[r_m,b,:]) * P_dir[u_m,b,:]              (per output channel)
 *   out    = act( A_f m_f + A_b m_b + dropout(H @ W_self) + b )
 *
 * Vf, Vb : [d, B, d];  Cf, Cb : [R, B, d];  Wself : [d, d];  b, db : [d].  `saved` (float [V_src, 2*B*d]) receives
 * P_f | P_b per row and must be handed unchanged to backward.
 * Backward:  G = dOut * relu'(out),  dS = G * mask / keep,  dWself = H^T dS,  db = column sums of G,
 *            dP_dir[u,b,:] = sum_{m from u} norm_m sigmoid(C[r_m,b,:]) * G[v_m,:],  dV_dir = H^T dP_dir,
 *            dH = dS W_self^T + sum_dir dP_dir V_dir^T,
 *            dC_dir[r,b,:] = s (1 - s) * sum_{m: r_m = r} norm_m P_dir[u_m,b,:] * G[v_m,:]   (s = sigmoid(C)).
 * Every output is overwritten.  The forward walks the destination-major CSR view, the backward both CSR and the
 * weight-id-major views: a graph prepared without all of them (graph_views != 3) is RGCN_ERR_INVALID.
 * Arguments are checked before any device work: null pointers, d % 4 != 0, B < 1 or keep <= 0 are RGCN_ERR_INVALID,
 * a short workspace RGCN_ERR_WORKSPACE; a host-only graph is RGCN_ERR_NODEVICE.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_basis_diagcoef_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward);

int rgcn_basis_diagcoef_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H, const float* Vf,
                                const float* Vb, const float* Cf, const float* Cb, const float* Wself, const float* b,
                                const uint8_t* drop_mask, float keep, int relu, float* out, float* saved,
                                void* workspace, int64_t workspace_bytes, void* stream);

int rgcn_basis_diagcoef_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H, const float* Vf,
                                 const float* Vb, const float* Cf, const float* Cb, const float* Wself,
                                 const uint8_t* drop_mask, float keep, int relu, const float* out, const float* saved,
                                 const float* dOut, float* dH, float* dVf, float* dVb, float* dCf, float* dCb,
                                 float* dWself, float* db, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Diagonal R-GCN layer (Name=gcn_diag, "DiagGcn", encoders/message_gcns/gcn_diag.py with message_gcn.py:49-79).
 * Messages as above (forward s->o with weight id r, backward o->s with weight id r+R), D = [Df; Db]:
 *
 *   out[v] = act( sum_{m -> v} norm_m * D[w_m] (.) H[src_m]  +  dropout(H[v] @ W_self)  +  b )
 *
 * H : [V_src, d] (V_src >= V_dst: rows [V_dst, V_src) are halo rows that only send);  Df, Db : [R, d] with
 * n_relw == 2R;  Wself : [d, d];  b, db : [d];  out, dOut : [V_dst, d].  d % 4 == 0.
 * Backward:  G = dOut * relu'(out),  dS = G * mask / keep,  db = column sums of G,  dWself = H^T dS,
 *            dH[u] = (dS W_self^T)[u] + sum_{m from u} norm_m D[w_m] (.) G[dst_m],
 *            dD[w] = sum_{m: w_m = w} norm_m G[dst_m] (.) H[src_m].
 * slice_sumsq2 (optional, float[2]; NULL skips it) receives, per direction, the sum of squares of the un-aggregated
 * per-message gradient slices of Df / Db (what tf.clip_by_global_norm sees through tf.nn.embedding_lookup):
 *            sum_m norm_m^2 sum_k G[dst_m,k]^2 H[src_m,k]^2.
 * Every output is overwritten.  The forward walks the destination-major CSR view, the backward the source-major one:
 * a graph prepared without the CSR views (graph_views == 2) is RGCN_ERR_INVALID.
 * Arguments are checked before any device work: null pointers, d % 4 != 0 or keep <= 0 are RGCN_ERR_INVALID, a short
 * workspace RGCN_ERR_WORKSPACE; a host-only graph is RGCN_ERR_NODEVICE.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_diag_workspace_bytes(const rgcn_graph_t* g, int32_t d, int backward);

int rgcn_diag_forward(const rgcn_graph_t* g, int32_t d, const float* H, const float* Df, const float* Db,
                      const float* Wself, const float* b, const uint8_t* drop_mask, float keep, int relu, float* out,
                      void* workspace, int64_t workspace_bytes, void* stream);

int rgcn_diag_backward(const rgcn_graph_t* g, int32_t d, const float* H, const float* Df, const float* Db,
                       const float* Wself, const uint8_t* drop_mask, float keep, int relu, const float* out,
                       const float* dOut, float* dH, float* dDf, float* dDb, float* dWself, float* db,
                       float* slice_sumsq2, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Highway skip connection between R-GCN layers (SkipConnections=Highway, model_builder.py:304-305;
 * extras/highway_layer.py:14-38).  c1 = the wrapped layer's output, c2 = the layer's input:
 *
 *   g = sigmoid(c2 W + b),   out = g * c1 + (1 - g) * c2          (highway_layer.py:21, :34-38)
 *
 * c1, c2, out, gate, dOut, dc1, dc2 : [V, d];  W, dW : [d, d] (z = c2 W, W indexed [in, out]);  b, db : [d].
 * The forward is one gate GEMM with the blend in its epilogue; `gate` (g) is written for the backward pass.
 * Backward:  dc1 = g dOut,  dz = dOut (c1 - c2) g (1 - g),  dc2 = (1 - g) dOut + dz W^T,  dW = c2^T dz,
 *            db = column sums of dz.  Every output is overwritten (dc2 does not include the gradient c2 receives
 *            through the wrapped layer).
 * Arguments are checked before any device work: null pointers, V < 0 or d <= 0 or d % 4 != 0 are RGCN_ERR_INVALID,
 * a short workspace RGCN_ERR_WORKSPACE.  V = 0 does nothing.  No device: RGCN_ERR_NODEVICE.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_highway_workspace_bytes(int64_t V, int32_t d, int backward);

int rgcn_highway_forward(const float* c1, const float* c2, const float* W, const float* b, int64_t V, int32_t d,
                         float* out, float* gate, void* workspace, int64_t workspace_bytes, void* stream);

int rgcn_highway_backward(const float* c1, const float* c2, const float* W, const float* gate, const float* dOut,
                          int64_t V, int32_t d, float* dc1, float* dc2, float* dW, float* db, void* workspace,
                          int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Variational head of the variational encoders (Name=variational_embedding / variational_gcn_basis,
 * model_builder.py:43-69, :186-254; extras/variational_encoding.py:14-31).  With l = log sigma:
 *
 *   z = mu + exp(l) * eps,    kl[0] = -0.0005 * sum over all V x w elements of (1 + 2 l - mu^2 - exp(2 l))
 *
 * Embedding variant (H == NULL, d == 0): mu = W_mu, l = W_sigma, both [V, w]; b_mu, b_sigma, P, dH, db_mu and
 * db_sigma are not used and may be NULL.
 * Gcn variant (H [V, d], d > 0): mu = H W_mu + b_mu, l = H W_sigma + b_sigma with W_mu, W_sigma [d, w] and b_mu,
 * b_sigma [w]; one 3xTF32 GEMM over the interleaved weight computes both and writes P [V, 2w] = (mu, l) interleaved
 * per element (P[v, 2j] = mu[v, j], P[v, 2j + 1] = l[v, j]), which the backward pass reads.
 * eps, z, dz : [V, w].  eps is drawn by the caller (N(0, 1)).
 * Backward, g = g_kl[0] (device memory, the incoming gradient of kl):
 *   dmu = dz + 0.001 g mu,  dl = dz exp(l) eps + 0.001 g (exp(2 l) - 1);
 *   embedding: dW_mu = dmu, dW_sigma = dl;  gcn: db = column sums of dmu / dl, dW = H^T dmu / H^T dl,
 *   dH = dmu W_mu^T + dl W_sigma^T.  Every output is overwritten.
 * kl and the db column sums are reduced in a fixed order (bitwise repeatable).
 * Arguments are checked before any device work: null pointers, H == NULL while d != 0 (or the reverse), V < 0,
 * d % 4 != 0 or w <= 0 or w % 4 != 0 are RGCN_ERR_INVALID, a short workspace RGCN_ERR_WORKSPACE, no device
 * RGCN_ERR_NODEVICE.  rgcn_variational_workspace_bytes takes d = 0 for the embedding variant.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_variational_workspace_bytes(int64_t V, int32_t d, int32_t w, int backward);

int rgcn_variational_forward(const float* H, int64_t V, int32_t d, int32_t w, const float* W_mu, const float* b_mu,
                             const float* W_sigma, const float* b_sigma, const float* eps, float* z, float* P,
                             float* kl, void* workspace, int64_t workspace_bytes, void* stream);

int rgcn_variational_backward(const float* H, int64_t V, int32_t d, int32_t w, const float* W_mu,
                              const float* W_sigma, const float* P, const float* eps, const float* dz,
                              const float* g_kl, float* dH, float* dW_mu, float* db_mu, float* dW_sigma,
                              float* db_sigma, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * DistMult triple scorer ("BilinearDiag", decoders/bilinear_diag.py:14-34, :63-69).
 *
 *   energy[n] = sum_k codes[X[n,0],k] * rel[X[n,1],k] * codes[X[n,2],k]
 *   loss_out[0] = mean_n( (1-y)x + log1p(exp(-|x|)) + max(-x,0) )            (only if Y != NULL)
 *   loss_out[1] = mean(e1^2) + mean(r^2) + mean(e2^2) over the gathered rows  (un-scaled; the
 *                 caller multiplies by RegularizationParameter, bilinear_diag.py:69)
 * codes : [V, d]; rel : [Vrel, d] (the reference sizes it [EntityCount, d], model_builder.py:134);
 * X : int32 [N,3] device; Y : float [N] device or NULL; energies : float [N]; loss_out : float [2].
 * ---------------------------------------------------------------------------------------------- */
int distmult_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                     const int32_t* X, int64_t N, const float* Y, float* energies, float* loss_out,
                     void* stream);

/* Backward: given upstream scalars g_loss (d total / d loss_out[0]) and g_reg (d total / d loss_out[1]),
 * optionally multiplied by DEVICE scalars g_scale_dev[2] (NULL = 1,1; lets an autograd engine pass
 * its upstream gradients without a host sync), and optionally a per-triple upstream gradient
 * g_energy[N] (NULL = none), ACCUMULATES (+=) into dcodes [V,d] and drel [Vrel,d] (the caller
 * zeroes them when it wants plain gradients). */
int distmult_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                      const int32_t* X, int64_t N, const float* Y, const float* energies,
                      float g_loss, float g_reg, const float* g_scale_dev, const float* g_energy,
                      float* dcodes, float* drel, void* stream);

/* Same as distmult_backward, additionally accumulating (+=) into the device float rel_slice_sumsq (may be NULL) the
 * sum over triples of |gradient slice of the gathered relation row|^2 -- the contribution of the relation table to
 * tf.clip_by_global_norm, which sees that gradient as un-aggregated IndexedSlices (bilinear_diag.py:18,
 * optimization/tensorflow_backend/algorithms.py:65-68). */
int distmult_backward_slices(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                             const int32_t* X, int64_t N, const float* Y, const float* energies, float g_loss,
                             float g_reg, const float* g_scale_dev, const float* g_energy, float* dcodes,
                             float* drel, float* rel_slice_sumsq, void* stream);

/* IndexedSlices norm of the block tables' gradients: sumsq2[0] (W_forward) and sumsq2[1] (W_backward), overwritten,
 * receive  sum_messages norm_m^2 * sum_b |G[dst_m]_b|^2 |H[src_m]_b|^2  -- the squared norm of the per-edge gradient
 * slices tf.gradients hands to tf.clip_by_global_norm for variables read through tf.nn.embedding_lookup
 * (gcn_basis_concat.py:38-39).  H [V_src,d] layer input, G [V_dst,d] = dOut * relu'(out). */
int64_t rgcn_block_slice_sumsq_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B);
int rgcn_block_slice_sumsq(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H, const float* G,
                           float* sumsq2, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * DistMult all-entity scoring + ranking, fused (next row N3): decoders/bilinear_diag.py:51-61
 * (predict_all_subject_scores / predict_all_object_scores) feeding the rank counts of
 * common/evaluation.py:148-159 and :355-367.  For every triple t of X and the corrupted side,
 *   score(t, v)      = sigmoid( sum_k q[t,k] * codes[v,k] ),  q = rel[r]*codes[o] (side 0: subjects) or
 *                      codes[s]*rel[r] (side 1: objects)
 *   raw_rank[t]      = #{ v : score(t, v) >= score(t, gold_t) }               (the gold entity counts itself)
 *   filtered_rank[t] = raw_rank[t] - #{ v in known(t) : score(t, v) >= score(t, gold_t) } + 1
 * The [n, V] score matrix the reference materialises per 1000-triple chunk is never written: the energies come
 * out of the wgmma 3xTF32 GEMM tile by tile and are compared in its epilogue.
 * known_mask : uint32 [n, ceil(V/32)] device, bit v of row t = v is a known true answer of t (the reference's
 *              known sets contain the evaluated triple itself, train.py:103-105), or NULL (then filtered_rank
 *              must be NULL).  raw_rank / filtered_rank : int32 [n] device.
 * workspace  : distmult_rank_workspace_bytes(V, d, n); its head holds the hi/lo split of `codes`:
 *              reuse_split != 0 skips re-splitting when the same workspace is passed again with unchanged codes.
 * ---------------------------------------------------------------------------------------------- */
int64_t distmult_rank_workspace_bytes(int32_t V, int32_t d, int64_t n);
int distmult_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d, const int32_t* X,
                  int64_t n, int side, const uint32_t* known_mask, int reuse_split, int32_t* raw_rank,
                  int32_t* filtered_rank, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * ComplEx triple scorer (decoders/complex.py).  Every row of width d is [real | imaginary] with h = d/2 columns
 * each (extract_real_and_imaginary, :71-75); d % 4 == 0 is required (then h is even), other widths return
 * RGCN_ERR_INVALID.  With a = codes[X[n,0]], b = rel[X[n,1]], c = codes[X[n,2]]:
 *
 *   energy[n] = sum_k ar*br*cr + ai*br*ci + ar*bi*ci - ai*bi*cr                 (:38-41)
 *   loss_out[0] = mean_n( (1-y)x + log1p(exp(-|x|)) + max(-x,0) )               (:43-45, only if Y != NULL)
 *   loss_out[1] = mean(a^2) + mean(b^2) + mean(c^2) over the gathered rows, all d columns  (:108-114, un-scaled;
 *                 the caller multiplies by RegularizationParameter)
 * Shapes, pointers and the backward's upstream gradients (g_loss, g_reg, g_scale_dev[2], g_energy[N]) are those of
 * distmult_forward / distmult_backward.  The backward ACCUMULATES (+=) into dcodes [V,d] and drel [Vrel,d]
 *   da = g [br cr + bi ci, br ci - bi cr],  db = g [ar cr + ai ci, ar ci - ai cr],  dc = g [ar br - ai bi, ai br + ar bi]
 * plus 2*g_reg*x/(N*d) each, and, when rel_slice_sumsq != NULL, adds to that device float the sum over triples of
 * |db|^2 (both halves): the relation table's IndexedSlices term of tf.clip_by_global_norm.
 * ---------------------------------------------------------------------------------------------- */
int rgcn_complex_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                         const int32_t* X, int64_t N, const float* Y, float* energies, float* loss_out,
                         void* stream);
int rgcn_complex_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                          const int32_t* X, int64_t N, const float* Y, const float* energies, float g_loss,
                          float g_reg, const float* g_scale_dev, const float* g_energy, float* dcodes, float* drel,
                          float* rel_slice_sumsq, void* stream);

/* ComplEx all-entity scoring + ranking, fused: predict_all_subject_scores / predict_all_object_scores
 * (complex.py:77-106) are one [n,d] x [d,V] product each, with the query rows
 *   side 0 (subjects corrupted): q = [br cr + bi ci, br ci - bi cr]      (c = codes[o] kept, gold = s)
 *   side 1 (objects corrupted):  q = [ar br - ai bi, ai br + ar bi]      (a = codes[s] kept, gold = o)
 * and the same counting rules, known-mask format, split reuse and error codes as distmult_rank (workspace too
 * small: RGCN_ERR_WORKSPACE). */
int64_t rgcn_complex_rank_workspace_bytes(int32_t V, int32_t d, int64_t n);
int rgcn_complex_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d, const int32_t* X,
                      int64_t n, int side, const uint32_t* known_mask, int reuse_split, int32_t* raw_rank,
                      int32_t* filtered_rank, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Ensemble ranking, fused (R-GCN+): the weighted sum of two models' scores (the reference's tools/ensemble.py
 * --method weighted_sum over Scorer.dump_all_scores files), without either [n, V] score matrix.  A member is a
 * DistMult or ComplEx decoder (decoder_x = RGCN_DECODER_*) over its own codes [V, d_x] and relation table
 * [Vrel_x, d_x]; both members share the V entities, their widths may differ.  For every triple t of X:
 *   s_X(t, v) = the float32 sigmoid score of member X's rank entry point (distmult_rank / rgcn_complex_rank)
 *   c(t, v)   = w s_A(t, v) + (1 - w) s_B(t, v)       in float64, separately rounded products and sum,
 *               1 - w formed once in double (the reference tool's Python arithmetic, bit for bit)
 *   G(t)      = w g_A(t) + (1 - w) g_B(t), g_X the member's gold score
 *   raw_rank[t]      = #{ v : c(t, v) >= G(t) }   (the gold entity counts itself)
 *   filtered_rank[t] = raw_rank[t] - #{ v in known(t) : c(t, v) >= G(t) } + 1
 * known_mask, side, X and the outputs as in distmult_rank.  weight = w must be finite and in [0, 1].
 * workspace  : rgcn_ensemble_rank_workspace_bytes(V, d_a, d_b, n); its head holds the hi/lo splits of codes_a and
 *              codes_b: reuse_split != 0 skips both when the same workspace is passed again with unchanged codes.
 * Errors, before any device work: RGCN_ERR_INVALID (unknown decoder kind, d_x % 4 != 0, bad weight, null pointers,
 * side, filtered ranks without a known mask), RGCN_ERR_WORKSPACE.  The *_workspace_bytes function returns
 * RGCN_ERR_INVALID (-1) on bad arguments.
 * ---------------------------------------------------------------------------------------------- */
#define RGCN_DECODER_DISTMULT 0
#define RGCN_DECODER_COMPLEX 1
int64_t rgcn_ensemble_rank_workspace_bytes(int32_t V, int32_t d_a, int32_t d_b, int64_t n);
int rgcn_ensemble_rank(int32_t decoder_a, const float* codes_a, const float* rel_a, int32_t Vrel_a, int32_t d_a,
                       int32_t decoder_b, const float* codes_b, const float* rel_b, int32_t Vrel_b, int32_t d_b,
                       int32_t V, double weight, const int32_t* X, int64_t n, int side, const uint32_t* known_mask,
                       int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Top-k entity prediction, fused: the k entities each query believes in most, without the [n, V] score matrix
 * that predict_all_subject_scores / predict_all_object_scores (bilinear_diag.py:51-61, complex.py:77-106)
 * materialise and Scorer.dump_all_scores (common/evaluation.py:391-408) writes out.  For every triple t of X:
 *   side 0 (predict subjects): q = rel[r] * codes[o]   (ComplEx: the rgcn_complex_rank side-0 row)
 *   side 1 (predict objects):  q = codes[s] * rel[r]   (ComplEx: the rgcn_complex_rank side-1 row)
 * the predicted column of X is not read.  energy(t, v) = sum_k q[k] * codes[v, k] (3xTF32 GEMM); the score is
 * sigmoid(energy) in float32.  ids[t, :] lists the entities in order of energy descending, the smaller id first on
 * ties (the energy keeps its order where the float32 sigmoid saturates to 1); energies[t, :] are their energies.
 * exclude_mask : uint32 [n, ceil(V/32)] device, bit v of row t = entity v never appears in row t (the known_mask
 *                format of distmult_rank), or NULL.
 * When fewer than k entities remain, the tail of the row is id -1, energy -inf.  1 <= k <= 128, else
 * RGCN_ERR_INVALID.  ids int32 [n, k], energies float32 [n, k] device.  The result is bitwise repeatable.
 * workspace  : rgcn_topk_workspace_bytes(V, d, n, k), linear in n (about 4 d + 8 k ceil(V/128) bytes per query; a
 *              caller with many queries over many entities calls in chunks).  Its head holds the hi/lo split of
 *              `codes` exactly as in distmult_rank's workspace: reuse_split != 0 skips re-splitting when the same
 *              workspace (or a rank workspace of the same codes) is passed again with unchanged codes.
 * Errors as distmult_rank: RGCN_ERR_INVALID (null pointers, d % 4 != 0, side, k), RGCN_ERR_WORKSPACE.
 * rgcn_topk_workspace_bytes returns RGCN_ERR_INVALID (-1) on bad arguments.
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_topk_workspace_bytes(int32_t V, int32_t d, int64_t n, int32_t k);
int distmult_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d, const int32_t* X,
                  int64_t n, int side, int32_t k, const uint32_t* exclude_mask, int reuse_split, int32_t* ids,
                  float* energies, void* workspace, int64_t workspace_bytes, void* stream);
int rgcn_complex_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d, const int32_t* X,
                      int64_t n, int side, int32_t k, const uint32_t* exclude_mask, int reuse_split, int32_t* ids,
                      float* energies, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Relation prediction, fused: (h, ?, t) queries scored against every relation.  Both decoders' energies are linear
 * in the relation row, so for every triple t = (h, r, t') of X
 *   DistMult: q = codes[h] * codes[t']
 *   ComplEx:  q = [hr tr + hi ti, hr ti - hi tr]    (h = codes[h], t = codes[t'], [real | imaginary] halves)
 * and energy(t, r) = sum_k q[k] * rel[r, k] (3xTF32 GEMM) equals the decoder's energy of (h, r, t').
 * Only the first R rows of `rel` are candidates: rows R..Vrel-1 (the R-GCN encoders keep a [V, d] relation table)
 * are never scored, counted or returned.  1 <= R <= Vrel, else RGCN_ERR_INVALID.
 *
 * *_relation_rank: the ranking rules of distmult_rank with relations in place of entities:
 *   raw_rank[t]      = #{r < R : sigmoid(energy(t, r)) >= sigmoid(energy(t, gold))}, gold = X[t, 1] in [0, R)
 *   filtered_rank[t] = raw_rank[t] - #{known r with score >= gold} + 1   (only when filtered_rank != NULL)
 *   known_mask : uint32 [n, ceil(R/32)] device, bit r of row t = (h, r, t') is a known triple; required for
 *                filtered ranks.
 *   workspace  : rgcn_relation_rank_workspace_bytes(R, d, n).
 * *_relation_topk: the k relations of highest energy per row, energy descending, the smaller relation id first on
 *   ties, never one whose bit is set in exclude_mask (uint32 [n, ceil(R/32)] device, or NULL); the tail of a row
 *   with fewer than k eligible relations is id -1, energy -inf.  1 <= k <= 128.  The relation column of X is not
 *   read.  ids int32 [n, k], energies float32 [n, k] device; bitwise repeatable.
 *   workspace  : rgcn_relation_topk_workspace_bytes(R, d, n, k), linear in n.
 * Both workspaces start with the hi/lo split of rel[0:R] in the same place, so reuse_split != 0 skips re-splitting
 * when a relation workspace (rank or top-k) is passed again with an unchanged relation table.  The split is not that
 * of the entity entry points: never pass an entity workspace with reuse_split != 0.
 * Errors: RGCN_ERR_INVALID (null pointers, V <= 0, d % 4 != 0, R out of range, k out of range, filtered ranks
 * without a known mask), RGCN_ERR_WORKSPACE.  The two *_workspace_bytes functions return RGCN_ERR_INVALID (-1) on
 * bad arguments (R <= 0, d % 4 != 0, n < 0, k out of range).
 * ---------------------------------------------------------------------------------------------- */
int64_t rgcn_relation_rank_workspace_bytes(int32_t R, int32_t d, int64_t n);
int distmult_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                           const int32_t* X, int64_t n, const uint32_t* known_mask, int reuse_split,
                           int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                           void* stream);
int rgcn_complex_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                               const int32_t* X, int64_t n, const uint32_t* known_mask, int reuse_split,
                               int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                               void* stream);
int64_t rgcn_relation_topk_workspace_bytes(int32_t R, int32_t d, int64_t n, int32_t k);
int distmult_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                           const int32_t* X, int64_t n, int32_t k, const uint32_t* exclude_mask, int reuse_split,
                           int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes, void* stream);
int rgcn_complex_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                               const int32_t* X, int64_t n, int32_t k, const uint32_t* exclude_mask, int reuse_split,
                               int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RGCN_B200_H */
