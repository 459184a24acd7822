// api.cu -- C-ABI entry points of librgcn_b200.so (see include/rgcn_b200.h).
// Orchestrates per-layer work on ONE stream: weight re-layout -> dense self-loop GEMM (own wgmma 3xTF32
// kernel, gemm_tf32x3.cu) -> warp-centric aggregation kernels.  No vendor-library compute anywhere.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "kernels.cuh"
#include "rgcn_b200.h"

namespace {

// GEMM dispatch.  Every dense product of the layers runs on this library's own wgmma 3xTF32 kernels
// (gemm_tf32x3.cu): the NT/NN forms (contraction along the contiguous dimension of A) through
// k_gemm_tf32x3 with the small operand B pre-split into hi/lo planes, the V-long reductions A^T B through
// k_gemm_tn_tf32x3.  There is NO library fallback: a shape the kernels do not cover is an explicit
// RGCN_ERR_INVALID (all layer entry points require d % 4 == 0, which makes every internal shape valid).
// Row-major: C[m,n] = op(A) op(B) + beta * C with beta in {0, 1};  split_ws: 2*n*k floats.
int gemm_any(cudaStream_t st, float* split_ws, bool ta, bool tb, int64_t m, int64_t n, int64_t k,
             const float* A, int64_t lda, const float* B, int64_t ldb, float beta, float* C, int64_t ldc) {
  if (m == 0 || n == 0) return RGCN_OK;
  if (beta != 0.f && beta != 1.f) {
    rgcn_set_error("gemm: beta must be 0 or 1");
    return RGCN_ERR_INVALID;
  }
  if (k == 0) {
    if (beta == 0.f)
      return rgcn_check_cuda(cudaMemset2DAsync(C, ldc * sizeof(float), 0, n * sizeof(float), m, st), "memset2d");
    return RGCN_OK;
  }
  const bool aligned = n % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ldc % 4 == 0;
  if (ta && !tb && aligned && m % 4 == 0 && k < 0x7fffffffLL && m < 0x7fffffffLL && n < 0x7fffffffLL)
    return launch_gemm_tn_tf32x3(A, lda, B, ldb, C, ldc, (int)m, (int)n, (int)k, beta != 0.f, st);
  if (!ta && aligned && k % 4 == 0 && split_ws && m < 0x7fffffffLL && n < 0x7fffffffLL && k < 0x7fffffffLL) {
    float* hi = split_ws;
    float* lo = split_ws + (size_t)n * k;
    int rc = launch_gemm_split_b(B, ldb, (int)n, (int)k, tb ? 0 : 1, hi, lo, st);
    if (rc) return rc;
    return launch_gemm_tf32x3(A, lda, hi, lo, k, C, ldc, (int)m, (int)n, (int)k, beta != 0.f, st);
  }
  rgcn_set_error("gemm: unsupported shape (dimensions and leading dimensions must be multiples of 4)");
  return RGCN_ERR_INVALID;
}

// ---- optional stage timing -------------------------------------------------------------------
struct Profile {
  bool enabled = false;
  static const int kMax = 96;
  cudaEvent_t ev[kMax];
  const char* name[kMax];
  bool created = false;
  int n = 0;
} g_prof;

void prof_mark(const char* name, cudaStream_t st) {
  if (!g_prof.enabled) return;
  if (!g_prof.created) {
    for (int i = 0; i < Profile::kMax; ++i) cudaEventCreate(&g_prof.ev[i]);
    g_prof.created = true;
  }
  if (g_prof.n >= Profile::kMax) return;
  g_prof.name[g_prof.n] = name;
  cudaEventRecord(g_prof.ev[g_prof.n], st);
  ++g_prof.n;
}
#define MARK(name_) prof_mark(name_, st)

inline int64_t align_up(int64_t x) { return (x + 255) & ~(int64_t)255; }

struct Carver {
  char* base;
  int64_t off = 0;
  int64_t cap;
  Carver(void* p, int64_t c) : base((char*)p), cap(c) {}
  template <typename T>
  T* take(int64_t count) {
    T* r = (T*)(base + off);
    off += align_up(count * (int64_t)sizeof(T));
    return r;
  }
};

int slabs_for(int d) {
  int nv = (d + 127) / 128;
  if (nv > 4) nv = 4;
  return (d + nv * 128 - 1) / (nv * 128);
}

// ---- argument checks ------------------------------------------------------------------------------------------------
// The block and basis entry points check the graph first.  The one-hot, per-channel and diagonal ones check shape,
// pointers and workspace first (nothing there touches the device, so those errors read the same for a host-only
// graph), then the graph.

int shape_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
  if (!g || d <= 0 || d % 4 != 0 || B <= 0) {
    rgcn_set_error(std::string(who) + ": need a graph, d > 0, d % 4 == 0, B > 0");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

// the views a code path walks must have been built (rgcn_set_option("graph_views", ...))
int need_views(const rgcn_graph_t* g, bool csr, bool rel, const char* who) {
  if ((csr && !g->has_csr) || (rel && !g->has_rel)) {
    rgcn_set_error(std::string(who) + ": the graph was prepared without the " + (csr && !g->has_csr ? "CSR" : "weight-id-major") +
                   " views this path needs (option graph_views)");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

// A graph on a device with 2R weight ids and the views (csr, rel) the path walks.  The layer entry points (self_loop)
// also need V_src >= V_dst: the self-loop term reads H rows [0, V_dst).
int graph_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who, bool self_loop, bool csr, bool rel) {
  if (!g) {
    rgcn_set_error(std::string(who) + ": null graph");
    return RGCN_ERR_INVALID;
  }
  if (g->device < 0) {
    rgcn_set_error(std::string(who) + ": graph was built host-only (device = -1)");
    return RGCN_ERR_NODEVICE;
  }
  if (d <= 0 || d % 4 != 0 || B <= 0) {
    rgcn_set_error(std::string(who) + ": need d > 0, d % 4 == 0, B > 0");
    return RGCN_ERR_INVALID;
  }
  if (g->n_relw % 2 != 0) {
    rgcn_set_error(std::string(who) + ": graph weight-id count must be 2R");
    return RGCN_ERR_INVALID;
  }
  if (self_loop && g->V_src < g->V_dst) {
    rgcn_set_error(std::string(who) + ": layer entry points need V_src >= V_dst (messages-only graphs go through rgcn_block_aggregate)");
    return RGCN_ERR_INVALID;
  }
  return need_views(g, csr, rel, who);
}

int block_size_checks(int32_t d, int32_t B, const char* who) {
  if (d % B != 0) {
    rgcn_set_error(std::string(who) + ": d must be a multiple of B (gcn_basis_concat.py:15)");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

int pointer_checks(bool pointers_ok, float keep, const char* who) {
  if (!pointers_ok || keep <= 0.f) {
    rgcn_set_error(std::string(who) + (pointers_ok ? ": keep <= 0" : ": null pointer"));
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

int workspace_checks(int64_t workspace_bytes, int64_t need, const char* who) {
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  return RGCN_OK;
}

// ---- layer frame: the host steps the layer entry points share ------------------------------------------------------

// The split-row scratch of a destination-major walk (partial rows of the rows whose messages span several work items)
// and its arrival counters, carved from the workspace and zeroed.
int split_scratch(Carver& ws, int64_t n_split, int d, float*& scratch, int*& counters, cudaStream_t st) {
  const int slabs = slabs_for(d);
  scratch = ws.take<float>(n_split * d);
  counters = ws.take<int>(n_split * slabs);
  if (n_split == 0) return RGCN_OK;
  return rgcn_check_cuda(cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
                         "memset(scratch)");
}

// [C_f; C_b]: the coefficient rows indexed by weight id, forward relations first; `count` floats per direction
int concat_coefficients(const float* Cf, const float* Cb, int64_t count, float* Ccat, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat, Cf, (size_t)count * 4, cudaMemcpyDeviceToDevice, st), "copy Cf");
  if (!rc)
    rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat + count, Cb, (size_t)count * 4, cudaMemcpyDeviceToDevice, st), "copy Cb");
  return rc;
}

int split_coefficients(const float* dCcat, int64_t count, float* dCf, float* dCb, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemcpyAsync(dCf, dCcat, (size_t)count * 4, cudaMemcpyDeviceToDevice, st), "copy dCf");
  if (!rc)
    rc = rgcn_check_cuda(cudaMemcpyAsync(dCb, dCcat + count, (size_t)count * 4, cudaMemcpyDeviceToDevice, st), "copy dCb");
  return rc;
}

// out = H[0:V_dst] W_self, then out *= mask / keep when a mask is given (a walk that applies the mask passes none)
int self_loop_forward(const rgcn_graph_t* g, int d, const float* H, const float* Wself, const uint8_t* mask, float keep,
                      float* out, float* split_ws, cudaStream_t st) {
  int rc = gemm_any(st, split_ws, false, false, g->V_dst, d, d, H, d, Wself, d, 0.f, out, d);
  if (rc) return rc;
  return launch_mask_relu(out, mask, 1.0f / keep, 0, (int64_t)g->V_dst * d, st);
}

// G = dOut * relu'(out);  dS = G * mask / keep  (dropout is on the self loop only).  G and dS come in as workspace
// slices; without a mask dS is G.  With neither a ReLU nor a mask there is nothing to apply (the node-sharded layers
// pass the already masked gradient): both are dOut, read in place instead of copied into the workspace (20 GB read +
// 20 GB written at the full benchmark size).
int grad_prologue(const float* dOut, const float* out, const uint8_t* mask, float keep, int relu, int64_t n, float*& G,
                  float*& dS, cudaStream_t st) {
  if (!relu && !mask) {
    G = dS = const_cast<float*>(dOut);
    return RGCN_OK;
  }
  if (!mask) dS = G;
  return launch_grad_prologue(dOut, out, mask, 1.0f / keep, relu, n, G, dS, st);
}

// dW_self = H[0:V_dst]^T dS, then dH[0:V_dst] = dS W_self^T; the halo rows of dH start at zero.  dW_mark, when given,
// names the profile stage of the dW_self GEMM.
int self_loop_backward(const rgcn_graph_t* g, int d, const float* H, const float* dS, const float* Wself, float* dWself,
                       float* dH, float* split_ws, const char* dW_mark, cudaStream_t st) {
  int rc = gemm_any(st, split_ws, true, false, d, d, g->V_dst, H, d, dS, d, 0.f, dWself, d);
  if (rc) return rc;
  if (dW_mark) prof_mark(dW_mark, st);
  rc = gemm_any(st, split_ws, false, true, g->V_dst, d, d, dS, d, Wself, d, 0.f, dH, d);
  if (rc || g->V_src == g->V_dst) return rc;
  return rgcn_check_cuda(
      cudaMemsetAsync(dH + (size_t)g->V_dst * d, 0, (size_t)(g->V_src - g->V_dst) * d * sizeof(float), st),
      "memset(dH halo)");
}

AggLaunch make_agg(const CsrSide& side, const float* X, int ldx, int d, float* scratch,
                   int* counters) {
  AggLaunch a;
  a.items = side.d_items;
  a.n_items = (int)side.n_items;
  a.nbr = side.d_nbr;
  a.relw = side.d_relw;
  a.norm = side.d_norm;
  a.X = X;
  a.ldx = ldx;
  a.d = d;
  a.split_nitems = side.d_split_nitems;
  a.scratch = scratch;
  a.counters = counters;
  return a;
}

}  // namespace

// block_algo: 0 = destination-major (deterministic, fused epilogue), 1 = weight-id major with the gathered rows in
// registers (rgcn_kernels.cu), 3 = weight-id major with TMA-staged rows (block_staged.cu; block sizes 4, 8, 16),
// -1 = auto: 3 where it applies, else 1 where it applies, else 0
static int g_block_algo = -1;

// The block message walk of one call, chosen once: weight-id major (`rel`; with TMA-staged gathers where the block size
// supports them, `staged`) or destination-major, and whether the weight-id-major dH walk also produces dW (`fused`).
struct BlockWalk {
  bool rel, staged, fused;
};

static BlockWalk choose_block_walk(int d, int s) {
  int algo = g_block_algo;
  if (const char* e = std::getenv("RGCN_BLOCK_ALGO")) algo = std::atoi(e);
  BlockWalk w;
  w.rel = algo != 0 && block_rel_supported(d, s);
  w.staged = (algo == 3 || algo == -1) && block_stg_supported(d, s);
  w.fused = w.rel && block_rel_fuse_dw_supported(d, s) && !std::getenv("RGCN_NO_FUSE_DW");
  return w;
}

static int launch_block_relmajor(const BlockWalk& w, const RelSide& side, const float* X, int d, int s, const float* Wt,
                                 float* out, const float* Hrow, int ldh, float* dWt, cudaStream_t st) {
  return (w.staged ? launch_block_stg : launch_block_rel)(side.d_items, (int)side.n_items, side.d_row, side.d_nbr,
                                                          side.d_norm, X, d, d, s, Wt, out, Hrow, ldh, dWt, st);
}

// out[dst] += sum_m norm_m W[relw_m] . X[src_m], with the layer's epilogue: the dropout mask on the self-loop term
// already in `out` (mask, inv_keep) and the ReLU.  The weight-id-major walks accumulate with vector reductions, so they
// apply the mask before the walk and leave the ReLU to the caller; the destination-major walk applies both.  scratch
// and counters: the zeroed split-row scratch of by_dst (split_scratch), read by the destination-major walk only.
static int block_walk_forward(const rgcn_graph_t* g, const BlockWalk& w, int d, int s, const float* X, const float* Wt,
                              float* out, const uint8_t* mask, float inv_keep, int relu, float* scratch, int* counters,
                              cudaStream_t st) {
  if (w.rel) {
    int rc = launch_mask_relu(out, mask, inv_keep, 0, (int64_t)g->V_dst * d, st);
    if (rc) return rc;
    return launch_block_relmajor(w, g->by_rel, X, d, s, Wt, out, nullptr, 0, nullptr, st);
  }
  return launch_block_agg(make_agg(g->by_dst, X, d, d, scratch, counters), s, Wt, out, mask, inv_keep, relu, st);
}

// dX[src] (+)= sum_m norm_m W[relw_m]^T G[dst_m] with the transposed table Wtt; dX starts at zero when zero_dX, else it
// holds the self-loop gradient.  dWt is zeroed and, when the walk is fused, accumulates dW in the same walk.  scratch
// and counters: the zeroed split-row scratch of by_src, read by the destination-major walk only.
static int block_walk_backward(const rgcn_graph_t* g, const BlockWalk& w, int d, int s, const float* X, const float* G,
                               const float* Wtt, float* dX, bool zero_dX, float* dWt, float* scratch, int* counters,
                               cudaStream_t st) {
  int rc = RGCN_OK;
  if (zero_dX) rc = rgcn_check_cuda(cudaMemsetAsync(dX, 0, (size_t)g->V_src * d * sizeof(float), st), "memset(dX)");
  if (rc) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(dWt, 0, (size_t)g->n_relw * s * d * sizeof(float), st), "memset(dWt)");
  if (rc) return rc;
  if (w.rel)
    return launch_block_relmajor(w, g->by_rel_src, G, d, s, Wtt, dX, w.fused ? X : nullptr, d, w.fused ? dWt : nullptr,
                                 st);
  return launch_block_agg(make_agg(g->by_src, G, d, d, scratch, counters), s, Wtt, dX, nullptr, 1.f, 0, st);
}

// dW[w] = sum_{m: relw_m = w} norm_m G[dst_m] (x)_block X[src_m], unless the dH walk produced it
static int block_walk_dw(const rgcn_graph_t* g, const BlockWalk& w, int d, int s, const float* X, const float* G,
                         float* dWt, cudaStream_t st) {
  if (w.fused) return RGCN_OK;
  return launch_block_dw(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row, g->by_rel.d_nbr,
                         g->by_rel.d_norm, X, d, G, d, d, s, dWt, st);
}

extern "C" int rgcn_set_option(const char* name, int64_t value) {
  if (name && std::string(name) == "block_algo") {
    g_block_algo = (int)value;
    return RGCN_OK;
  }
  if (name && std::string(name) == "graph_views") {
    if (value < 1 || value > 3) {
      rgcn_set_error("rgcn_set_option: graph_views must be 1 (CSR), 2 (weight-id major) or 3 (both)");
      return RGCN_ERR_INVALID;
    }
    g_graph_views = (int)value;
    return RGCN_OK;
  }
  rgcn_set_error("rgcn_set_option: unknown option");
  return RGCN_ERR_INVALID;
}

extern "C" int rgcn_gemm_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, int b_is_nk,
                                float* C, int64_t ldc, int32_t M, int32_t N, int32_t K,
                                int accumulate, void* workspace, int64_t workspace_bytes,
                                void* stream) {
  if (!A || !B || !C || !workspace || M < 0 || N <= 0 || K <= 0) {
    rgcn_set_error("rgcn_gemm_tf32x3: bad arguments");
    return RGCN_ERR_INVALID;
  }
  // the GEMM launcher's own checks, made before the split so that a refused call launches nothing
  if (K % 4 != 0 || N % 4 != 0 || lda % 4 != 0 || ldc % 4 != 0) {
    rgcn_set_error("rgcn_gemm_tf32x3: K, N, lda and ldc must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < (int64_t)2 * N * K * 4) {
    rgcn_set_error("rgcn_gemm_tf32x3: workspace too small (need 2*N*K floats)");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* hi = (float*)workspace;
  float* lo = hi + (size_t)N * K;
  int rc = launch_gemm_split_b(B, ldb, N, K, b_is_nk ? 0 : 1, hi, lo, st);
  if (rc) return rc;
  return launch_gemm_tf32x3(A, lda, hi, lo, K, C, ldc, M, N, K, accumulate, st);
}

extern "C" int rgcn_gemm_tn_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, float* C,
                                   int64_t ldc, int32_t M, int32_t N, int32_t K, int accumulate,
                                   void* stream) {
  if (!A || !B || !C || M <= 0 || N <= 0 || K < 0) {
    rgcn_set_error("rgcn_gemm_tn_tf32x3: bad arguments");
    return RGCN_ERR_INVALID;
  }
  return launch_gemm_tn_tf32x3(A, lda, B, ldb, C, ldc, M, N, K, accumulate, (cudaStream_t)stream);
}

extern "C" int64_t rgcn_launch_count(void) { return g_rgcn_launches; }

extern "C" int rgcn_profile_enable(int enable) {
  g_prof.enabled = enable != 0;
  g_prof.n = 0;
  return RGCN_OK;
}

extern "C" int rgcn_profile_read(float* ms_out, int max_entries, char* names_out, int names_cap) {
  int count = 0;
  std::string names;
  for (int i = 1; i < g_prof.n; ++i) {
    // a mark named "start" opens a new call: no duration is attributed to it
    if (std::string(g_prof.name[i]) == "start") continue;
    if (count >= max_entries) break;
    if (cudaEventSynchronize(g_prof.ev[i]) != cudaSuccess) break;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, g_prof.ev[i - 1], g_prof.ev[i]) != cudaSuccess) break;
    if (ms_out) ms_out[count] = ms;
    names += g_prof.name[i];
    names += "\n";
    ++count;
  }
  if (names_out && names_cap > 0) {
    size_t n = names.size() < (size_t)names_cap - 1 ? names.size() : (size_t)names_cap - 1;
    memcpy(names_out, names.data(), n);
    names_out[n] = 0;
  }
  g_prof.n = 0;
  return count;
}

// ------------------------------------------------------------------------------------------------
// Block-diagonal layer
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_block_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B,
                                              int backward) {
  if (!g || d <= 0 || B <= 0 || d % B != 0) {
    rgcn_set_error("rgcn_block_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  const int64_t s = d / B;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  const int slabs = slabs_for(d);
  int64_t bytes = align_up((int64_t)2 * d * d * 4);  // hi/lo split of W_self for the tensor-core GEMM
  if (!backward) {
    bytes += align_up(wt * 4);
    bytes += align_up(g->by_dst.n_split * d * 4);
    bytes += align_up(g->by_dst.n_split * slabs * 4);
  } else {
    bytes += 2 * align_up(wt * 4);
    bytes += 2 * align_up((int64_t)g->V_dst * d * 4);
    bytes += align_up(g->by_src.n_split * d * 4);
    bytes += align_up(g->by_src.n_split * slabs * 4);
  }
  return bytes + 256;
}

extern "C" int rgcn_block_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                  const float* Wf, const float* Wb, const float* Wself,
                                  const uint8_t* drop_mask, float keep, int relu, float* out,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_block_forward";
  int rc = graph_checks(g, d, B, who, true, false, false);
  if (!rc) rc = block_size_checks(d, B, who);
  if (!rc) rc = pointer_checks(H && Wf && Wb && Wself && out && workspace, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_block_workspace_bytes(g, d, B, 0), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  const BlockWalk walk = choose_block_walk(d, s);
  rc = need_views(g, !walk.rel, walk.rel, who);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* Wt = ws.take<float>((int64_t)g->n_relw * s * d);

  MARK("start");
  rc = launch_block_relayout(Wf, Wb, R, B, s, /*transpose=*/0, Wt, st);
  if (rc) return rc;
  MARK("block_relayout");
  float* scratch;
  int* counters;
  rc = split_scratch(ws, g->by_dst.n_split, d, scratch, counters, st);
  if (rc) return rc;
  // self-loop term S = H[0:V_dst] @ W_self written straight into `out` (gcn_basis_concat.py:65-66); the walk applies
  // the dropout mask to it
  rc = self_loop_forward(g, d, H, Wself, nullptr, keep, out, split_ws, st);
  if (rc) return rc;
  MARK("gemm_self_loop");
  rc = block_walk_forward(g, walk, d, s, H, Wt, out, drop_mask, 1.0f / keep, relu, scratch, counters, st);
  MARK("block_agg_fwd");
  if (rc || !walk.rel) return rc;
  rc = launch_mask_relu(out, nullptr, 1.f, relu, (int64_t)g->V_dst * d, st);
  MARK("relu_epilogue");
  return rc;
}

extern "C" int rgcn_block_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                   const float* Wf, const float* Wb, const float* Wself,
                                   const uint8_t* drop_mask, float keep, int relu, const float* out,
                                   const float* dOut, float* dH, float* dWf, float* dWb,
                                   float* dWself, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  const char* who = "rgcn_block_backward";
  int rc = graph_checks(g, d, B, who, true, false, false);
  if (!rc) rc = block_size_checks(d, B, who);
  if (!rc)
    rc = pointer_checks(H && Wf && Wb && Wself && dOut && dH && dWf && dWb && dWself && workspace && (!relu || out),
                        keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_block_workspace_bytes(g, d, B, 1), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  const BlockWalk walk = choose_block_walk(d, s);
  rc = need_views(g, !walk.rel, true, who);
  if (rc) return rc;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* Wtt = ws.take<float>(wt);
  float* dWt = ws.take<float>(wt);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);

  MARK("start");
  rc = grad_prologue(dOut, out, drop_mask, keep, relu, (int64_t)g->V_dst * d, G, dS, st);  // message_gcn.py:64
  if (rc) return rc;
  MARK("grad_prologue");
  rc = self_loop_backward(g, d, H, dS, Wself, dWself, dH, split_ws, "gemm_dWself", st);
  if (rc) return rc;
  MARK("gemm_dH_self");
  // dH[u] += sum_{m: src_m = u} norm_m W[relw_m]^T G[dst_m]   (same kernel, transposed table)
  rc = launch_block_relayout(Wf, Wb, R, B, s, /*transpose=*/1, Wtt, st);
  if (rc) return rc;
  MARK("block_relayout_T");
  float* scratch;
  int* counters;
  rc = split_scratch(ws, g->by_src.n_split, d, scratch, counters, st);
  if (rc) return rc;
  // dW accumulates in the j-major layout; when the block size allows, the dH pass produces it in the same walk (one
  // round of gathers for the whole backward of the messages)
  rc = block_walk_backward(g, walk, d, s, H, G, Wtt, dH, false, dWt, scratch, counters, st);
  if (rc) return rc;
  MARK("block_agg_dH");
  rc = block_walk_dw(g, walk, d, s, H, G, dWt, st);
  if (rc) return rc;
  MARK("block_dW");
  rc = launch_block_unlayout(dWt, R, B, s, dWf, dWb, 0, walk.fused ? 1 : 0, st);
  MARK("block_unlayout");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Messages-only parts of the block layer (used by the node-sharded path to overlap the halo exchange:
// the local-source messages go through rgcn_block_forward/backward, the halo-source messages here)
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_block_aggregate_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B,
                                                        int backward) {
  if (!g || d <= 0 || B <= 0 || d % B != 0) {
    rgcn_set_error("rgcn_block_aggregate_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  const int64_t s = d / B;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  const int slabs = slabs_for(d);
  const int64_t n_split = backward ? g->by_src.n_split : g->by_dst.n_split;
  return (backward ? 2 : 1) * align_up(wt * 4) + align_up(n_split * d * 4) + align_up(n_split * slabs * 4) + 256;
}

extern "C" int rgcn_block_aggregate(const rgcn_graph_t* g, int32_t d, int32_t B, const float* X,
                                    const float* Wf, const float* Wb, float* out, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_block_aggregate";
  int rc = graph_checks(g, d, B, who, false, false, false);
  if (!rc) rc = block_size_checks(d, B, who);
  if (!rc) rc = pointer_checks(X && Wf && Wb && out && workspace, 1.f, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_block_aggregate_workspace_bytes(g, d, B, 0), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  const BlockWalk walk = choose_block_walk(d, s);
  rc = need_views(g, !walk.rel, walk.rel, who);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* Wt = ws.take<float>((int64_t)g->n_relw * s * d);
  MARK("start");
  float* scratch;
  int* counters;
  rc = launch_block_relayout(Wf, Wb, R, B, s, 0, Wt, st);
  if (!rc) rc = split_scratch(ws, g->by_dst.n_split, d, scratch, counters, st);
  if (rc) return rc;
  rc = block_walk_forward(g, walk, d, s, X, Wt, out, nullptr, 1.f, 0, scratch, counters, st);  // out = out + sum
  MARK("block_aggregate");
  return rc;
}

extern "C" int rgcn_block_aggregate_backward(const rgcn_graph_t* g, int32_t d, int32_t B,
                                             const float* X, const float* Wf, const float* Wb,
                                             const float* G, float* dX, float* dWf, float* dWb,
                                             int accumulate_dW, void* workspace,
                                             int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_block_aggregate_backward";
  int rc = graph_checks(g, d, B, who, false, false, false);
  if (!rc) rc = block_size_checks(d, B, who);
  if (!rc) rc = pointer_checks(X && Wf && Wb && G && dX && dWf && dWb && workspace, 1.f, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_block_aggregate_workspace_bytes(g, d, B, 1), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  const BlockWalk walk = choose_block_walk(d, s);
  rc = need_views(g, !walk.rel, true, who);
  if (rc) return rc;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  Carver ws(workspace, workspace_bytes);
  float* Wtt = ws.take<float>(wt);
  float* dWt = ws.take<float>(wt);
  MARK("start");
  float* scratch;
  int* counters;
  rc = launch_block_relayout(Wf, Wb, R, B, s, 1, Wtt, st);
  if (!rc) rc = split_scratch(ws, g->by_src.n_split, d, scratch, counters, st);
  if (!rc) rc = block_walk_backward(g, walk, d, s, X, G, Wtt, dX, true, dWt, scratch, counters, st);
  if (!rc) rc = block_walk_dw(g, walk, d, s, X, G, dWt, st);
  if (rc) return rc;
  MARK("block_aggregate_bwd");
  return launch_block_unlayout(dWt, R, B, s, dWf, dWb, accumulate_dW, walk.fused ? 1 : 0, st);
}

// dst[rows[i], :] += src[i, :] (rows unique): unpack of the returned halo gradients, one peer segment per call
extern "C" int rgcn_rows_add(float* dst, const int64_t* rows, const float* src, int64_t n, int32_t d, void* stream) {
  if (n < 0 || d <= 0 || d % 4 != 0 || (n > 0 && (!dst || !rows || !src))) {
    rgcn_set_error("rgcn_rows_add: bad arguments (d % 4 == 0)");
    return RGCN_ERR_INVALID;
  }
  return launch_rows_add(dst, rows, src, n, d, (cudaStream_t)stream);
}

// G = dOut * relu'(out): the gradient prologue alone (the node-sharded layers need G before their first kernel)
extern "C" int rgcn_relu_backward(const float* dOut, const float* out, float* G, int64_t n, void* stream) {
  if (n < 0 || n % 4 != 0 || (n > 0 && (!dOut || !out || !G))) {
    rgcn_set_error("rgcn_relu_backward: bad arguments (n % 4 == 0)");
    return RGCN_ERR_INVALID;
  }
  return launch_grad_prologue(dOut, out, nullptr, 1.0f, 1, n, G, G, (cudaStream_t)stream);
}

// dst[i, :] = src[rows[i], :]; dst may be peer-mapped memory (halo push over NVLink)
extern "C" int rgcn_rows_gather(float* dst, const float* src, const int64_t* rows, int64_t n, int32_t d,
                                int32_t max_ctas, void* stream) {
  if (n < 0 || d <= 0 || d % 4 != 0 || max_ctas < 0 || (n > 0 && (!dst || !rows || !src))) {
    rgcn_set_error("rgcn_rows_gather: bad arguments (d % 4 == 0)");
    return RGCN_ERR_INVALID;
  }
  return launch_rows_gather(dst, src, rows, n, d, max_ctas, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Basis layer
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_basis_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B,
                                              int backward) {
  if (!g || d <= 0 || B <= 0) {
    rgcn_set_error("rgcn_basis_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = align_up((int64_t)g->n_relw * B * 4);  // concatenated coefficient table
  bytes += align_up((int64_t)2 * d * d * B * 4);           // hi/lo split of the GEMM B operands
  if (backward) {
    bytes += align_up((int64_t)g->n_relw * B * 4);           // dC (concatenated)
    bytes += 2 * align_up((int64_t)g->V_dst * d * 4);        // G, dS
    bytes += align_up((int64_t)g->V_dst * 2 * d * B * 4);    // dAgg
    bytes += align_up((int64_t)g->V_src * 2 * d * B * 4);    // P (planar)
  }
  return bytes + 256;
}

extern "C" int rgcn_basis_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                  const float* Vf, const float* Vb, const float* Cf,
                                  const float* Cb, const float* Wself, const uint8_t* drop_mask,
                                  float keep, int relu, float* out, float* saved, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_forward";
  int rc = graph_checks(g, d, B, who, true, true, false);
  if (!rc) rc = pointer_checks(H && Vf && Vb && Cf && Cb && Wself && out && saved && workspace, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_workspace_bytes(g, d, B, 0), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  float* split_ws = ws.take<float>((int64_t)2 * d * d * B);
  rc = concat_coefficients(Cf, Cb, (int64_t)R * B, Ccat, st);
  if (rc) return rc;
  MARK("start");
  // Agg[v][dir][k*B+b] = sum_m norm_m C[relw_m,b] H[src_m,k]
  rc = launch_zero_rows(saved, 2 * dB, g->by_dst.d_split_rows, (int)g->by_dst.n_split, st);
  if (rc) return rc;
  AggLaunch a = make_agg(g->by_dst, H, d, d, nullptr, nullptr);
  rc = launch_basis_agg(a, Ccat, B, g->n_relw, /*layout=*/0, saved, st);
  if (rc) return rc;
  MARK("basis_agg_fwd");
  rc = self_loop_forward(g, d, H, Wself, drop_mask, keep, out, split_ws, st);
  if (rc) return rc;
  // out += Agg_f @ Vf.reshape(d*B, d) + Agg_b @ Vb.reshape(d*B, d)    (gcn_basis.py:60-68 re-associated)
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, dB, saved, 2 * dB, Vf, d, 1.f, out, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, dB, saved + dB, 2 * dB, Vb, d, 1.f, out, d);
  if (rc) return rc;
  MARK("basis_gemms_fwd");
  rc = launch_mask_relu(out, nullptr, 1.f, relu, (int64_t)g->V_dst * d, st);
  MARK("relu_epilogue");
  return rc;
}

extern "C" int rgcn_basis_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                   const float* Vf, const float* Vb, const float* Cf,
                                   const float* Cb, const float* Wself, const uint8_t* drop_mask,
                                   float keep, int relu, const float* out, const float* saved,
                                   const float* dOut, float* dH, float* dVf, float* dVb, float* dCf,
                                   float* dCb, float* dWself, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_backward";
  int rc = graph_checks(g, d, B, who, true, true, false);
  if (!rc)
    rc = pointer_checks(H && Vf && Vb && Cf && Cb && Wself && saved && dOut && dH && dVf && dVb && dCf && dCb &&
                            dWself && workspace && (!relu || out),
                        keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_workspace_bytes(g, d, B, 1), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  float* split_ws = ws.take<float>((int64_t)2 * d * d * B);
  float* dCcat = ws.take<float>((int64_t)g->n_relw * B);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);
  float* dAgg = ws.take<float>((int64_t)g->V_dst * 2 * dB);
  float* P = ws.take<float>((int64_t)g->V_src * 2 * dB);
  rc = concat_coefficients(Cf, Cb, (int64_t)R * B, Ccat, st);
  if (rc) return rc;

  MARK("start");
  rc = grad_prologue(dOut, out, drop_mask, keep, relu, (int64_t)g->V_dst * d, G, dS, st);
  if (!rc) rc = self_loop_backward(g, d, H, dS, Wself, dWself, dH, split_ws, nullptr, st);
  if (rc) return rc;
  MARK("basis_self_loop_bwd");
  // dV_dir.reshape(d*B, d) = Agg_dir^T G
  rc = gemm_any(st, split_ws, true, false, dB, d, g->V_dst, saved, 2 * dB, G, d, 0.f, dVf, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, true, false, dB, d, g->V_dst, saved + dB, 2 * dB, G, d, 0.f, dVb, d);
  if (rc) return rc;
  // dAgg_dir = G V_dir.reshape(d*B, d)^T
  rc = gemm_any(st, split_ws, false, true, g->V_dst, dB, d, G, d, Vf, d, 0.f, dAgg, 2 * dB);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, true, g->V_dst, dB, d, G, d, Vb, d, 0.f, dAgg + dB, 2 * dB);
  if (rc) return rc;
  MARK("basis_gemms_dV_dAgg");
  // dC[w,b] = sum_m norm_m < H[src_m], dAgg[dst_m][dir][:,b] >
  rc = rgcn_check_cuda(cudaMemsetAsync(dCcat, 0, (size_t)g->n_relw * B * 4, st), "memset(dC)");
  if (rc) return rc;
  AggLaunch a = make_agg(g->by_dst, H, d, d, nullptr, nullptr);
  rc = launch_basis_dc(a, dAgg, B, g->n_relw, dCcat, st);
  if (rc) return rc;
  MARK("basis_dC");
  rc = split_coefficients(dCcat, (int64_t)R * B, dCf, dCb, st);
  if (rc) return rc;
  // P[u][dir][b*d+n] = sum_{m: src_m=u} norm_m C[relw_m,b] G[dst_m,n];  dH += P_dir V_dir.reshape(d, B*d)^T
  rc = launch_zero_rows(P, 2 * dB, g->by_src.d_split_rows, (int)g->by_src.n_split, st);
  if (rc) return rc;
  AggLaunch as = make_agg(g->by_src, G, d, d, nullptr, nullptr);
  rc = launch_basis_agg(as, Ccat, B, g->n_relw, /*layout=*/1, P, st);
  if (rc) return rc;
  MARK("basis_agg_dH");
  rc = gemm_any(st, split_ws, false, true, g->V_src, d, dB, P, 2 * dB, Vf, dB, 1.f, dH, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, true, g->V_src, d, dB, P + dB, 2 * dB, Vb, dB, 1.f, dH, d);
  MARK("basis_gemms_dH");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// One-hot (featureless) basis layer: layer 0 of gcn_basis with UseInputTransform=No
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_basis_onehot_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward) {
  if (!g || d <= 0 || B <= 0) {
    rgcn_set_error("rgcn_basis_onehot_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = align_up((int64_t)g->n_relw * B * 4);  // concatenated coefficient table
  if (backward) {
    bytes += align_up((int64_t)g->n_relw * B * 4);       // dC (concatenated)
    bytes += align_up((int64_t)g->V_dst * d * 4);        // G (used when a dropout mask is given)
  }
  return bytes + 256;
}

extern "C" int rgcn_basis_onehot_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* Wf,
                                         const float* Wb, const float* Cf, const float* Cb, const float* Wself,
                                         const uint8_t* drop_mask, float keep, int relu, float* out, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_onehot_forward";
  int rc = shape_checks(g, d, B, who);
  if (!rc) rc = pointer_checks(Wf && Wb && Cf && Cb && Wself && out && workspace, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_onehot_workspace_bytes(g, d, B, 0), who);
  if (!rc) rc = graph_checks(g, d, B, who, true, true, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t n = (int64_t)g->V_dst * d;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  rc = concat_coefficients(Cf, Cb, (int64_t)R * B, Ccat, st);
  if (rc) return rc;
  MARK("start");
  // out = dropout(W_self)  (the self loop looks up W_self with tf.range(V): message_gcn.py:56, gcn_basis.py:70-71)
  rc = rgcn_check_cuda(cudaMemcpyAsync(out, Wself, (size_t)n * 4, cudaMemcpyDeviceToDevice, st), "copy W_self");
  if (!rc) rc = launch_mask_relu(out, drop_mask, 1.0f / keep, 0, n, st);
  if (rc) return rc;
  MARK("onehot_self_loop");
  // out[dst] += norm * sum_b C[relw,b] W_dir[src,b,:]
  rc = launch_basis_onehot_push(g->by_src.d_items, (int)g->by_src.n_items, g->by_src.d_nbr, g->by_src.d_relw,
                                g->by_src.d_norm, Wf, Wb, Ccat, B, d, g->n_relw, out, st);
  if (rc) return rc;
  MARK("onehot_push_fwd");
  rc = launch_mask_relu(out, nullptr, 1.f, relu, n, st);
  MARK("relu_epilogue");
  return rc;
}

extern "C" int rgcn_basis_onehot_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* Wf,
                                          const float* Wb, const float* Cf, const float* Cb,
                                          const uint8_t* drop_mask, float keep, int relu, const float* out,
                                          const float* dOut, float* dWf, float* dWb, float* dCf, float* dCb,
                                          float* dWself, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_onehot_backward";
  int rc = shape_checks(g, d, B, who);
  if (!rc)
    rc = pointer_checks(
        Wf && Wb && Cf && Cb && dOut && dWf && dWb && dCf && dCb && dWself && workspace && (!relu || out), keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_onehot_workspace_bytes(g, d, B, 1), who);
  if (!rc) rc = graph_checks(g, d, B, who, true, true, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  float* dCcat = ws.take<float>((int64_t)g->n_relw * B);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  rc = concat_coefficients(Cf, Cb, (int64_t)R * B, Ccat, st);
  if (rc) return rc;
  MARK("start");
  // G = dOut * relu'(out);  dW_self = G * mask / keep (without a mask dW_self IS G: written once, read in place)
  if (!drop_mask) G = dWself;
  rc = launch_grad_prologue(dOut, out, drop_mask, 1.0f / keep, relu, (int64_t)g->V_dst * d, G, dWself, st);
  if (rc) return rc;
  MARK("grad_prologue");
  // dW_dir[u] = sum_{m from u} norm C[relw] (x) G[dst];  dC[relw] += < W_dir[u], sum_run norm G[dst] >
  rc = rgcn_check_cuda(cudaMemsetAsync(dCcat, 0, (size_t)g->n_relw * B * 4, st), "memset(dC)");
  if (!rc) rc = launch_zero_rows(dWf, dB, g->by_src.d_split_rows, (int)g->by_src.n_split, st);
  if (!rc) rc = launch_zero_rows(dWb, dB, g->by_src.d_split_rows, (int)g->by_src.n_split, st);
  if (rc) return rc;
  AggLaunch a = make_agg(g->by_src, G, d, d, nullptr, nullptr);
  rc = launch_basis_agg_dc(a, Ccat, B, g->n_relw, Wf, Wb, dWf, dWb, dCcat, st);
  if (rc) return rc;
  MARK("onehot_agg_dW_dC");
  return split_coefficients(dCcat, (int64_t)R * B, dCf, dCb, st);
}

// ------------------------------------------------------------------------------------------------
// Basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes, basis_diagcoef.cu)
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_basis_diagcoef_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B, int backward) {
  if (!g || d <= 0 || B <= 0) {
    rgcn_set_error("rgcn_basis_diagcoef_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  const int64_t dB = (int64_t)d * B;
  int64_t bytes = align_up((int64_t)g->n_relw * dB * 4);  // sigmoid(C) table
  bytes += align_up((int64_t)2 * d * dB * 4);              // hi/lo split of the GEMM B operands
  if (backward) {
    bytes += 2 * align_up((int64_t)g->V_dst * d * 4);      // G, dS
    bytes += align_up((int64_t)g->V_src * 2 * dB * 4);     // dP (planar, both directions)
  }
  return bytes + 256;
}

extern "C" int rgcn_basis_diagcoef_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                           const float* Vf, const float* Vb, const float* Cf, const float* Cb,
                                           const float* Wself, const float* b, const uint8_t* drop_mask, float keep,
                                           int relu, float* out, float* saved, void* workspace,
                                           int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_diagcoef_forward";
  int rc = shape_checks(g, d, B, who);
  if (!rc) rc = pointer_checks(H && Vf && Vb && Cf && Cb && Wself && b && out && saved && workspace, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_diagcoef_workspace_bytes(g, d, B, 0), who);
  if (!rc) rc = graph_checks(g, d, B, who, true, true, true);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* sig = ws.take<float>((int64_t)g->n_relw * dB);
  float* split_ws = ws.take<float>((int64_t)2 * d * dB);
  MARK("start");
  rc = launch_diagcoef_sigmoid(Cf, Cb, (int64_t)R * dB, sig, st);
  if (rc) return rc;
  // saved = P: row u holds P_f[u] | P_b[u]  (P_dir = H V_dir.reshape(d, B*d), gcn_basis_times_diag.py:61-72)
  rc = gemm_any(st, split_ws, false, false, g->V_src, dB, d, H, d, Vf, dB, 0.f, saved, 2 * dB);
  if (!rc) rc = gemm_any(st, split_ws, false, false, g->V_src, dB, d, H, d, Vb, dB, 0.f, saved + dB, 2 * dB);
  if (rc) return rc;
  MARK("diagcoef_gemms_P");
  rc = self_loop_forward(g, d, H, Wself, drop_mask, keep, out, split_ws, st);
  if (rc) return rc;
  MARK("gemm_self_loop");
  rc = launch_diagcoef_fwd(g->by_dst.d_items, (int)g->by_dst.n_items, g->by_dst.d_nbr, g->by_dst.d_relw,
                           g->by_dst.d_norm, saved, sig, B, d, g->n_relw, out, st);
  if (rc) return rc;
  MARK("diagcoef_walk_fwd");
  rc = launch_diagcoef_bias_act(out, b, g->V_dst, d, relu, st);
  MARK("bias_act_epilogue");
  return rc;
}

extern "C" int rgcn_basis_diagcoef_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                            const float* Vf, const float* Vb, const float* Cf, const float* Cb,
                                            const float* Wself, const uint8_t* drop_mask, float keep, int relu,
                                            const float* out, const float* saved, const float* dOut, float* dH,
                                            float* dVf, float* dVb, float* dCf, float* dCb, float* dWself, float* db,
                                            void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_basis_diagcoef_backward";
  int rc = shape_checks(g, d, B, who);
  if (!rc)
    rc = pointer_checks(H && Vf && Vb && Cf && Cb && Wself && saved && dOut && dH && dVf && dVb && dCf && dCb &&
                            dWself && db && workspace && (!relu || out),
                        keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_basis_diagcoef_workspace_bytes(g, d, B, 1), who);
  if (!rc) rc = graph_checks(g, d, B, who, true, true, true);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* sig = ws.take<float>((int64_t)g->n_relw * dB);
  float* split_ws = ws.take<float>((int64_t)2 * d * dB);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);
  float* dP = ws.take<float>((int64_t)g->V_src * 2 * dB);

  MARK("start");
  rc = launch_diagcoef_sigmoid(Cf, Cb, (int64_t)R * dB, sig, st);
  if (!rc) rc = grad_prologue(dOut, out, drop_mask, keep, relu, (int64_t)g->V_dst * d, G, dS, st);
  if (!rc) rc = launch_diagcoef_colsum(G, g->V_dst, d, db, st);
  if (rc) return rc;
  MARK("grad_prologue_db");
  rc = self_loop_backward(g, d, H, dS, Wself, dWself, dH, split_ws, nullptr, st);
  if (rc) return rc;
  MARK("diagcoef_self_loop_bwd");
  // dP[u][dir][b][:] = sum_{m from u} norm_m sig[relw_m,b,:] G[dst_m,:]
  rc = launch_zero_rows(dP, 2 * dB, g->by_src.d_split_rows, (int)g->by_src.n_split, st);
  if (!rc)
    rc = launch_diagcoef_dp(g->by_src.d_items, (int)g->by_src.n_items, g->by_src.d_nbr, g->by_src.d_relw,
                            g->by_src.d_norm, G, sig, B, d, g->n_relw, dP, st);
  if (rc) return rc;
  MARK("diagcoef_walk_dP");
  // dV_dir.reshape(d, B*d) = H^T dP_dir;  dH += dP_dir V_dir.reshape(d, B*d)^T
  rc = gemm_any(st, split_ws, true, false, d, dB, g->V_src, H, d, dP, 2 * dB, 0.f, dVf, dB);
  if (!rc) rc = gemm_any(st, split_ws, true, false, d, dB, g->V_src, H, d, dP + dB, 2 * dB, 0.f, dVb, dB);
  if (!rc) rc = gemm_any(st, split_ws, false, true, g->V_src, d, dB, dP, 2 * dB, Vf, dB, 1.f, dH, d);
  if (!rc) rc = gemm_any(st, split_ws, false, true, g->V_src, d, dB, dP + dB, 2 * dB, Vb, dB, 1.f, dH, d);
  if (rc) return rc;
  MARK("diagcoef_gemms_dV_dH");
  // dC_dir[w][b][:] = sig' * sum_{m: relw_m = w} norm_m P[src_m][dir][b][:] G[dst_m,:]
  rc = rgcn_check_cuda(cudaMemsetAsync(dCf, 0, (size_t)R * dB * 4, st), "memset(dCf)");
  if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(dCb, 0, (size_t)R * dB * 4, st), "memset(dCb)");
  if (!rc)
    rc = launch_diagcoef_dc(g->by_rel_src.d_items, (int)g->by_rel_src.n_items, g->by_rel_src.d_row,
                            g->by_rel_src.d_nbr, g->by_rel_src.d_norm, saved, G, sig, B, d, g->n_relw, dCf, dCb, st);
  MARK("diagcoef_walk_dC");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Diagonal R-GCN layer (Name=gcn_diag, gcn_diag.cu)
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_diag_workspace_bytes(const rgcn_graph_t* g, int32_t d, int backward) {
  if (!g || d <= 0) {
    rgcn_set_error("rgcn_diag_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = align_up((int64_t)2 * d * d * 4);  // hi/lo split of W_self for the tensor-core GEMM
  if (!backward) {
    bytes += align_up(g->by_dst.n_split * d * 4);                    // split-row scratch
    bytes += align_up(g->by_dst.n_split * slabs_for(d) * 4);         // split-row arrival counters
  } else {
    bytes += 2 * align_up((int64_t)g->V_dst * d * 4);                // G, dS
  }
  return bytes + 256;
}

extern "C" int rgcn_diag_forward(const rgcn_graph_t* g, int32_t d, const float* H, const float* Df, const float* Db,
                                 const float* Wself, const float* b, const uint8_t* drop_mask, float keep, int relu,
                                 float* out, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_diag_forward";
  int rc = shape_checks(g, d, 1, who);
  if (!rc) rc = pointer_checks(H && Df && Db && Wself && b && out && workspace, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_diag_workspace_bytes(g, d, 0), who);
  if (!rc) rc = graph_checks(g, d, 1, who, true, true, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* scratch;
  int* counters;
  MARK("start");
  rc = split_scratch(ws, g->by_dst.n_split, d, scratch, counters, st);
  if (rc) return rc;
  // self-loop term H[0:V_dst] W_self written straight into `out`; the walk applies the dropout mask (gcn_diag.py:39-40)
  rc = self_loop_forward(g, d, H, Wself, nullptr, keep, out, split_ws, st);
  if (rc) return rc;
  MARK("gemm_self_loop");
  // out[v] = act(dropout(out[v]) + sum_{m into v} norm_m D[relw_m] (.) H[src_m] + b)   (gcn_diag.py:29-58)
  rc = launch_diaggcn_fwd(g->by_dst.d_items, (int)g->by_dst.n_items, g->by_dst.d_nbr, g->by_dst.d_relw,
                          g->by_dst.d_norm, H, Df, Db, d, g->n_relw, b, drop_mask, 1.0f / keep, relu,
                          g->by_dst.d_split_nitems, scratch, counters, out, st);
  MARK("diag_walk_fwd");
  return rc;
}

extern "C" int rgcn_diag_backward(const rgcn_graph_t* g, int32_t d, const float* H, const float* Df, const float* Db,
                                  const float* Wself, const uint8_t* drop_mask, float keep, int relu, const float* out,
                                  const float* dOut, float* dH, float* dDf, float* dDb, float* dWself, float* db,
                                  float* slice_sumsq2, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_diag_backward";
  int rc = shape_checks(g, d, 1, who);
  if (!rc)
    rc = pointer_checks(
        H && Df && Db && Wself && dOut && dH && dDf && dDb && dWself && db && workspace && (!relu || out), keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_diag_workspace_bytes(g, d, 1), who);
  if (!rc) rc = graph_checks(g, d, 1, who, true, true, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);

  MARK("start");
  rc = grad_prologue(dOut, out, drop_mask, keep, relu, (int64_t)g->V_dst * d, G, dS, st);
  if (!rc) rc = launch_diagcoef_colsum(G, g->V_dst, d, db, st);
  if (rc) return rc;
  MARK("grad_prologue_db");
  rc = self_loop_backward(g, d, H, dS, Wself, dWself, dH, split_ws, nullptr, st);
  if (rc) return rc;
  MARK("diag_self_loop_bwd");
  // dH[u] += sum_{m from u} norm_m D[relw_m] (.) G[dst_m];  dD[w] = sum_{m: relw_m = w} norm_m H[src_m] (.) G[dst_m]
  rc = rgcn_check_cuda(cudaMemsetAsync(dDf, 0, (size_t)R * d * 4, st), "memset(dDf)");
  if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(dDb, 0, (size_t)R * d * 4, st), "memset(dDb)");
  if (!rc && slice_sumsq2) rc = rgcn_check_cuda(cudaMemsetAsync(slice_sumsq2, 0, 2 * 4, st), "memset(sumsq2)");
  if (!rc)
    rc = launch_diaggcn_bwd(g->by_src.d_items, (int)g->by_src.n_items, g->by_src.d_nbr, g->by_src.d_relw,
                            g->by_src.d_norm, G, H, Df, Db, d, g->n_relw, dH, dDf, dDb, slice_sumsq2, st);
  MARK("diag_walk_bwd");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// CompGCN layer (Name=compgcn, compgcn.cu): the walk writes the GEMM operand Cat, one GEMM with the bias + ReLU
// epilogue makes `out`, a second one the next relation table
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_compgcn_workspace_bytes(const rgcn_graph_t* g, int32_t d_in, int32_t d_out, int backward) {
  if (!g || d_in <= 0 || d_out <= 0) {
    rgcn_set_error("rgcn_compgcn_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = align_up((int64_t)2 * 3 * d_in * d_out * 4);  // hi/lo split of W_cat (the largest split operand)
  if (backward) {
    bytes += align_up((int64_t)g->V_dst * d_out * 4);      // G
    bytes += align_up((int64_t)g->V_dst * 3 * d_in * 4);   // dCat
  }
  return bytes + 256;
}

// shape, pointer and workspace checks come first (they need no device), then the graph
static int compgcn_checks(const rgcn_graph_t* g, int32_t d_in, int32_t d_out, int composition, bool pointers_ok,
                          float keep, int backward, int64_t workspace_bytes, const char* who) {
  int rc = shape_checks(g, d_in, 1, who);
  if (!rc && (d_out <= 0 || d_out % 4 != 0)) {
    rgcn_set_error(std::string(who) + ": need d_out > 0, d_out % 4 == 0");
    rc = RGCN_ERR_INVALID;
  }
  if (!rc && composition != RGCN_COMPOSITION_MULT && composition != RGCN_COMPOSITION_SUB) {
    rgcn_set_error(std::string(who) + ": composition must be RGCN_COMPOSITION_MULT or RGCN_COMPOSITION_SUB");
    rc = RGCN_ERR_INVALID;
  }
  if (!rc) rc = pointer_checks(pointers_ok, keep, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_compgcn_workspace_bytes(g, d_in, d_out, backward), who);
  if (!rc) rc = graph_checks(g, d_in, 1, who, true, true, false);
  return rc;
}

extern "C" int rgcn_compgcn_forward(const rgcn_graph_t* g, int32_t d_in, int32_t d_out, int composition,
                                    const float* H, const float* Z, const float* z_loop, const float* W_cat,
                                    const float* W_rel, const float* b, const uint8_t* drop_mask, float keep, int relu,
                                    float* Cat, float* out, float* Z_next, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
  const char* who = "rgcn_compgcn_forward";
  int rc = compgcn_checks(g, d_in, d_out, composition,
                          H && Z && z_loop && W_cat && W_rel && b && Cat && out && Z_next && workspace, keep, 0,
                          workspace_bytes, who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * 3 * d_in * d_out);
  const int64_t ldc = 3 * (int64_t)d_in;
  MARK("start");
  // Cat = [mask / keep (.) [A_f | A_b] | phi(H, z_loop)] / 3; the split rows are reduced into zeroed rows
  rc = launch_zero_rows(Cat, ldc, g->by_dst.d_split_rows, (int)g->by_dst.n_split, st);
  if (!rc)
    rc = launch_compgcn_fwd(composition, g->by_dst.d_items, (int)g->by_dst.n_items, g->by_dst.d_nbr, g->by_dst.d_relw,
                            g->by_dst.d_norm, H, Z, z_loop, d_in, g->n_relw, drop_mask, 1.0f / keep, Cat, st);
  if (rc) return rc;
  MARK("compgcn_walk_fwd");
  // out = act(Cat W_cat + b)
  rc = launch_gemm_split_b(W_cat, d_out, d_out, (int)ldc, 1, split_ws, split_ws + (size_t)d_out * ldc, st);
  if (!rc)
    rc = launch_gemm_bias_act_tf32x3(Cat, ldc, split_ws, split_ws + (size_t)d_out * ldc, ldc, b, relu, out, d_out,
                                     g->V_dst, d_out, (int)ldc, st);
  if (rc) return rc;
  MARK("compgcn_gemm_out");
  // Z_next = Z W_rel
  rc = gemm_any(st, split_ws, false, false, g->n_relw, d_out, d_in, Z, d_in, W_rel, d_out, 0.f, Z_next, d_out);
  MARK("compgcn_gemm_rel");
  return rc;
}

extern "C" int rgcn_compgcn_backward(const rgcn_graph_t* g, int32_t d_in, int32_t d_out, int composition,
                                     const float* H, const float* Z, const float* z_loop, const float* W_cat,
                                     const float* W_rel, const uint8_t* drop_mask, float keep, int relu,
                                     const float* Cat, const float* out, const float* dOut, const float* dZ_next,
                                     float* dH, float* dZ, float* dz_loop, float* dW_cat, float* dW_rel, float* db,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_compgcn_backward";
  int rc = compgcn_checks(g, d_in, d_out, composition,
                          H && Z && z_loop && W_cat && W_rel && Cat && dOut && dZ_next && dH && dZ && dz_loop &&
                              dW_cat && dW_rel && db && workspace && (!relu || out),
                          keep, 1, workspace_bytes, who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * 3 * d_in * d_out);
  float* G = ws.take<float>((int64_t)g->V_dst * d_out);
  float* dCat = ws.take<float>((int64_t)g->V_dst * 3 * d_in);
  const int64_t ldc = 3 * (int64_t)d_in;
  MARK("start");
  // G = dOut * relu'(out) (the dropout is inside Cat);  db = column sums of G
  float* dS = G;
  rc = grad_prologue(dOut, out, nullptr, 1.f, relu, (int64_t)g->V_dst * d_out, G, dS, st);
  if (!rc) rc = launch_diagcoef_colsum(G, g->V_dst, d_out, db, st);
  if (rc) return rc;
  MARK("grad_prologue_db");
  // dW_cat = Cat^T G,  dCat = G W_cat^T
  rc = gemm_any(st, split_ws, true, false, ldc, d_out, g->V_dst, Cat, ldc, G, d_out, 0.f, dW_cat, d_out);
  if (!rc) rc = gemm_any(st, split_ws, false, true, g->V_dst, ldc, d_out, G, d_out, W_cat, d_out, 0.f, dCat, ldc);
  if (rc) return rc;
  MARK("compgcn_gemms_cat");
  // dW_rel = Z^T dZ_next;  dZ = dZ_next W_rel^T, then the walk adds its terms
  rc = gemm_any(st, split_ws, true, false, d_in, d_out, g->n_relw, Z, d_in, dZ_next, d_out, 0.f, dW_rel, d_out);
  if (!rc) rc = gemm_any(st, split_ws, false, true, g->n_relw, d_in, d_out, dZ_next, d_out, W_rel, d_out, 0.f, dZ, d_in);
  if (rc) return rc;
  MARK("compgcn_gemms_rel");
  rc = rgcn_check_cuda(cudaMemsetAsync(dz_loop, 0, (size_t)d_in * 4, st), "memset(dz_loop)");
  if (!rc) rc = launch_zero_rows(dH, d_in, g->by_src.d_split_rows, (int)g->by_src.n_split, st);
  if (!rc)
    rc = launch_compgcn_bwd(composition, g->by_src.d_items, (int)g->by_src.n_items, g->by_src.d_nbr, g->by_src.d_relw,
                            g->by_src.d_norm, dCat, H, Z, z_loop, d_in, g->n_relw, g->V_dst, drop_mask, 1.0f / keep,
                            dH, dZ, dz_loop, st);
  MARK("compgcn_walk_bwd");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Highway skip connection (extras/highway_layer.py): one gate GEMM with the blend epilogue forward; an elementwise
// prologue and two GEMMs backward
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_highway_workspace_bytes(int64_t V, int32_t d, int backward) {
  if (V < 0 || d <= 0) {
    rgcn_set_error("rgcn_highway_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = align_up((int64_t)2 * d * d * 4);     // hi / lo planes of the pre-split W (or W^T)
  if (backward) bytes += align_up(V * d * 4);           // dz
  return bytes + 256;
}

static int highway_checks(bool ok, int64_t V, int32_t d, int64_t workspace_bytes, int backward, const char* who) {
  if (!ok || V < 0 || V > 0x7fffffffLL || d <= 0 || d % 4 != 0) {
    rgcn_set_error(std::string(who) + ": need non-null pointers, 0 <= V < 2^31, d > 0, d % 4 == 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_highway_workspace_bytes(V, d, backward)) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  if (V == 0) return RGCN_OK;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    rgcn_set_error(std::string(who) + ": no CUDA device");
    return RGCN_ERR_NODEVICE;
  }
  return RGCN_OK;
}

extern "C" int rgcn_highway_forward(const float* c1, const float* c2, const float* W, const float* b, int64_t V,
                                    int32_t d, float* out, float* gate, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
  int rc = highway_checks(c1 && c2 && W && b && out && gate && workspace, V, d, workspace_bytes, 0,
                          "rgcn_highway_forward");
  if (rc || V == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)2 * d * d);
  float* lo = hi + (size_t)d * d;
  MARK("start");
  // Bt = W^T (B = W is [K = in, N = out]); the split is d^2 elements, the GEMM V d^2
  rc = launch_gemm_split_b(W, d, d, d, /*transposed=*/1, hi, lo, st);
  if (rc) return rc;
  rc = launch_gemm_highway_tf32x3(c2, hi, lo, b, c1, out, gate, (int)V, d, st);
  MARK("highway_gate_gemm");
  return rc;
}

extern "C" int rgcn_highway_backward(const float* c1, const float* c2, const float* W, const float* gate,
                                     const float* dOut, int64_t V, int32_t d, float* dc1, float* dc2, float* dW,
                                     float* db, void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = highway_checks(c1 && c2 && W && gate && dOut && dc1 && dc2 && dW && db && workspace, V, d,
                          workspace_bytes, 1, "rgcn_highway_backward");
  if (rc || V == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)2 * d * d);
  float* lo = hi + (size_t)d * d;
  float* dz = ws.take<float>(V * d);
  MARK("start");
  rc = launch_highway_prologue(c1, c2, gate, dOut, V, d, dc1, dz, dc2, db, st);
  if (rc) return rc;
  MARK("highway_prologue");
  // dc2 += dz W^T: Bt = W itself ([N = in, K = out], already K-major)
  rc = launch_gemm_split_b(W, d, d, d, /*transposed=*/0, hi, lo, st);
  if (!rc) rc = launch_gemm_tf32x3(dz, d, hi, lo, d, dc2, d, (int)V, d, d, /*accumulate=*/1, st);
  if (rc) return rc;
  MARK("highway_dc2_gemm");
  // dW = c2^T dz (contraction over V)
  rc = launch_gemm_tn_tf32x3(c2, d, dz, d, dW, d, d, d, (int)V, /*accumulate=*/0, st);
  MARK("highway_dW_gemm");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// Variational head (extras/variational_encoding.py): d == 0 (H == NULL) is the embedding variant, mu and log sigma
// are the [V, w] tables themselves; otherwise mu / log sigma = H W + b through one GEMM with interleaved weights.
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_variational_workspace_bytes(int64_t V, int32_t d, int32_t w, int backward) {
  if (V < 0 || V > 0x7fffffffLL || d < 0 || d % 4 != 0 || w <= 0 || w % 4 != 0) {
    rgcn_set_error("rgcn_variational_workspace_bytes: need 0 <= V < 2^31, d >= 0, d % 4 == 0, w > 0, w % 4 == 0");
    return RGCN_ERR_INVALID;
  }
  int64_t bytes = 0;
  if (d == 0) {
    if (!backward) bytes += align_up(var_emb_kl_parts(V, w) * 4);
  } else if (!backward) {
    bytes += align_up((int64_t)2 * (2 * w) * d * 4);                       // hi / lo planes of W_int^T
    bytes += align_up(std::max<int64_t>(1, gemm_variational_kl_parts(V, w)) * 4);
  } else {
    bytes += align_up((int64_t)2 * d * (2 * w) * 4);                       // hi / lo planes of W_int
    bytes += align_up(V * 2 * w * 4);                                      // dP
    bytes += align_up((int64_t)d * 2 * w * 4);                             // dW_int
    bytes += align_up(var_colsum_parts(V) * 2 * w * 4);                   // db parts
  }
  return bytes + 256;
}

static int variational_checks(bool ok, const float* H, int64_t V, int32_t d, int32_t w, int64_t workspace_bytes,
                              int backward, const char* who) {
  if (!ok || (H == nullptr) != (d == 0)) {
    rgcn_set_error(std::string(who) + ": null pointer (H is NULL exactly when d == 0, the embedding variant)");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = rgcn_variational_workspace_bytes(V, d, w, backward);
  if (need < 0) {
    rgcn_set_error(std::string(who) + ": need 0 <= V < 2^31, d >= 0, d % 4 == 0, w > 0, w % 4 == 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    rgcn_set_error(std::string(who) + ": no CUDA device");
    return RGCN_ERR_NODEVICE;
  }
  return RGCN_OK;
}

extern "C" int rgcn_variational_forward(const float* H, int64_t V, int32_t d, int32_t w, const float* W_mu,
                                        const float* b_mu, const float* W_sigma, const float* b_sigma,
                                        const float* eps, float* z, float* P, float* kl, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  const bool gcn = d != 0;
  int rc = variational_checks(W_mu && W_sigma && eps && z && kl && workspace && (!gcn || (b_mu && b_sigma && P)), H,
                              V, d, w, workspace_bytes, 0, "rgcn_variational_forward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0) return rgcn_check_cuda(cudaMemsetAsync(kl, 0, sizeof(float), st), "memset(kl)");
  Carver ws(workspace, workspace_bytes);
  MARK("start");
  if (!gcn) {
    float* part = ws.take<float>(var_emb_kl_parts(V, w));
    rc = launch_var_emb_forward(W_mu, W_sigma, eps, V, w, z, part, st);
    if (!rc) rc = launch_var_kl_reduce(part, var_emb_kl_parts(V, w), kl, st);
    MARK("variational_emb_fwd");
    return rc;
  }
  float* hi = ws.take<float>((int64_t)2 * 2 * w * d);
  float* lo = hi + (size_t)2 * w * d;
  float* part = ws.take<float>(gemm_variational_kl_parts(V, w));
  rc = launch_gemm_split_b_interleave(W_mu, W_sigma, d, w, /*transposed=*/1, hi, lo, st);
  if (!rc) rc = launch_gemm_variational_tf32x3(H, hi, lo, b_mu, b_sigma, eps, P, z, part, (int)V, d, w, st);
  if (!rc) rc = launch_var_kl_reduce(part, gemm_variational_kl_parts(V, w), kl, st);
  MARK("variational_gemm");
  return rc;
}

extern "C" int rgcn_variational_backward(const float* H, int64_t V, int32_t d, int32_t w, const float* W_mu,
                                         const float* W_sigma, const float* P, const float* eps, const float* dz,
                                         const float* g_kl, float* dH, float* dW_mu, float* db_mu, float* dW_sigma,
                                         float* db_sigma, void* workspace, int64_t workspace_bytes, void* stream) {
  const bool gcn = d != 0;
  int rc = variational_checks(W_mu && W_sigma && eps && dz && g_kl && dW_mu && dW_sigma && workspace &&
                                  (!gcn || (P && dH && db_mu && db_sigma)),
                              H, V, d, w, workspace_bytes, 1, "rgcn_variational_backward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  MARK("start");
  if (!gcn) {
    rc = launch_var_emb_backward(W_mu, W_sigma, eps, dz, g_kl, V, w, dW_mu, dW_sigma, st);
    MARK("variational_emb_bwd");
    return rc;
  }
  if (V == 0) {   // no rows: every gradient is zero
    rc = rgcn_check_cuda(cudaMemsetAsync(dW_mu, 0, (size_t)d * w * 4, st), "memset(dW_mu)");
    if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(dW_sigma, 0, (size_t)d * w * 4, st), "memset(dW_sigma)");
    if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(db_mu, 0, (size_t)w * 4, st), "memset(db_mu)");
    if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(db_sigma, 0, (size_t)w * 4, st), "memset(db_sigma)");
    return rc;
  }
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)2 * d * 2 * w);
  float* lo = hi + (size_t)d * 2 * w;
  float* dP = ws.take<float>(V * 2 * w);
  float* dWint = ws.take<float>((int64_t)d * 2 * w);
  float* col_part = ws.take<float>(var_colsum_parts(V) * 2 * w);
  rc = launch_var_prologue(P, eps, dz, g_kl, V, w, dP, col_part, st);
  if (!rc) rc = launch_var_colsum_finish(col_part, var_colsum_parts(V), w, db_mu, db_sigma, st);
  if (rc) return rc;
  MARK("variational_prologue");
  // dW_int = H^T dP (contraction over V), then split into the two tables
  rc = launch_gemm_tn_tf32x3(H, d, dP, 2 * w, dWint, 2 * w, d, 2 * w, (int)V, /*accumulate=*/0, st);
  if (!rc) rc = launch_var_deinterleave(dWint, d, w, dW_mu, dW_sigma, st);
  if (rc) return rc;
  MARK("variational_dW_gemm");
  // dH = dP W_int^T: Bt = W_int [N = d, K = 2w]
  rc = launch_gemm_split_b_interleave(W_mu, W_sigma, d, w, /*transposed=*/0, hi, lo, st);
  if (!rc) rc = launch_gemm_tf32x3(dP, 2 * w, hi, lo, 2 * w, dH, d, (int)V, d, 2 * w, /*accumulate=*/0, st);
  MARK("variational_dH_gemm");
  return rc;
}

// ------------------------------------------------------------------------------------------------
// DistMult
// ------------------------------------------------------------------------------------------------
extern "C" int distmult_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                int32_t d, const int32_t* X, int64_t N, const float* Y,
                                float* energies, float* loss_out, void* stream) {
  if (!codes || !rel || (N > 0 && (!X || !energies)) || !loss_out || d <= 0 || d % 4 != 0 || V <= 0 ||
      Vrel <= 0 || N < 0) {
    rgcn_set_error("distmult_forward: bad arguments (need d % 4 == 0, non-null pointers)");
    return RGCN_ERR_INVALID;
  }
  return launch_distmult_forward(codes, rel, d, X, N, Y, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int distmult_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                 int32_t d, const int32_t* X, int64_t N, const float* Y,
                                 const float* energies, float g_loss, float g_reg,
                                 const float* g_scale_dev, const float* g_energy, float* dcodes,
                                 float* drel, void* stream) {
  if (!codes || !rel || (N > 0 && !X) || !dcodes || !drel || d <= 0 || d % 4 != 0 || V <= 0 ||
      Vrel <= 0 || N < 0 || (Y && !energies)) {
    rgcn_set_error("distmult_backward: bad arguments");
    return RGCN_ERR_INVALID;
  }
  return launch_distmult_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev,
                                  g_energy, dcodes, drel, nullptr, (cudaStream_t)stream);
}

extern "C" int distmult_backward_slices(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                        const int32_t* X, int64_t N, const float* Y, const float* energies,
                                        float g_loss, float g_reg, const float* g_scale_dev, const float* g_energy,
                                        float* dcodes, float* drel, float* rel_slice_sumsq, void* stream) {
  if (!codes || !rel || (N > 0 && !X) || !dcodes || !drel || d <= 0 || d % 4 != 0 || V <= 0 ||
      Vrel <= 0 || N < 0 || (Y && !energies)) {
    rgcn_set_error("distmult_backward_slices: bad arguments");
    return RGCN_ERR_INVALID;
  }
  return launch_distmult_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev,
                                  g_energy, dcodes, drel, rel_slice_sumsq, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// IndexedSlices norm of the block tables' gradients (see slice_norm.cu)
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_block_slice_sumsq_workspace_bytes(const rgcn_graph_t* g, int32_t d, int32_t B) {
  if (!g || d <= 0 || B <= 0 || d % B != 0) {
    rgcn_set_error("rgcn_block_slice_sumsq_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  return align_up((int64_t)g->V_src * B * 4) + align_up((int64_t)g->V_dst * B * 4) + 256;
}

extern "C" int rgcn_block_slice_sumsq(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H, const float* G,
                                      float* sumsq2, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_block_slice_sumsq";
  int rc = graph_checks(g, d, B, who, false, false, false);
  if (!rc) rc = block_size_checks(d, B, who);
  if (!rc) rc = pointer_checks(H && G && sumsq2 && workspace, 1.f, who);
  if (!rc) rc = need_views(g, false, true, who);
  if (!rc) rc = workspace_checks(workspace_bytes, rgcn_block_slice_sumsq_workspace_bytes(g, d, B), who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* HB = ws.take<float>((int64_t)g->V_src * B);
  float* GB = ws.take<float>((int64_t)g->V_dst * B);
  const int s = d / B;
  rc = launch_block_sqnorm(H, g->V_src, d, B, s, HB, st);
  if (!rc) rc = launch_block_sqnorm(G, g->V_dst, d, B, s, GB, st);
  if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(sumsq2, 0, 2 * sizeof(float), st), "memset(sumsq2)");
  if (!rc)
    rc = launch_block_slice_sumsq(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row, g->by_rel.d_nbr,
                                  g->by_rel.d_norm, GB, HB, B, g->n_relw / 2, sumsq2, st);
  return rc;
}

// ------------------------------------------------------------------------------------------------
// DistMult all-entity scoring + ranking, fused (next row N3)
// ------------------------------------------------------------------------------------------------
// The decoder-independent body of the rank entry points (entity and relation queries, DistMult and ComplEx): the
// argument checks, the hi/lo split of the candidate rows (unless reused), the decoder's query rows + gold scores, the
// scoring GEMM with its rank-counting epilogue, raw/filtered ranks.  The candidates are the first N rows of `table`:
// the codes (N = V) for entity queries, the relation table (N = R) for relation queries.
// Workspace layout: [hi N*d | lo N*d | Q n*d | gold_sig n | gold_col n | raw_cnt n | known_cnt n].
typedef int (*RankPrepareFn)(const float*, const float*, int, const int32_t*, int64_t, int, float*, float*, int32_t*,
                             cudaStream_t);
// the prepare step of the rank and top-k bodies: a RankPrepareFn, or a callable that owns more state (ConvE's network)
typedef std::function<int(const float*, const float*, int, const int32_t*, int64_t, int, float*, float*, int32_t*,
                          cudaStream_t)>
    RankPrepare;
typedef int64_t (*RankWorkspaceFn)(int32_t, int32_t, int64_t);

static int rank_with_queries(const char* who, const RankPrepare& prepare, const float* table, int32_t N,
                             RankWorkspaceFn workspace_fn, const float* codes, const float* rel, int32_t V,
                             int32_t Vrel, int32_t d, const int32_t* X, int64_t n, int side,
                             const uint32_t* known_mask, int reuse_split, int32_t* raw_rank, int32_t* filtered_rank,
                             void* workspace, int64_t workspace_bytes, cudaStream_t st) {
  if (!codes || !rel || (n > 0 && (!X || !raw_rank)) || !workspace || V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 ||
      n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1)) {
    rgcn_set_error(std::string(who) + ": bad arguments (need non-null pointers, d % 4 == 0, side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  if (filtered_rank && !known_mask) {
    rgcn_set_error(std::string(who) + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = workspace_fn(N, d, n);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)N * d);
  float* lo = ws.take<float>((int64_t)N * d);
  float* Q = ws.take<float>(n * d);
  float* gold_sig = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(table, d, N, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (rc) return rc;
  rc = prepare(codes, rel, d, X, n, side, Q, gold_sig, gold_col, st);
  if (rc) return rc;
  rc = launch_gemm_rank_tf32x3(Q, d, hi, lo, d, (int)n, N, d, gold_sig, gold_col, known_mask, (N + 31) / 32, raw_cnt,
                               known_cnt, st);
  if (rc) return rc;
  return launch_distmult_rank_finalize(raw_cnt, known_cnt, n, raw_rank, filtered_rank, st);
}

extern "C" int64_t distmult_rank_workspace_bytes(int32_t V, int32_t d, int64_t n) {
  if (V <= 0 || d <= 0 || n < 0) {
    rgcn_set_error("distmult_rank_workspace_bytes: bad arguments");
    return RGCN_ERR_INVALID;
  }
  return 2 * align_up((int64_t)V * d * 4) + align_up(n * d * 4) + 4 * align_up(n * 4) + 256;
}

extern "C" int distmult_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                             const int32_t* X, int64_t n, int side, const uint32_t* known_mask, int reuse_split,
                             int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  return rank_with_queries("distmult_rank", launch_distmult_rank_prepare, codes, V, distmult_rank_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, known_mask, reuse_split, raw_rank, filtered_rank, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// ComplEx (complex.cu): scorer, backward and fused all-entity ranking
// ------------------------------------------------------------------------------------------------
extern "C" int rgcn_complex_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                    const int32_t* X, int64_t N, const float* Y, float* energies, float* loss_out,
                                    void* stream) {
  if (!codes || !rel || (N > 0 && (!X || !energies)) || !loss_out || d <= 0 || d % 4 != 0 || V <= 0 ||
      Vrel <= 0 || N < 0) {
    rgcn_set_error("rgcn_complex_forward: bad arguments (need d % 4 == 0, non-null pointers)");
    return RGCN_ERR_INVALID;
  }
  return launch_complex_forward(codes, rel, d, X, N, Y, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                     const int32_t* X, int64_t N, const float* Y, const float* energies, float g_loss,
                                     float g_reg, const float* g_scale_dev, const float* g_energy, float* dcodes,
                                     float* drel, float* rel_slice_sumsq, void* stream) {
  if (!codes || !rel || (N > 0 && !X) || !dcodes || !drel || d <= 0 || d % 4 != 0 || V <= 0 || Vrel <= 0 ||
      N < 0 || (Y && !energies)) {
    rgcn_set_error("rgcn_complex_backward: bad arguments (need d % 4 == 0, non-null pointers, energies with Y)");
    return RGCN_ERR_INVALID;
  }
  return launch_complex_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev, g_energy, dcodes,
                                 drel, rel_slice_sumsq, (cudaStream_t)stream);
}

extern "C" int64_t rgcn_complex_rank_workspace_bytes(int32_t V, int32_t d, int64_t n) {
  if (V <= 0 || d <= 0 || d % 4 != 0 || n < 0) {
    rgcn_set_error("rgcn_complex_rank_workspace_bytes: bad arguments (need d % 4 == 0)");
    return RGCN_ERR_INVALID;
  }
  return distmult_rank_workspace_bytes(V, d, n);  // same layout (rank_with_queries)
}

extern "C" int rgcn_complex_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                 const int32_t* X, int64_t n, int side, const uint32_t* known_mask, int reuse_split,
                                 int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  return rank_with_queries("rgcn_complex_rank", launch_complex_rank_prepare, codes, V, rgcn_complex_rank_workspace_bytes,
                           codes, rel, V, Vrel, d, X, n, side, known_mask, reuse_split, raw_rank, filtered_rank,
                           workspace, workspace_bytes, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Ensemble ranking (R-GCN+), fused: two members' scores combined by a weighted sum in float64
// ------------------------------------------------------------------------------------------------
// Workspace layout: [hi_A V*d_A | lo_A V*d_A | hi_B V*d_B | lo_B V*d_B | Q_A n*d_A | Q_A lo n*d_A | Q_B n*d_B |
// Q_B lo n*d_B | gold_sig_A n | gold_sig_B n | gold_col n | raw_cnt n | known_cnt n].  Q_X holds the member's query
// rows (its rank prepare kernel) and then, split in place, their TF32 hi part.
static RankPrepareFn ensemble_prepare(int32_t decoder) {
  if (decoder == RGCN_DECODER_DISTMULT) return launch_distmult_rank_prepare;
  if (decoder == RGCN_DECODER_COMPLEX) return launch_complex_rank_prepare;
  return nullptr;
}

// The body of rgcn_ensemble_rank and rgcn_ensemble_relation_rank, after their argument checks: the candidates are the
// first N rows of table_a / table_b (the codes, N = V, or the relation tables, N = R), the query rows come from
// prep_a / prep_b (the members' entity or relation prepare kernels).
static int ensemble_rank_body(RankPrepareFn prep_a, const float* table_a, RankPrepareFn prep_b, const float* table_b,
                              int32_t N, const float* codes_a, const float* rel_a, int32_t d_a, const float* codes_b,
                              const float* rel_b, int32_t d_b, double weight, const int32_t* X, int64_t n, int side,
                              const uint32_t* known_mask, int reuse_split, int32_t* raw_rank, int32_t* filtered_rank,
                              void* workspace, int64_t workspace_bytes, cudaStream_t st) {
  Carver ws(workspace, workspace_bytes);
  float* hi_a = ws.take<float>((int64_t)N * d_a);
  float* lo_a = ws.take<float>((int64_t)N * d_a);
  float* hi_b = ws.take<float>((int64_t)N * d_b);
  float* lo_b = ws.take<float>((int64_t)N * d_b);
  float* q_a = ws.take<float>(n * d_a);
  float* ql_a = ws.take<float>(n * d_a);
  float* q_b = ws.take<float>(n * d_b);
  float* ql_b = ws.take<float>(n * d_b);
  float* gs_a = ws.take<float>(n);
  float* gs_b = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  int rc = RGCN_OK;
  if (!reuse_split) {
    rc = launch_gemm_split_b(table_a, d_a, N, d_a, /*transposed=*/0, hi_a, lo_a, st);
    if (!rc) rc = launch_gemm_split_b(table_b, d_b, N, d_b, /*transposed=*/0, hi_b, lo_b, st);
  }
  if (rc || n == 0) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (!rc) rc = prep_a(codes_a, rel_a, d_a, X, n, side, q_a, gs_a, gold_col, st);
  if (!rc) rc = prep_b(codes_b, rel_b, d_b, X, n, side, q_b, gs_b, gold_col, st);   // the same gold column
  if (!rc) rc = launch_split_trunc(q_a, ql_a, n * d_a, st);
  if (!rc) rc = launch_split_trunc(q_b, ql_b, n * d_b, st);
  if (rc) return rc;
  rc = launch_gemm_ensemble_rank_tf32x3(q_a, ql_a, hi_a, lo_a, gs_a, d_a, q_b, ql_b, hi_b, lo_b, gs_b, d_b, (int)n, N,
                                        weight, 1.0 - weight, gold_col, known_mask, (N + 31) / 32, raw_cnt, known_cnt,
                                        st);
  if (rc) return rc;
  return launch_distmult_rank_finalize(raw_cnt, known_cnt, n, raw_rank, filtered_rank, st);
}

extern "C" int64_t rgcn_ensemble_rank_workspace_bytes(int32_t V, int32_t d_a, int32_t d_b, int64_t n) {
  if (V <= 0 || d_a <= 0 || d_a % 4 != 0 || d_b <= 0 || d_b % 4 != 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_ensemble_rank_workspace_bytes: bad arguments (need V > 0, d > 0, d % 4 == 0, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  return 2 * align_up((int64_t)V * d_a * 4) + 2 * align_up((int64_t)V * d_b * 4) + 2 * align_up(n * d_a * 4) +
         2 * align_up(n * d_b * 4) + 5 * align_up(n * 4) + 256;
}

// The argument checks every ensemble entry point shares; relation queries (R > 0) also need R <= Vrel of both.
static bool ensemble_args_ok(const char* who, RankPrepareFn prep_a, RankPrepareFn prep_b, const float* codes_a,
                             const float* rel_a, int32_t Vrel_a, int32_t d_a, const float* codes_b, const float* rel_b,
                             int32_t Vrel_b, int32_t d_b, int32_t V, int32_t R, double weight, const int32_t* X,
                             int64_t n, int side, const void* out, const void* workspace) {
  const std::string w(who);
  if (!prep_a || !prep_b) {
    rgcn_set_error(w + ": unknown decoder kind (RGCN_DECODER_DISTMULT or RGCN_DECODER_COMPLEX)");
    return false;
  }
  if (d_a <= 0 || d_a % 4 != 0 || d_b <= 0 || d_b % 4 != 0) {
    rgcn_set_error(w + ": bad arguments (need d % 4 == 0 for both members)");
    return false;
  }
  if (!(weight >= 0.0 && weight <= 1.0)) {   // also refuses NaN
    rgcn_set_error(w + ": bad arguments (the weight must be finite and in [0, 1])");
    return false;
  }
  if (!codes_a || !rel_a || !codes_b || !rel_b || (n > 0 && (!X || !out)) || !workspace || V <= 0 || Vrel_a <= 0 ||
      Vrel_b <= 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error(w + ": bad arguments (null pointer or bad size)");
    return false;
  }
  if (side != 0 && side != 1) {
    rgcn_set_error(w + ": bad arguments (side in {0,1})");
    return false;
  }
  if (R != 0 && (R < 1 || R > Vrel_a || R > Vrel_b)) {
    rgcn_set_error(w + ": R = " + std::to_string(R) + " relations, need 1 <= R <= Vrel of both members (" +
                   std::to_string(Vrel_a) + ", " + std::to_string(Vrel_b) + ")");
    return false;
  }
  return true;
}

static bool ensemble_k_ok(const char* who, int32_t k) {
  if (k < 1 || k > 128) {
    rgcn_set_error(std::string(who) + ": k = " + std::to_string(k) + " is out of range (1 <= k <= 128)");
    return false;
  }
  return true;
}

static bool ensemble_workspace_ok(const char* who, int64_t need, int64_t workspace_bytes) {
  if (need < 0 || workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return false;
  }
  return true;
}

extern "C" int rgcn_ensemble_rank(int32_t decoder_a, const float* codes_a, const float* rel_a, int32_t Vrel_a,
                                  int32_t d_a, int32_t decoder_b, const float* codes_b, const float* rel_b,
                                  int32_t Vrel_b, int32_t d_b, int32_t V, double weight, const int32_t* X, int64_t n,
                                  int side, const uint32_t* known_mask, int reuse_split, int32_t* raw_rank,
                                  int32_t* filtered_rank, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_ensemble_rank";
  const RankPrepareFn prep_a = ensemble_prepare(decoder_a), prep_b = ensemble_prepare(decoder_b);
  if (!ensemble_args_ok(who, prep_a, prep_b, codes_a, rel_a, Vrel_a, d_a, codes_b, rel_b, Vrel_b, d_b, V, 0, weight, X,
                        n, side, raw_rank, workspace))
    return RGCN_ERR_INVALID;
  if (filtered_rank && !known_mask) {
    rgcn_set_error(std::string(who) + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_workspace_ok(who, rgcn_ensemble_rank_workspace_bytes(V, d_a, d_b, n), workspace_bytes))
    return RGCN_ERR_WORKSPACE;
  return ensemble_rank_body(prep_a, codes_a, prep_b, codes_b, V, codes_a, rel_a, d_a, codes_b, rel_b, d_b, weight, X,
                            n, side, known_mask, reuse_split, raw_rank, filtered_rank, workspace, workspace_bytes,
                            (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Top-k prediction over all entities, fused (DistMult and ComplEx)
// ------------------------------------------------------------------------------------------------
// The decoder-independent body of distmult_topk / rgcn_complex_topk: the hi/lo split of `codes` (unless reused),
// the decoder's query rows, the scoring GEMM with its top-k epilogue (each row's best k of every 128-entity tile),
// and the merge of those candidates.
// Workspace layout: [hi V*d | lo V*d | Q n*d | cand n*ceil(V/128)*k (energy, id) pairs]; the head is the same as
// rank_with_queries', so one workspace with its split serves both.
static int64_t topk_per_row_bytes(int32_t V, int32_t d, int32_t k) {
  return (int64_t)d * 4 + (int64_t)((V + 127) / 128) * k * 8;
}

extern "C" int64_t rgcn_topk_workspace_bytes(int32_t V, int32_t d, int64_t n, int32_t k) {
  if (V <= 0 || d <= 0 || d % 4 != 0 || n < 0 || k < 1 || k > 128 ||
      (n > 0 && topk_per_row_bytes(V, d, k) > ((int64_t)1 << 60) / n)) {
    rgcn_set_error("rgcn_topk_workspace_bytes: bad arguments (need V > 0, d > 0, d % 4 == 0, n >= 0, 1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  const int64_t tn = (V + 127) / 128;
  return 2 * align_up((int64_t)V * d * 4) + align_up(n * d * 4) + align_up(n * tn * k * 8) + 256;
}

// The candidates are the first N rows of `table`, as in rank_with_queries.
typedef int64_t (*TopkWorkspaceFn)(int32_t, int32_t, int64_t, int32_t);

static int topk_with_queries(const char* who, const RankPrepare& prepare, const float* table, int32_t N,
                             TopkWorkspaceFn workspace_fn, const float* codes, const float* rel, int32_t V,
                             int32_t Vrel, int32_t d, const int32_t* X, int64_t n, int side, int32_t k,
                             const uint32_t* exclude_mask, int reuse_split, int32_t* ids, float* energies,
                             void* workspace, int64_t workspace_bytes, cudaStream_t st) {
  if (!codes || !rel || (n > 0 && (!X || !ids || !energies)) || !workspace || V <= 0 || Vrel <= 0 || d <= 0 ||
      d % 4 != 0 || n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1)) {
    rgcn_set_error(std::string(who) + ": bad arguments (need non-null pointers, d % 4 == 0, side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  if (k < 1 || k > 128) {
    rgcn_set_error(std::string(who) + ": k = " + std::to_string(k) + " is out of range (1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = workspace_fn(N, d, n, k);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  const int tn = (N + 127) / 128;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)N * d);
  float* lo = ws.take<float>((int64_t)N * d);
  float* Q = ws.take<float>(n * d);
  uint2* cand = ws.take<uint2>(n * tn * k);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(table, d, N, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = prepare(codes, rel, d, X, n, side, Q, nullptr, nullptr, st);
  if (rc) return rc;
  rc = launch_gemm_topk_tf32x3(Q, d, hi, lo, d, (int)n, N, d, exclude_mask, (N + 31) / 32, k, cand, st);
  if (rc) return rc;
  return launch_topk_merge(cand, n, tn * k, k, ids, energies, st);
}

extern "C" int distmult_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                             const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                             int reuse_split, int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  return topk_with_queries("distmult_topk", launch_distmult_rank_prepare, codes, V, rgcn_topk_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, k, exclude_mask, reuse_split, ids, energies, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                 const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                                 int reuse_split, int32_t* ids, float* energies, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  return topk_with_queries("rgcn_complex_topk", launch_complex_rank_prepare, codes, V, rgcn_topk_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, k, exclude_mask, reuse_split, ids, energies, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Relation prediction over all relations, fused (DistMult and ComplEx): queries (h, ?, t)
// ------------------------------------------------------------------------------------------------
// Both decoders' energies are linear in the relation row, so a pair query is one row Q[t] (the decoder's relation
// prepare kernel) and the energies of all relations are Q @ rel[0:R]^T: the entity-side scoring GEMM with its rank or
// top-k epilogue, run with Bt = the hi/lo split of the first R relation rows and N = R.  Rows R..Vrel-1 of `rel` (the
// R-GCN encoders keep a [V, d] relation table) are never split, scored, counted or returned.
// The entry points are rank_with_queries / topk_with_queries with the candidates rel[0:R] (N = R); one relation
// workspace with its split serves both, never the entity split.

// The relation prepare kernels in the RankPrepareFn shape: a pair query has no corruption side.
static int distmult_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int,
                                     float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  return launch_distmult_relation_prepare(codes, rel, d, X, n, Q, gold_sig, gold_col, st);
}

static int complex_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int,
                                    float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  return launch_complex_relation_prepare(codes, rel, d, X, n, Q, gold_sig, gold_col, st);
}

static bool relation_sizes_ok(int32_t R, int32_t d, int64_t n, int64_t per_row) {
  return R > 0 && d > 0 && d % 4 == 0 && n >= 0 && (n == 0 || per_row <= ((int64_t)1 << 60) / n);
}

extern "C" int64_t rgcn_relation_rank_workspace_bytes(int32_t R, int32_t d, int64_t n) {
  if (!relation_sizes_ok(R, d, n, (int64_t)d * 4 + 16)) {
    rgcn_set_error("rgcn_relation_rank_workspace_bytes: bad arguments (need R > 0, d > 0, d % 4 == 0, n >= 0)");
    return RGCN_ERR_INVALID;
  }
  return distmult_rank_workspace_bytes(R, d, n);
}

extern "C" int64_t rgcn_relation_topk_workspace_bytes(int32_t R, int32_t d, int64_t n, int32_t k) {
  if (!relation_sizes_ok(R, d, n, 0) || k < 1 || k > 128 ||
      (n > 0 && topk_per_row_bytes(R, d, k) > ((int64_t)1 << 60) / n)) {
    rgcn_set_error("rgcn_relation_topk_workspace_bytes: bad arguments (need R > 0, d > 0, d % 4 == 0, n >= 0, "
                   "1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  return rgcn_topk_workspace_bytes(R, d, n, k);
}

// the candidates are rel[0:R], which must be rows of the table
static bool relation_count_ok(const char* who, int32_t R, int32_t Vrel) {
  if (R < 1 || R > Vrel) {
    rgcn_set_error(std::string(who) + ": R = " + std::to_string(R) + " relations, need 1 <= R <= Vrel = " +
                   std::to_string(Vrel));
    return false;
  }
  return true;
}

extern "C" int distmult_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                      int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                      int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                      int64_t workspace_bytes, void* stream) {
  const char* who = "distmult_relation_rank";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return rank_with_queries(who, distmult_relation_prepare, rel, R, rgcn_relation_rank_workspace_bytes, codes, rel, V,
                           Vrel, d, X, n, 0, known_mask, reuse_split, raw_rank, filtered_rank, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                          int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                          int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                          int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_complex_relation_rank";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return rank_with_queries(who, complex_relation_prepare, rel, R, rgcn_relation_rank_workspace_bytes, codes, rel, V,
                           Vrel, d, X, n, 0, known_mask, reuse_split, raw_rank, filtered_rank, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

extern "C" int distmult_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                      int32_t d, const int32_t* X, int64_t n, int32_t k, const uint32_t* exclude_mask,
                                      int reuse_split, int32_t* ids, float* energies, void* workspace,
                                      int64_t workspace_bytes, void* stream) {
  const char* who = "distmult_relation_topk";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return topk_with_queries(who, distmult_relation_prepare, rel, R, rgcn_relation_topk_workspace_bytes, codes, rel, V,
                           Vrel, d, X, n, 0, k, exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

extern "C" int rgcn_complex_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                          int32_t d, const int32_t* X, int64_t n, int32_t k,
                                          const uint32_t* exclude_mask, int reuse_split, int32_t* ids,
                                          float* energies, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_complex_relation_topk";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return topk_with_queries(who, complex_relation_prepare, rel, R, rgcn_relation_topk_workspace_bytes, codes, rel, V,
                           Vrel, d, X, n, 0, k, exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Ensemble (R-GCN+) top-k and relation prediction, fused: the two members' entity or relation candidates in one
// two-member GEMM (k_gemm_ensemble) with the rank epilogue of rgcn_ensemble_rank or the (u, id) top-k epilogue
// ------------------------------------------------------------------------------------------------
// Entity top-k workspace: [hi_A V*d_A | lo_A | hi_B V*d_B | lo_B | Q_A n*d_A | Q_A lo | Q_B n*d_B | Q_B lo |
// cand n*ceil(V/64)*min(k,64) (u, id)]: the head is rgcn_ensemble_rank's, so one workspace with its splits serves
// both.  The relation workspaces have the same shape with the splits of rel_A[0:R] / rel_B[0:R] and N = R.
static RankPrepareFn ensemble_relation_prepare(int32_t decoder) {
  if (decoder == RGCN_DECODER_DISTMULT) return distmult_relation_prepare;
  if (decoder == RGCN_DECODER_COMPLEX) return complex_relation_prepare;
  return nullptr;
}

static int64_t ensemble_topk_bytes(int32_t N, int32_t d_a, int32_t d_b, int64_t n, int32_t k) {
  if (N <= 0 || d_a <= 0 || d_a % 4 != 0 || d_b <= 0 || d_b % 4 != 0 || n < 0 || n > 0x7fffffffLL || k < 1 ||
      k > 128)
    return RGCN_ERR_INVALID;
  const int64_t cand_per_row = (int64_t)((N + 63) / 64) * ensemble_topk_per_tile(k) * 16;
  if (n > 0 && 8 * ((int64_t)d_a + d_b) + cand_per_row > ((int64_t)1 << 60) / n) return RGCN_ERR_INVALID;
  return 2 * align_up((int64_t)N * d_a * 4) + 2 * align_up((int64_t)N * d_b * 4) + 2 * align_up(n * d_a * 4) +
         2 * align_up(n * d_b * 4) + align_up(n * cand_per_row) + 256;
}

extern "C" int64_t rgcn_ensemble_topk_workspace_bytes(int32_t V, int32_t d_a, int32_t d_b, int64_t n, int32_t k) {
  const int64_t b = ensemble_topk_bytes(V, d_a, d_b, n, k);
  if (b < 0)
    rgcn_set_error("rgcn_ensemble_topk_workspace_bytes: bad arguments (need V > 0, d > 0, d % 4 == 0, 0 <= n < 2^31, "
                   "1 <= k <= 128)");
  return b;
}

extern "C" int64_t rgcn_ensemble_relation_rank_workspace_bytes(int32_t R, int32_t d_a, int32_t d_b, int64_t n) {
  if (R <= 0) {
    rgcn_set_error("rgcn_ensemble_relation_rank_workspace_bytes: bad arguments (need R > 0)");
    return RGCN_ERR_INVALID;
  }
  return rgcn_ensemble_rank_workspace_bytes(R, d_a, d_b, n);   // the same layout with N = R
}

extern "C" int64_t rgcn_ensemble_relation_topk_workspace_bytes(int32_t R, int32_t d_a, int32_t d_b, int64_t n,
                                                               int32_t k) {
  const int64_t b = ensemble_topk_bytes(R, d_a, d_b, n, k);
  if (b < 0)
    rgcn_set_error("rgcn_ensemble_relation_topk_workspace_bytes: bad arguments (need R > 0, d > 0, d % 4 == 0, "
                   "0 <= n < 2^31, 1 <= k <= 128)");
  return b;
}

// The body of the two top-k entry points after their checks (candidates: the first N rows of table_a / table_b)
static int ensemble_topk_body(RankPrepareFn prep_a, const float* table_a, RankPrepareFn prep_b, const float* table_b,
                              int32_t N, const float* codes_a, const float* rel_a, int32_t d_a, const float* codes_b,
                              const float* rel_b, int32_t d_b, double weight, const int32_t* X, int64_t n, int side,
                              int32_t k, const uint32_t* exclude_mask, int reuse_split, int32_t* ids, double* u,
                              double* scores, void* workspace, int64_t workspace_bytes, cudaStream_t st) {
  const int kt = ensemble_topk_per_tile(k), tn = (N + 63) / 64;
  Carver ws(workspace, workspace_bytes);
  float* hi_a = ws.take<float>((int64_t)N * d_a);
  float* lo_a = ws.take<float>((int64_t)N * d_a);
  float* hi_b = ws.take<float>((int64_t)N * d_b);
  float* lo_b = ws.take<float>((int64_t)N * d_b);
  float* q_a = ws.take<float>(n * d_a);
  float* ql_a = ws.take<float>(n * d_a);
  float* q_b = ws.take<float>(n * d_b);
  float* ql_b = ws.take<float>(n * d_b);
  EnsCand* cand = ws.take<EnsCand>(n * tn * kt);
  int rc = RGCN_OK;
  if (!reuse_split) {
    rc = launch_gemm_split_b(table_a, d_a, N, d_a, /*transposed=*/0, hi_a, lo_a, st);
    if (!rc) rc = launch_gemm_split_b(table_b, d_b, N, d_b, /*transposed=*/0, hi_b, lo_b, st);
  }
  if (rc || n == 0) return rc;
  rc = prep_a(codes_a, rel_a, d_a, X, n, side, q_a, nullptr, nullptr, st);
  if (!rc) rc = prep_b(codes_b, rel_b, d_b, X, n, side, q_b, nullptr, nullptr, st);
  if (!rc) rc = launch_split_trunc(q_a, ql_a, n * d_a, st);
  if (!rc) rc = launch_split_trunc(q_b, ql_b, n * d_b, st);
  if (!rc)
    rc = launch_gemm_ensemble_topk_tf32x3(q_a, ql_a, hi_a, lo_a, d_a, q_b, ql_b, hi_b, lo_b, d_b, (int)n, N, weight,
                                          1.0 - weight, exclude_mask, (N + 31) / 32, k, cand, st);
  if (rc) return rc;
  return launch_ensemble_topk_merge(cand, n, tn * kt, k, ids, u, scores, st);
}

extern "C" int rgcn_ensemble_topk(int32_t decoder_a, const float* codes_a, const float* rel_a, int32_t Vrel_a,
                                  int32_t d_a, int32_t decoder_b, const float* codes_b, const float* rel_b,
                                  int32_t Vrel_b, int32_t d_b, int32_t V, double weight, const int32_t* X, int64_t n,
                                  int side, int32_t k, const uint32_t* exclude_mask, int reuse_split, int32_t* ids,
                                  double* u, double* scores, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_ensemble_topk";
  const RankPrepareFn prep_a = ensemble_prepare(decoder_a), prep_b = ensemble_prepare(decoder_b);
  if (!ensemble_args_ok(who, prep_a, prep_b, codes_a, rel_a, Vrel_a, d_a, codes_b, rel_b, Vrel_b, d_b, V, 0, weight, X,
                        n, side, ids, workspace) ||
      !ensemble_k_ok(who, k))
    return RGCN_ERR_INVALID;
  if (n > 0 && (!u || !scores)) {
    rgcn_set_error(std::string(who) + ": bad arguments (null pointer)");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_workspace_ok(who, ensemble_topk_bytes(V, d_a, d_b, n, k), workspace_bytes)) return RGCN_ERR_WORKSPACE;
  return ensemble_topk_body(prep_a, codes_a, prep_b, codes_b, V, codes_a, rel_a, d_a, codes_b, rel_b, d_b, weight, X, n,
                            side, k, exclude_mask, reuse_split, ids, u, scores, workspace, workspace_bytes,
                            (cudaStream_t)stream);
}

extern "C" int rgcn_ensemble_relation_rank(int32_t decoder_a, const float* codes_a, const float* rel_a,
                                           int32_t Vrel_a, int32_t d_a, int32_t decoder_b, const float* codes_b,
                                           const float* rel_b, int32_t Vrel_b, int32_t d_b, int32_t V, int32_t R,
                                           double weight, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                           int reuse_split, int32_t* raw_rank, int32_t* filtered_rank,
                                           void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_ensemble_relation_rank";
  const RankPrepareFn prep_a = ensemble_relation_prepare(decoder_a), prep_b = ensemble_relation_prepare(decoder_b);
  if (R <= 0) {
    rgcn_set_error(std::string(who) + ": R = " + std::to_string(R) + " relations, need R >= 1");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_args_ok(who, prep_a, prep_b, codes_a, rel_a, Vrel_a, d_a, codes_b, rel_b, Vrel_b, d_b, V, R, weight, X,
                        n, 0, raw_rank, workspace))
    return RGCN_ERR_INVALID;
  if (filtered_rank && !known_mask) {
    rgcn_set_error(std::string(who) + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_workspace_ok(who, rgcn_ensemble_rank_workspace_bytes(R, d_a, d_b, n), workspace_bytes))
    return RGCN_ERR_WORKSPACE;
  return ensemble_rank_body(prep_a, rel_a, prep_b, rel_b, R, codes_a, rel_a, d_a, codes_b, rel_b, d_b, weight, X, n, 0,
                            known_mask, reuse_split, raw_rank, filtered_rank, workspace, workspace_bytes,
                            (cudaStream_t)stream);
}

extern "C" int rgcn_ensemble_relation_topk(int32_t decoder_a, const float* codes_a, const float* rel_a,
                                           int32_t Vrel_a, int32_t d_a, int32_t decoder_b, const float* codes_b,
                                           const float* rel_b, int32_t Vrel_b, int32_t d_b, int32_t V, int32_t R,
                                           double weight, const int32_t* X, int64_t n, int32_t k,
                                           const uint32_t* exclude_mask, int reuse_split, int32_t* ids, double* u,
                                           double* scores, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_ensemble_relation_topk";
  const RankPrepareFn prep_a = ensemble_relation_prepare(decoder_a), prep_b = ensemble_relation_prepare(decoder_b);
  if (R <= 0) {
    rgcn_set_error(std::string(who) + ": R = " + std::to_string(R) + " relations, need R >= 1");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_args_ok(who, prep_a, prep_b, codes_a, rel_a, Vrel_a, d_a, codes_b, rel_b, Vrel_b, d_b, V, R, weight, X,
                        n, 0, ids, workspace) ||
      !ensemble_k_ok(who, k))
    return RGCN_ERR_INVALID;
  if (n > 0 && (!u || !scores)) {
    rgcn_set_error(std::string(who) + ": bad arguments (null pointer)");
    return RGCN_ERR_INVALID;
  }
  if (!ensemble_workspace_ok(who, ensemble_topk_bytes(R, d_a, d_b, n, k), workspace_bytes)) return RGCN_ERR_WORKSPACE;
  return ensemble_topk_body(prep_a, rel_a, prep_b, rel_b, R, codes_a, rel_a, d_a, codes_b, rel_b, d_b, weight, X, n, 0,
                            k, exclude_mask, reuse_split, ids, u, scores, workspace, workspace_bytes,
                            (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// 1-N training (DistMult and ComplEx): every query scored against every entity, BCE loss and gradients fused
// ------------------------------------------------------------------------------------------------
// The queries (anchor, r, side) come from the HOST, so every id is checked before any device work; they go to the
// device as the triples (anchor, r, anchor) the rank prepare kernels read, and each maximal run of one side is one
// launch of the prepare, label and query-backward kernels (callers that sort by side make two runs).
// Per chunk of c queries (cp = c rounded up to 8, so that a warp's Gt stores are whole 32 B sectors):
// Q = prepare(queries) [cp, d]; the BCE GEMM writes the loss parts and Gt [V, cp] (transposed energy gradients);
// dQ = Gt^T codes (TN GEMM, contraction over V);
// dcodes (+)= Gt Q (NT GEMM over the split of Q^T, contraction over the chunk); the query backward turns dQ and the
// L2 term into the anchor and relation gradients.  Workspace layout: [hi V*d | lo V*d | X n*3 | reg parts |
// loss parts | Q cp*d | dQ cp*d | Qt hi d*cp | Qt lo d*cp | Gt V*cp].
struct OnenRun {
  int64_t begin, end;
  int side;
};

static int onen_query_checks(const char* who, const int32_t* queries, int64_t n, int32_t V, int32_t R,
                             std::vector<OnenRun>* runs) {
  for (int64_t t = 0; t < n; ++t) {
    const int32_t a = queries[3 * t], r = queries[3 * t + 1], s = queries[3 * t + 2];
    if (a < 0 || a >= V || r < 0 || r >= R || (s != 0 && s != 1)) {
      rgcn_set_error(std::string(who) + ": query " + std::to_string(t) +
                     " is invalid (need 0 <= anchor < V, 0 <= relation < R, side in {0,1})");
      return RGCN_ERR_INVALID;
    }
    if (runs->empty() || runs->back().side != s) runs->push_back(OnenRun{t, t, s});
    runs->back().end = t + 1;
  }
  return RGCN_OK;
}

static int onen_device_checks(const char* who) {
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    rgcn_set_error(std::string(who) + ": no CUDA device");
    return RGCN_ERR_NODEVICE;
  }
  return RGCN_OK;
}

// the queries as device triples (anchor, r, anchor)
static int onen_upload(const int32_t* queries, int64_t n, int32_t* X, cudaStream_t st) {
  std::vector<int32_t> tri((size_t)n * 3);
  for (int64_t t = 0; t < n; ++t) {
    tri[3 * t] = tri[3 * t + 2] = queries[3 * t];
    tri[3 * t + 1] = queries[3 * t + 1];
  }
  // from pageable memory: the call returns once the host buffer has been read
  return rgcn_check_cuda(cudaMemcpyAsync(X, tri.data(), tri.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st),
                         "memcpy(queries)");
}

static int64_t onen_chunk(int64_t n, int64_t chunk) { return std::max<int64_t>(1, std::min(chunk, n)); }

static int64_t onen_loss_parts(int64_t n, int64_t c, int32_t V) {
  return n == 0 ? 0 : (n / c) * gemm_onen_loss_parts(c, V) + (n % c ? gemm_onen_loss_parts(n % c, V) : 0);
}

extern "C" int64_t rgcn_one_to_n_workspace_bytes(int32_t V, int32_t d, int64_t n, int64_t chunk) {
  if (V <= 0 || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL || chunk < 1) {
    rgcn_set_error("rgcn_one_to_n_workspace_bytes: bad arguments (need V > 0, d > 0, d % 4 == 0, 0 <= n < 2^31, "
                   "chunk >= 1)");
    return RGCN_ERR_INVALID;
  }
  const int64_t c = onen_chunk(n, chunk), cp = (c + 7) / 8 * 8;
  return 2 * align_up((int64_t)V * d * 4) + align_up(n * 12) + align_up(onen_reg_parts(n) * 4) +
         align_up(onen_loss_parts(n, c, V) * 4) + 2 * align_up(cp * d * 4) + 2 * align_up((int64_t)d * cp * 4) +
         align_up((int64_t)V * cp * 4) + 256;
}

// The decoder's two per-chunk steps: prepare writes the query rows Q [c1 - c0, d] of queries c0 .. c1 - 1, query_bwd
// turns their dQ and the L2 term (c_reg) into the row gradients.  X holds the uploaded queries, runs their side runs.
struct OnenChunk {
  const int32_t* X;
  const std::vector<OnenRun>* runs;
  int64_t c0, c1;
  float c_reg;
  const float* Q;   // the chunk's query rows, as prepare wrote them
};
typedef std::function<int(const OnenChunk&, float*)> OnenStep;

// DistMult and ComplEx: the rank prepare and query-backward kernels, one launch per side run in the chunk
static void onen_row_steps(int complex, const float* codes, const float* rel, int d, const float* g_scale,
                           float* dcodes, float* drel, cudaStream_t st, OnenStep* prepare, OnenStep* query_bwd) {
  const RankPrepareFn prep = complex ? launch_complex_rank_prepare : launch_distmult_rank_prepare;
  *prepare = [=](const OnenChunk& k, float* Q) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (b < e) rc = prep(codes, rel, d, k.X + 3 * b, e - b, run.side, Q + (b - k.c0) * d, nullptr, nullptr, st);
      if (rc) return rc;
    }
    return rc;
  };
  *query_bwd = [=](const OnenChunk& k, float* dQ) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (!rc && b < e)
        rc = launch_onen_query_bwd(complex, codes, rel, d, k.X + 3 * b, e - b, run.side, dQ + (b - k.c0) * d, g_scale,
                                   k.c_reg, dcodes, drel, st);
    }
    return rc;
  };
}

// repeatable: the dQ GEMM runs without split-K, so dQ and what query_bwd derives from it are bitwise repeatable
static int one_to_n(const char* who, const OnenStep& prepare, const OnenStep& query_bwd, bool repeatable,
                    const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                    const int32_t* queries, int64_t n, const uint32_t* labels, float smoothing, const float* g_scale,
                    float* loss, float* dcodes, float* drel, int64_t chunk, void* workspace, int64_t workspace_bytes,
                    cudaStream_t st) {
  if (!codes || !rel || !loss || !workspace || (n > 0 && (!queries || !labels)) || (!dcodes != !drel)) {
    rgcn_set_error(std::string(who) + ": null pointer (dcodes and drel are both given or both NULL)");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || R < 1 || R > Vrel || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL || chunk < 1) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, 1 <= R <= Vrel, d > 0, d % 4 == 0, 0 <= n < 2^31, "
                   "chunk >= 1)");
    return RGCN_ERR_INVALID;
  }
  if (!(smoothing >= 0.f && smoothing < 1.f)) {   // also refuses NaN
    rgcn_set_error(std::string(who) + ": label smoothing must be in [0, 1)");
    return RGCN_ERR_INVALID;
  }
  std::vector<OnenRun> runs;
  int rc = onen_query_checks(who, queries, n, V, R, &runs);
  if (rc) return rc;
  if (workspace_bytes < rgcn_one_to_n_workspace_bytes(V, d, n, chunk)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_one_to_n_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;

  const bool grads = dcodes != nullptr;
  if (n == 0) {   // no queries: zero loss and gradients
    rc = rgcn_check_cuda(cudaMemsetAsync(loss, 0, 2 * sizeof(float), st), "memset(loss)");
    if (!rc && grads) rc = rgcn_check_cuda(cudaMemsetAsync(dcodes, 0, (size_t)V * d * 4, st), "memset(dcodes)");
    if (!rc && grads) rc = rgcn_check_cuda(cudaMemsetAsync(drel, 0, (size_t)Vrel * d * 4, st), "memset(drel)");
    return rc;
  }
  const int64_t c = onen_chunk(n, chunk), cp = (c + 7) / 8 * 8;
  const int words = (V + 31) / 32;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)V * d);
  float* lo = ws.take<float>((int64_t)V * d);
  int32_t* X = ws.take<int32_t>(n * 3);
  float* reg_part = ws.take<float>(onen_reg_parts(n));
  float* loss_part = ws.take<float>(onen_loss_parts(n, c, V));
  float* Q = ws.take<float>(cp * d);
  float* dQ = ws.take<float>(cp * d);
  float* qt_hi = ws.take<float>((int64_t)d * cp);
  float* qt_lo = ws.take<float>((int64_t)d * cp);
  float* Gt = ws.take<float>((int64_t)V * cp);
  const float pos = (float)((1.0 - smoothing) + (double)smoothing / V), neg = (float)((double)smoothing / V);
  const float scale = (float)(1.0 / ((double)n * V));
  const float c_reg = (float)(2.0 / ((double)n * d));

  MARK("start");
  rc = onen_upload(queries, n, X, st);
  if (!rc) rc = launch_gemm_split_b(codes, d, V, d, /*transposed=*/0, hi, lo, st);
  if (!rc) rc = launch_onen_reg(codes, rel, d, X, n, reg_part, st);
  if (!rc && grads) rc = rgcn_check_cuda(cudaMemsetAsync(drel, 0, (size_t)Vrel * d * 4, st), "memset(drel)");
  if (rc) return rc;
  MARK("onen_setup");
  int64_t part = 0;
  for (int64_t c0 = 0; c0 < n; c0 += c) {
    const int64_t c1 = std::min(n, c0 + c), m = c1 - c0, mp = (m + 7) / 8 * 8;
    const OnenChunk k{X, &runs, c0, c1, c_reg, Q};
    rc = prepare(k, Q);
    if (rc) return rc;
    rc = launch_gemm_onen_tf32x3(Q, d, hi, lo, d, (int)m, V, d, labels + c0 * words, pos, neg, scale, g_scale,
                                 grads ? Gt : nullptr, mp, loss_part + part, st);
    if (rc) return rc;
    part += gemm_onen_loss_parts(m, V);
    MARK("onen_scoring_gemm");
    if (!grads) continue;
    if (mp > m) {   // the K padding of the dcodes GEMM: zero rows of Q, zero columns of Gt
      rc = rgcn_check_cuda(cudaMemsetAsync(Q + m * d, 0, (size_t)(mp - m) * d * 4, st), "memset(Q pad)");
      if (!rc)
        rc = rgcn_check_cuda(cudaMemset2DAsync(Gt + m, (size_t)mp * 4, 0, (size_t)(mp - m) * 4, V, st),
                             "memset(Gt pad)");
      if (rc) return rc;
    }
    rc = launch_gemm_tn_tf32x3(Gt, mp, codes, d, dQ, d, (int)mp, d, V, /*accumulate=*/0, st, repeatable ? 1 : 0);
    MARK("onen_dQ_gemm");
    if (!rc) rc = launch_gemm_split_b(Q, d, d, (int)mp, /*transposed=*/1, qt_hi, qt_lo, st);
    if (!rc) rc = launch_gemm_tf32x3(Gt, mp, qt_hi, qt_lo, mp, dcodes, d, V, d, (int)mp, c0 > 0, st);
    MARK("onen_dcodes_gemm");
    if (!rc) rc = query_bwd(k, dQ);
    if (rc) return rc;
    MARK("onen_query_bwd");
  }
  return launch_onen_loss_reduce(loss_part, part, reg_part, onen_reg_parts(n), 1.0 / ((double)n * V),
                                 1.0 / ((double)n * d), loss, st);
}

extern "C" int distmult_one_to_n(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                                 const int32_t* queries, int64_t n, const uint32_t* labels, float smoothing,
                                 const float* g_scale, float* loss, float* dcodes, float* drel, int64_t chunk,
                                 void* workspace, int64_t workspace_bytes, void* stream) {
  OnenStep prepare, query_bwd;
  onen_row_steps(0, codes, rel, d, g_scale, dcodes, drel, (cudaStream_t)stream, &prepare, &query_bwd);
  return one_to_n("distmult_one_to_n", prepare, query_bwd, false, codes, rel, V, Vrel, R, d, queries, n, labels,
                  smoothing, g_scale, loss, dcodes, drel, chunk, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_one_to_n(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                     int32_t d, const int32_t* queries, int64_t n, const uint32_t* labels,
                                     float smoothing, const float* g_scale, float* loss, float* dcodes, float* drel,
                                     int64_t chunk, void* workspace, int64_t workspace_bytes, void* stream) {
  OnenStep prepare, query_bwd;
  onen_row_steps(1, codes, rel, d, g_scale, dcodes, drel, (cudaStream_t)stream, &prepare, &query_bwd);
  return one_to_n("rgcn_complex_one_to_n", prepare, query_bwd, false, codes, rel, V, Vrel, R, d, queries, n, labels,
                  smoothing, g_scale, loss, dcodes, drel, chunk, workspace, workspace_bytes, (cudaStream_t)stream);
}

// The backward of a call made with g_scale = (1, 0): its dcodes / drel are the loss's gradient alone, so the gradient
// of g[0] loss[0] + g[1] loss[1] is g[0] times them plus g[1] times the L2 term's gradient, which needs no GEMM.
extern "C" int64_t rgcn_one_to_n_finish_workspace_bytes(int64_t n) {
  if (n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_one_to_n_finish_workspace_bytes: need 0 <= n < 2^31");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * 12) + 256;
}

extern "C" int rgcn_one_to_n_finish(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                                    const int32_t* queries, int64_t n, const float* g_scale, const float* dcodes_loss,
                                    const float* drel_loss, float* dcodes, float* drel, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_one_to_n_finish";
  if (!codes || !rel || !g_scale || !dcodes_loss || !drel_loss || !dcodes || !drel || !workspace ||
      (n > 0 && !queries)) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || R < 1 || R > Vrel || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, 1 <= R <= Vrel, d > 0, d % 4 == 0, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  std::vector<OnenRun> runs;
  int rc = onen_query_checks(who, queries, n, V, R, &runs);
  if (rc) return rc;
  if (workspace_bytes < rgcn_one_to_n_finish_workspace_bytes(n)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_one_to_n_finish_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = launch_onen_scale(dcodes_loss, g_scale, (int64_t)V * d, dcodes, st);
  if (!rc) rc = launch_onen_scale(drel_loss, g_scale, (int64_t)Vrel * d, drel, st);
  if (rc || n == 0) return rc;
  int32_t* X = (int32_t*)workspace;
  rc = onen_upload(queries, n, X, st);
  const float c_reg = (float)(2.0 / ((double)n * d));
  for (const OnenRun& run : runs) {   // the L2 term is the same for both decoders
    if (!rc)
      rc = launch_onen_query_bwd(0, codes, rel, d, X + 3 * run.begin, run.end - run.begin, run.side, nullptr, g_scale,
                                 c_reg, dcodes, drel, st);
  }
  return rc;
}

extern "C" int64_t rgcn_one_to_n_labels_workspace_bytes(int64_t n) {
  if (n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_one_to_n_labels_workspace_bytes: need 0 <= n < 2^31");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * 12) + 256;
}

extern "C" int rgcn_one_to_n_labels(const int64_t* keys, const int64_t* offsets, const int32_t* entities,
                                    int64_t n_keys, int32_t V, int32_t R, const int32_t* queries, int64_t n,
                                    uint32_t* bits, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_one_to_n_labels";
  if (!offsets || !workspace || (n_keys > 0 && (!keys || !entities)) || (n > 0 && (!queries || !bits))) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || R <= 0 || n_keys < 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, R > 0, n_keys >= 0, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  std::vector<OnenRun> runs;
  int rc = onen_query_checks(who, queries, n, V, R, &runs);
  if (rc) return rc;
  if (workspace_bytes < rgcn_one_to_n_labels_workspace_bytes(n)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_one_to_n_labels_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc || n == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* X = (int32_t*)workspace;
  rc = onen_upload(queries, n, X, st);
  const int words = (V + 31) / 32;
  for (const OnenRun& run : runs) {
    if (!rc)
      rc = launch_onen_labels(keys, offsets, entities, n_keys, X + 3 * run.begin, run.end - run.begin, run.side, V,
                              words, bits + run.begin * words, st);
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------
// ConvE (conve.cu): the query network in front of the 1-N, rank and top-k bodies above
// ------------------------------------------------------------------------------------------------
// Evaluation queries run through the network in passes of this many rows (the feature rows of a pass are F floats
// each, about 112 KB at d = 500, h = 20, C = 32)
constexpr int64_t CONVE_EVAL_CHUNK = 1024;

static int64_t conve_F(int32_t d, int32_t h, int32_t C) { return (int64_t)C * (2 * h - 2) * (d / h - 2); }
static int64_t conve_Fp(int32_t d, int32_t h, int32_t C) { return (conve_F(d, h, C) + 3) / 4 * 4; }

static bool conve_shape_ok(int32_t d, int32_t h, int32_t C) {
  return d > 0 && d % 4 == 0 && h >= 2 && d % h == 0 && d / h >= 3 && C >= 1 && conve_F(d, h, C) < (1LL << 30) &&
         conve_smem_bytes(d, h, d / h, C) <= 227 * 1024;
}

static int conve_net_checks(const char* who, int32_t d, const rgcn_conve_net_t* net) {
  const std::string w(who);
  if (!net || !net->rel_inv || !net->filters || !net->conv_bias || !net->W_fc || !net->b_fc) {
    rgcn_set_error(w + ": null pointer in the network (rel_inv, filters, conv_bias, W_fc, b_fc)");
    return RGCN_ERR_INVALID;
  }
  if (!conve_shape_ok(d, net->h, net->C)) {
    rgcn_set_error(w + ": bad shape (need d % 4 == 0, h >= 2, d = h w with w >= 3, C >= 1)");
    return RGCN_ERR_INVALID;
  }
  for (float k : {net->input_keep, net->feature_keep, net->hidden_keep}) {
    if (!(k > 0.f && k <= 1.f)) {   // also refuses NaN
      rgcn_set_error(w + ": keep probabilities must be in (0, 1]");
      return RGCN_ERR_INVALID;
    }
  }
  return RGCN_OK;
}

// The network's workspace for passes of up to c queries (cp = c rounded up to 8): the splits of W_fc for the forward
// ([d, Fp]) and the backward ([Fp, d]), the feature rows [cp, Fp]; with grads, the split of the feature rows'
// transpose [Fp, cp] (whose hi plane then holds dF [cp, Fp]), dZ [cp, d], dZt [d, cp], dWt [d, Fp] and the filter
// parts.
struct ConvEWork {
  float *wt_hi, *wt_lo, *w_hi, *w_lo, *feat, *ft_hi, *ft_lo, *dz, *dzt, *dwt, *part;
};

static int64_t conve_work_bytes(int32_t d, int32_t h, int32_t C, int64_t c, bool grads) {
  const int64_t Fp = conve_Fp(d, h, C), cp = (std::max<int64_t>(c, 1) + 7) / 8 * 8;
  int64_t b = 2 * align_up(d * Fp * 4) + align_up(cp * Fp * 4);
  if (grads)
    b += 2 * align_up(Fp * d * 4) + 2 * align_up(Fp * cp * 4) + 2 * align_up(cp * d * 4) + align_up(d * Fp * 4) +
         align_up(conve_conv_parts(cp) * 10 * C * 4);
  return b;
}

static ConvEWork conve_carve(Carver& ws, int32_t d, int32_t h, int32_t C, int64_t c, bool grads) {
  const int64_t Fp = conve_Fp(d, h, C), cp = (std::max<int64_t>(c, 1) + 7) / 8 * 8;
  ConvEWork w{};
  w.wt_hi = ws.take<float>(d * Fp);
  w.wt_lo = ws.take<float>(d * Fp);
  w.feat = ws.take<float>(cp * Fp);
  if (grads) {
    w.w_hi = ws.take<float>(Fp * d);
    w.w_lo = ws.take<float>(Fp * d);
    w.ft_hi = ws.take<float>(Fp * cp);
    w.ft_lo = ws.take<float>(Fp * cp);
    w.dz = ws.take<float>(cp * d);
    w.dzt = ws.take<float>(d * cp);
    w.dwt = ws.take<float>(d * Fp);
    w.part = ws.take<float>(conve_conv_parts(cp) * 10 * C);
  }
  return w;
}

static const uint8_t* mask_rows(const uint8_t* m, int64_t row0, int64_t width) {
  return m ? m + row0 * width : nullptr;
}

// Q [m, d] of the queries X[0 .. m) (anchor in column acol, relation row reltab[X[t][1]], mask rows from row0); the
// feature rows stay in w.feat for the backward.  The forward split of W_fc must be in w.wt_hi / w.wt_lo.
static int conve_forward(const float* codes, const float* reltab, int32_t d, const rgcn_conve_net_t* net,
                         const int32_t* X, int acol, int64_t m, int64_t row0, const ConvEWork& w, float* Q,
                         cudaStream_t st) {
  const int Fp = (int)conve_Fp(d, net->h, net->C);
  int rc = launch_conve_conv_fwd(codes, reltab, d, net->h, net->C, X, acol, m, net->filters, net->conv_bias,
                                 mask_rows(net->input_mask, row0, 2 * d), 1.f / net->input_keep,
                                 mask_rows(net->feature_mask, row0, net->C), 1.f / net->feature_keep, Fp, w.feat, st);
  if (!rc) rc = launch_gemm_tf32x3(w.feat, Fp, w.wt_hi, w.wt_lo, Fp, Q, d, (int)m, d, Fp, /*accumulate=*/0, st);
  if (!rc)
    rc = launch_conve_fc_act(Q, m, d, net->b_fc, mask_rows(net->hidden_mask, row0, d), 1.f / net->hidden_keep, st);
  return rc;
}

// The evaluation prepare: the forward split of W_fc, then Q of the n triples X of one side in passes of
// CONVE_EVAL_CHUNK, and (gold_sig non-null) the gold scores
static RankPrepare conve_prepare(const rgcn_conve_net_t* net, const ConvEWork& w) {
  return [net, w](const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side, float* Q,
                  float* gold_sig, int32_t* gold_col, cudaStream_t st) {
    const int F = (int)conve_F(d, net->h, net->C), Fp = (int)conve_Fp(d, net->h, net->C);
    int rc = launch_conve_split_w(net->W_fc, F, d, Fp, /*transposed=*/1, w.wt_hi, w.wt_lo, st);
    const float* reltab = side == 0 ? net->rel_inv : rel;
    for (int64_t c0 = 0; !rc && c0 < n; c0 += CONVE_EVAL_CHUNK) {
      const int64_t m = std::min(CONVE_EVAL_CHUNK, n - c0);
      rc = conve_forward(codes, reltab, d, net, X + 3 * c0, side == 0 ? 2 : 0, m, c0, w, Q + c0 * d, st);
    }
    if (!rc && gold_sig) rc = launch_conve_gold(Q, codes, d, X, n, side, gold_sig, gold_col, st);
    return rc;
  };
}

extern "C" int64_t rgcn_conve_one_to_n_workspace_bytes(int32_t V, int32_t R, int32_t d, int32_t h, int32_t C,
                                                       int64_t n, int64_t chunk) {
  if (R < 1 || !conve_shape_ok(d, h, C) || V <= 0 || n < 0 || n > 0x7fffffffLL || chunk < 1) {
    rgcn_set_error("rgcn_conve_one_to_n_workspace_bytes: bad arguments (need V > 0, R > 0, a valid ConvE shape, "
                   "0 <= n < 2^31, chunk >= 1)");
    return RGCN_ERR_INVALID;
  }
  // [1-N body | relation rows [rel ; rel_inv] and their gradient | network]
  return rgcn_one_to_n_workspace_bytes(V, d, n, chunk) + 2 * align_up((int64_t)2 * R * d * 4) +
         conve_work_bytes(d, h, C, onen_chunk(n, chunk), true) + 256;
}

static bool conve_grads_ok(const rgcn_conve_grads_t* g) {
  return g && g->rel_inv && g->filters && g->conv_bias && g->W_fc && g->b_fc;
}

// The 1-N body with the relation table [rel[0:R] ; rel_inv] (2R rows): a subject query (a, r, 0) reads row R + r, so
// the body's L2 term and the network's image gradient need no side; drel and grads->rel_inv are split from its
// gradient afterwards.
extern "C" int rgcn_conve_one_to_n(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                                   const rgcn_conve_net_t* net, const int32_t* queries, int64_t n,
                                   const uint32_t* labels, float smoothing, const float* g_scale, float* loss,
                                   float* dcodes, float* drel, const rgcn_conve_grads_t* grads, int64_t chunk,
                                   void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_conve_one_to_n";
  cudaStream_t st = (cudaStream_t)stream;
  if (!codes || !rel || !loss || !workspace || (n > 0 && (!queries || !labels)) || (!dcodes != !drel) ||
      (dcodes && !conve_grads_ok(grads))) {
    rgcn_set_error(std::string(who) + ": null pointer (dcodes, drel and the five network gradients are all given or "
                   "dcodes and drel are both NULL)");
    return RGCN_ERR_INVALID;
  }
  int rc = conve_net_checks(who, d, net);
  if (rc) return rc;
  if (V <= 0 || Vrel <= 0 || R < 1 || R > Vrel || n < 0 || n > 0x7fffffffLL || chunk < 1) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, 1 <= R <= Vrel, 0 <= n < 2^31, chunk >= 1)");
    return RGCN_ERR_INVALID;
  }
  if (!(smoothing >= 0.f && smoothing < 1.f)) {
    rgcn_set_error(std::string(who) + ": label smoothing must be in [0, 1)");
    return RGCN_ERR_INVALID;
  }
  std::vector<OnenRun> runs;
  rc = onen_query_checks(who, queries, n, V, R, &runs);
  if (rc) return rc;
  const int64_t body = rgcn_one_to_n_workspace_bytes(V, d, n, chunk);
  if (body < 0 || workspace_bytes < rgcn_conve_one_to_n_workspace_bytes(V, R, d, net->h, net->C, n, chunk)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_conve_one_to_n_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;

  const bool grads_on = dcodes != nullptr;
  const int h = net->h, C = net->C, F = (int)conve_F(d, h, C), Fp = (int)conve_Fp(d, h, C);
  if (n == 0) {   // no queries: zero loss and gradients
    rc = rgcn_check_cuda(cudaMemsetAsync(loss, 0, 2 * sizeof(float), st), "memset(loss)");
    if (grads_on) {
      const std::pair<float*, int64_t> zero[] = {{dcodes, (int64_t)V * d}, {drel, (int64_t)Vrel * d},
                                                 {grads->rel_inv, (int64_t)R * d}, {grads->filters, 9LL * C},
                                                 {grads->conv_bias, C}, {grads->W_fc, (int64_t)F * d},
                                                 {grads->b_fc, d}};
      for (const auto& z : zero)
        if (!rc) rc = rgcn_check_cuda(cudaMemsetAsync(z.first, 0, (size_t)z.second * 4, st), "memset(gradient)");
    }
    return rc;
  }
  Carver ws((char*)workspace + body, workspace_bytes - body);
  float* relcat = ws.take<float>((int64_t)2 * R * d);
  float* drelcat = ws.take<float>((int64_t)2 * R * d);
  const ConvEWork w = conve_carve(ws, d, h, C, onen_chunk(n, chunk), grads_on);
  std::vector<int32_t> q2(queries, queries + 3 * n);
  for (int64_t t = 0; t < n; ++t)
    if (q2[3 * t + 2] == 0) q2[3 * t + 1] += R;

  rc = rgcn_check_cuda(cudaMemcpyAsync(relcat, rel, (size_t)R * d * 4, cudaMemcpyDeviceToDevice, st), "copy(rel)");
  if (!rc)
    rc = rgcn_check_cuda(cudaMemcpyAsync(relcat + (size_t)R * d, net->rel_inv, (size_t)R * d * 4,
                                         cudaMemcpyDeviceToDevice, st), "copy(rel_inv)");
  if (!rc) rc = launch_conve_split_w(net->W_fc, F, d, Fp, /*transposed=*/1, w.wt_hi, w.wt_lo, st);
  if (!rc && grads_on) rc = launch_conve_split_w(net->W_fc, F, d, Fp, /*transposed=*/0, w.w_hi, w.w_lo, st);
  if (rc) return rc;

  const OnenStep prepare = [=](const OnenChunk& k, float* Q) {
    return conve_forward(codes, relcat, d, net, k.X + 3 * k.c0, 0, k.c1 - k.c0, k.c0, w, Q, st);
  };
  // dZ through the ReLU and the hidden mask; db_fc, dW_fc^T (+)= dZ^T Feat, dF = dZ W_fc^T, the convolution backward;
  // then the L2 term of the two gathered rows
  const OnenStep query_bwd = [=](const OnenChunk& k, float* dQ) {
    const int64_t c0 = k.c0, m = k.c1 - c0, mp = (m + 7) / 8 * 8;
    const int acc = c0 > 0;   // the network gradients accumulate over the chunks
    int rc = launch_conve_dz(k.Q, dQ, m, d, mask_rows(net->hidden_mask, c0, d), 1.f / net->hidden_keep, w.dz, w.dzt,
                             mp, st);
    if (!rc) rc = launch_conve_rowsum(w.dzt, d, m, mp, grads->b_fc, acc, st);
    if (!rc && mp > m)   // the K padding of the dW GEMM: zero feature rows, zero columns of dZt
      rc = rgcn_check_cuda(cudaMemsetAsync(w.feat + m * Fp, 0, (size_t)(mp - m) * Fp * 4, st), "memset(Feat pad)");
    if (!rc) rc = launch_gemm_split_b(w.feat, Fp, Fp, (int)mp, /*transposed=*/1, w.ft_hi, w.ft_lo, st);
    if (!rc) rc = launch_gemm_tf32x3(w.dzt, mp, w.ft_hi, w.ft_lo, mp, w.dwt, Fp, d, Fp, (int)mp, acc, st);
    float* dF = w.ft_hi;   // the split of Feat^T is consumed
    if (!rc) rc = launch_gemm_tf32x3(w.dz, d, w.w_hi, w.w_lo, d, dF, Fp, (int)m, Fp, d, /*accumulate=*/0, st);
    if (!rc)
      rc = launch_conve_conv_bwd(codes, relcat, d, h, C, k.X + 3 * c0, m, net->filters,
                                 mask_rows(net->input_mask, c0, 2 * d), 1.f / net->input_keep, w.feat, dF,
                                 1.f / net->feature_keep, Fp, w.part, dcodes, drelcat, st);
    if (!rc)
      rc = launch_conve_filter_reduce(w.part, (int)conve_conv_parts(m), C, grads->filters, grads->conv_bias, acc,
                                      st);
    if (!rc)
      rc = launch_onen_query_bwd(0, codes, relcat, d, k.X + 3 * c0, m, 1, nullptr, g_scale, k.c_reg, dcodes, drelcat,
                                 st);
    return rc;
  };
  rc = one_to_n(who, prepare, query_bwd, true, codes, relcat, V, 2 * R, 2 * R, d, q2.data(), n, labels, smoothing,
                g_scale, loss, dcodes, grads_on ? drelcat : nullptr, chunk, workspace, workspace_bytes, st);
  if (rc || !grads_on) return rc;
  rc = launch_conve_transpose(w.dwt, F, d, Fp, grads->W_fc, st);
  if (!rc)
    rc = rgcn_check_cuda(cudaMemcpyAsync(drel, drelcat, (size_t)R * d * 4, cudaMemcpyDeviceToDevice, st), "copy(drel)");
  if (!rc && Vrel > R)
    rc = rgcn_check_cuda(cudaMemsetAsync(drel + (size_t)R * d, 0, (size_t)(Vrel - R) * d * 4, st), "memset(drel)");
  if (!rc)
    rc = rgcn_check_cuda(cudaMemcpyAsync(grads->rel_inv, drelcat + (size_t)R * d, (size_t)R * d * 4,
                                         cudaMemcpyDeviceToDevice, st), "copy(drel_inv)");
  return rc;
}

extern "C" int64_t rgcn_conve_one_to_n_finish_workspace_bytes(int64_t n) {
  if (n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_conve_one_to_n_finish_workspace_bytes: need 0 <= n < 2^31");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * 12) + 256;
}

extern "C" int rgcn_conve_one_to_n_finish(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                          int32_t d, const rgcn_conve_net_t* net, const int32_t* queries, int64_t n,
                                          const float* g_scale, const float* dcodes_loss, const float* drel_loss,
                                          const rgcn_conve_grads_t* loss_grads, float* dcodes, float* drel,
                                          const rgcn_conve_grads_t* grads, void* workspace, int64_t workspace_bytes,
                                          void* stream) {
  const char* who = "rgcn_conve_one_to_n_finish";
  if (!codes || !rel || !g_scale || !dcodes_loss || !drel_loss || !conve_grads_ok(loss_grads) || !dcodes || !drel ||
      !conve_grads_ok(grads) || !workspace || (n > 0 && !queries)) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  int rc = conve_net_checks(who, d, net);
  if (rc) return rc;
  if (V <= 0 || Vrel <= 0 || R < 1 || R > Vrel || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, 1 <= R <= Vrel, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  std::vector<OnenRun> runs;
  rc = onen_query_checks(who, queries, n, V, R, &runs);
  if (rc) return rc;
  if (workspace_bytes < rgcn_conve_one_to_n_finish_workspace_bytes(n)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_conve_one_to_n_finish_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int C = net->C;
  rc = launch_onen_scale(dcodes_loss, g_scale, (int64_t)V * d, dcodes, st);
  if (!rc) rc = launch_onen_scale(drel_loss, g_scale, (int64_t)Vrel * d, drel, st);
  if (!rc) rc = launch_onen_scale(loss_grads->rel_inv, g_scale, (int64_t)R * d, grads->rel_inv, st);
  if (!rc) rc = launch_conve_scale(loss_grads->filters, g_scale, 9LL * C, grads->filters, st);
  if (!rc) rc = launch_conve_scale(loss_grads->conv_bias, g_scale, C, grads->conv_bias, st);
  if (!rc) rc = launch_conve_scale(loss_grads->W_fc, g_scale, conve_F(d, net->h, C) * d, grads->W_fc, st);
  if (!rc) rc = launch_conve_scale(loss_grads->b_fc, g_scale, d, grads->b_fc, st);
  if (rc || n == 0) return rc;
  int32_t* X = (int32_t*)workspace;
  rc = onen_upload(queries, n, X, st);
  const float c_reg = (float)(2.0 / ((double)n * d));
  for (const OnenRun& run : runs) {   // the L2 term: object queries read rel, subject queries rel_inv
    const bool inv = run.side == 0;
    if (!rc)
      rc = launch_onen_query_bwd(0, codes, inv ? net->rel_inv : rel, d, X + 3 * run.begin, run.end - run.begin,
                                 run.side, nullptr, g_scale, c_reg, dcodes, inv ? grads->rel_inv : drel, st);
  }
  return rc;
}

// the evaluation entries' shared checks (X, side, R)
static int conve_eval_checks(const char* who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                             int32_t R, int32_t d, const rgcn_conve_net_t* net, const int32_t* X, int64_t n, int side) {
  if (!codes || !rel || (n > 0 && !X)) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  int rc = conve_net_checks(who, d, net);
  if (rc) return rc;
  if (V <= 0 || Vrel <= 0 || R < 1 || R > Vrel || n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1)) {
    rgcn_set_error(std::string(who) + ": bad sizes (need V > 0, 1 <= R <= Vrel, 0 <= n < 2^31, side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

extern "C" int64_t rgcn_conve_query_rows_workspace_bytes(int32_t d, int32_t h, int32_t C, int64_t n) {
  if (!conve_shape_ok(d, h, C) || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_conve_query_rows_workspace_bytes: bad arguments (need a valid ConvE shape, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  return conve_work_bytes(d, h, C, std::min(n, CONVE_EVAL_CHUNK), false) + 256;
}

extern "C" int rgcn_conve_query_rows(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                     int32_t d, const rgcn_conve_net_t* net, const int32_t* X, int64_t n, int side,
                                     float* Q, void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_conve_query_rows";
  int rc = conve_eval_checks(who, codes, rel, V, Vrel, R, d, net, X, n, side);
  if (rc) return rc;
  if (!workspace || (n > 0 && !Q)) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_conve_query_rows_workspace_bytes(d, net->h, net->C, n)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_conve_query_rows_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc || n == 0) return rc;
  Carver ws(workspace, workspace_bytes);
  const ConvEWork w = conve_carve(ws, d, net->h, net->C, std::min(n, CONVE_EVAL_CHUNK), false);
  return conve_prepare(net, w)(codes, rel, d, X, n, side, Q, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int64_t rgcn_conve_rank_workspace_bytes(int32_t V, int32_t d, int32_t h, int32_t C, int64_t n) {
  if (!conve_shape_ok(d, h, C) || V <= 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_conve_rank_workspace_bytes: bad arguments (need V > 0, a valid ConvE shape, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  // [distmult_rank's workspace (its split of codes reused) | network]
  return distmult_rank_workspace_bytes(V, d, n) + conve_work_bytes(d, h, C, std::min(n, CONVE_EVAL_CHUNK), false);
}

extern "C" int rgcn_conve_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                               const rgcn_conve_net_t* net, const int32_t* X, int64_t n, int side,
                               const uint32_t* known_mask, int reuse_split, int32_t* raw_rank, int32_t* filtered_rank,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_conve_rank";
  int rc = conve_eval_checks(who, codes, rel, V, Vrel, R, d, net, X, n, side);
  if (rc) return rc;
  if (!workspace) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_conve_rank_workspace_bytes(V, d, net->h, net->C, n)) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_conve_rank_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;
  const int64_t body = distmult_rank_workspace_bytes(V, d, n);
  Carver ws((char*)workspace + body, workspace_bytes - body);
  const ConvEWork w = conve_carve(ws, d, net->h, net->C, std::min(n, CONVE_EVAL_CHUNK), false);
  return rank_with_queries(who, conve_prepare(net, w), codes, V, distmult_rank_workspace_bytes, codes, rel, V, Vrel, d,
                           X, n, side, known_mask, reuse_split, raw_rank, filtered_rank, workspace, body,
                           (cudaStream_t)stream);
}

extern "C" int64_t rgcn_conve_topk_workspace_bytes(int32_t V, int32_t d, int32_t h, int32_t C, int64_t n, int32_t k) {
  if (!conve_shape_ok(d, h, C) || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error("rgcn_conve_topk_workspace_bytes: bad arguments (need a valid ConvE shape, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  const int64_t body = rgcn_topk_workspace_bytes(V, d, n, k);
  if (body < 0) return body;
  return body + conve_work_bytes(d, h, C, std::min(n, CONVE_EVAL_CHUNK), false);
}

extern "C" int rgcn_conve_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                               const rgcn_conve_net_t* net, const int32_t* X, int64_t n, int side, int32_t k,
                               const uint32_t* exclude_mask, int reuse_split, int32_t* ids, float* energies,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_conve_topk";
  int rc = conve_eval_checks(who, codes, rel, V, Vrel, R, d, net, X, n, side);
  if (rc) return rc;
  if (!workspace) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = rgcn_conve_topk_workspace_bytes(V, d, net->h, net->C, n, k);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_conve_topk_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who);
  if (rc) return rc;
  const int64_t body = rgcn_topk_workspace_bytes(V, d, n, k);
  Carver ws((char*)workspace + body, workspace_bytes - body);
  const ConvEWork w = conve_carve(ws, d, net->h, net->C, std::min(n, CONVE_EVAL_CHUNK), false);
  return topk_with_queries(who, conve_prepare(net, w), codes, V, rgcn_topk_workspace_bytes, codes, rel, V, Vrel, d, X,
                           n, side, k, exclude_mask, reuse_split, ids, energies, workspace, body, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Self-adversarial negative sampling (DistMult and ComplEx): the per-positive softmax weights over its corruptions
// and the weighted loss in one kernel (self_adversarial.cu); the backward is the scorer's own with g_energy = coef.
// Workspace layout: [loss parts n | norm parts n], n = N / (K + 1).
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_self_adversarial_workspace_bytes(int64_t N, int32_t K) {
  if (N < 0 || K < 1 || N % ((int64_t)K + 1) != 0) {
    rgcn_set_error("rgcn_self_adversarial_workspace_bytes: bad arguments (need N >= 0, K >= 1, N % (K + 1) == 0)");
    return RGCN_ERR_INVALID;
  }
  return align_up(2 * (N / ((int64_t)K + 1)) * 4) + 256;
}

// the argument checks of both self-adversarial entry points, in order, before any device work
static int self_adversarial_checks(const std::string& who, bool pointers_ok, int32_t V, int32_t Vrel, int32_t d,
                                   int64_t N, int32_t K, float alpha, int64_t workspace_bytes) {
  if (!pointers_ok) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || N < 0) {
    rgcn_set_error(who + ": bad sizes (need V > 0, Vrel > 0, d > 0, d % 4 == 0, N >= 0)");
    return RGCN_ERR_INVALID;
  }
  if (K < 1 || N % ((int64_t)K + 1) != 0) {
    rgcn_set_error(who + ": N = " + std::to_string(N) + " triples are not n positives with K = " + std::to_string(K) +
                   " corruptions each (need K >= 1 and N % (K + 1) == 0)");
    return RGCN_ERR_INVALID;
  }
  if (!(alpha >= 0.0f && alpha < INFINITY)) {   // also refuses NaN
    rgcn_set_error(who + ": the adversarial temperature must be finite and >= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_self_adversarial_workspace_bytes(N, K)) {
    rgcn_set_error(who + ": workspace too small (rgcn_self_adversarial_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  return onen_device_checks(who.c_str());
}

extern "C" int rgcn_self_adversarial_forward(int32_t decoder, const float* codes, const float* rel, int32_t V,
                                             int32_t Vrel, int32_t d, const int32_t* X, int64_t N, int32_t K,
                                             float alpha, float* energies, float* coef, float* loss_out,
                                             void* workspace, int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_self_adversarial_forward";
  if (decoder != RGCN_DECODER_DISTMULT && decoder != RGCN_DECODER_COMPLEX) {
    rgcn_set_error(who + ": unknown decoder kind (RGCN_DECODER_DISTMULT or RGCN_DECODER_COMPLEX)");
    return RGCN_ERR_INVALID;
  }
  const int rc = self_adversarial_checks(
      who, codes && rel && loss_out && workspace && (N <= 0 || (X && energies && coef)), V, Vrel, d, N, K, alpha,
      workspace_bytes);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* parts = ws.take<float>(2 * (N / ((int64_t)K + 1)));
  return launch_self_adversarial_forward(decoder == RGCN_DECODER_COMPLEX ? SELFADV_COMPLEX : SELFADV_DISTMULT, codes,
                                         rel, d, X, N, K, alpha, 0.f, energies, coef, loss_out, parts,
                                         (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// RotatE (rotate.cu): scorer, backward, self-adversarial forward and all-entity ranking by distance.  Every argument
// is checked before any device work, with the ComplEx rules plus a finite gamma.
// ------------------------------------------------------------------------------------------------
static int rotate_checks(const std::string& who, bool pointers_ok, int32_t V, int32_t Vrel, int32_t d, int64_t N,
                         float gamma) {
  if (!pointers_ok) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || N < 0) {
    rgcn_set_error(who + ": bad sizes (need V > 0, Vrel > 0, d > 0, d % 4 == 0, N >= 0)");
    return RGCN_ERR_INVALID;
  }
  if (!std::isfinite(gamma)) {
    rgcn_set_error(who + ": the margin gamma must be finite");
    return RGCN_ERR_INVALID;
  }
  return onen_device_checks(who.c_str());
}

extern "C" int rgcn_rotate_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                   const int32_t* X, int64_t N, const float* Y, float gamma, float* energies,
                                   float* loss_out, void* stream) {
  const int rc = rotate_checks("rgcn_rotate_forward", codes && rel && loss_out && (N <= 0 || (X && energies)), V, Vrel,
                               d, N, gamma);
  if (rc) return rc;
  return launch_rotate_forward(codes, rel, d, X, N, Y, gamma, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int rgcn_rotate_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                    const int32_t* X, int64_t N, const float* Y, float gamma, const float* energies,
                                    float g_loss, float g_reg, const float* g_scale_dev, const float* g_energy,
                                    float* dcodes, float* drel, float* rel_slice_sumsq, void* stream) {
  const int rc = rotate_checks("rgcn_rotate_backward",
                               codes && rel && dcodes && drel && (N <= 0 || X) && (!Y || energies), V, Vrel, d, N,
                               gamma);
  if (rc) return rc;
  return launch_rotate_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev, g_energy, dcodes, drel,
                                rel_slice_sumsq, (cudaStream_t)stream);
}

extern "C" int rgcn_rotate_self_adversarial_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                                    int32_t d, const int32_t* X, int64_t N, int32_t K, float alpha,
                                                    float gamma, float* energies, float* coef, float* loss_out,
                                                    void* workspace, int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_rotate_self_adversarial_forward";
  if (!std::isfinite(gamma)) {
    rgcn_set_error(who + ": the margin gamma must be finite");
    return RGCN_ERR_INVALID;
  }
  const int rc = self_adversarial_checks(
      who, codes && rel && loss_out && workspace && (N <= 0 || (X && energies && coef)), V, Vrel, d, N, K, alpha,
      workspace_bytes);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* parts = ws.take<float>(2 * (N / ((int64_t)K + 1)));
  return launch_self_adversarial_forward(SELFADV_ROTATE, codes, rel, d, X, N, K, alpha, gamma, energies, coef,
                                         loss_out, parts, (cudaStream_t)stream);
}

// Workspace layout: [Q n*d | gold_D n | gold_col n | raw_cnt n | known_cnt n]
extern "C" int64_t rgcn_rotate_rank_workspace_bytes(int32_t V, int32_t d, int64_t n) {
  if (V <= 0 || d <= 0 || d % 4 != 0 || n < 0) {
    rgcn_set_error("rgcn_rotate_rank_workspace_bytes: bad arguments (need V > 0, d % 4 == 0, n >= 0)");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * d * 4) + 4 * align_up(n * 4) + 256;
}

extern "C" int rgcn_rotate_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                const int32_t* X, int64_t n, int side, const uint32_t* known_mask,
                                int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                                void* stream) {
  const std::string who = "rgcn_rotate_rank";
  if (!codes || !rel || !workspace || (n > 0 && (!X || !raw_rank))) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1)) {
    rgcn_set_error(who + ": bad arguments (need V > 0, Vrel > 0, d % 4 == 0, 0 <= n < 2^31, side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  if (filtered_rank && !known_mask) {
    rgcn_set_error(who + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_rotate_rank_workspace_bytes(V, d, n)) {
    rgcn_set_error(who + ": workspace too small (rgcn_rotate_rank_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  int rc = onen_device_checks(who.c_str());
  if (rc || n == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Carver ws(workspace, workspace_bytes);
  float* Q = ws.take<float>(n * d);
  float* gold_D = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (!rc) rc = launch_rotate_rank_prepare(codes, rel, d, X, n, side, Q, gold_D, gold_col, st);
  if (!rc) rc = launch_rotate_rank(Q, codes, V, d, n, gold_D, gold_col, known_mask, raw_cnt, known_cnt, st);
  if (!rc) rc = launch_distmult_rank_finalize(raw_cnt, known_cnt, n, raw_rank, filtered_rank, st);
  return rc;
}

// ------------------------------------------------------------------------------------------------
// TransE (transe.cu): scorer, backward, self-adversarial forward, and ranking and top-k by L1 distance over all
// entities or over the first R relations.  Every argument is checked before any device work, with RotatE's rules.
// ------------------------------------------------------------------------------------------------
extern "C" int rgcn_transe_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                   const int32_t* X, int64_t N, const float* Y, float gamma, float* energies,
                                   float* loss_out, void* stream) {
  const int rc = rotate_checks("rgcn_transe_forward", codes && rel && loss_out && (N <= 0 || (X && energies)), V, Vrel,
                               d, N, gamma);
  if (rc) return rc;
  return launch_transe_forward(codes, rel, d, X, N, Y, gamma, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int rgcn_transe_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                    const int32_t* X, int64_t N, const float* Y, float gamma, const float* energies,
                                    float g_loss, float g_reg, const float* g_scale_dev, const float* g_energy,
                                    float* dcodes, float* drel, float* rel_slice_sumsq, void* stream) {
  const int rc = rotate_checks("rgcn_transe_backward",
                               codes && rel && dcodes && drel && (N <= 0 || X) && (!Y || energies), V, Vrel, d, N,
                               gamma);
  if (rc) return rc;
  return launch_transe_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev, g_energy, dcodes, drel,
                                rel_slice_sumsq, (cudaStream_t)stream);
}

extern "C" int rgcn_transe_self_adversarial_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                                    int32_t d, const int32_t* X, int64_t N, int32_t K, float alpha,
                                                    float gamma, float* energies, float* coef, float* loss_out,
                                                    void* workspace, int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_transe_self_adversarial_forward";
  if (!std::isfinite(gamma)) {
    rgcn_set_error(who + ": the margin gamma must be finite");
    return RGCN_ERR_INVALID;
  }
  const int rc = self_adversarial_checks(
      who, codes && rel && loss_out && workspace && (N <= 0 || (X && energies && coef)), V, Vrel, d, N, K, alpha,
      workspace_bytes);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* parts = ws.take<float>(2 * (N / ((int64_t)K + 1)));
  return launch_self_adversarial_forward(SELFADV_TRANSE, codes, rel, d, X, N, K, alpha, gamma, energies, coef,
                                         loss_out, parts, (cudaStream_t)stream);
}

// Rank workspace: [Q n*d | gold_D n | gold_col n | raw_cnt n | known_cnt n] (rgcn_rotate_rank's); top-k workspace:
// [Q n*d | cand n*ceil(C/128)*k (-D, id) pairs], C the candidate count (V or R).  No split: nothing to reuse.
static bool transe_sizes_ok(int32_t C, int32_t d, int64_t n, int64_t per_row) {
  return C > 0 && d > 0 && d % 4 == 0 && n >= 0 && (n == 0 || per_row <= ((int64_t)1 << 60) / n);
}

static int64_t transe_rank_bytes(const char* who, int32_t C, int32_t d, int64_t n) {
  if (!transe_sizes_ok(C, d, n, (int64_t)d * 4 + 16)) {
    rgcn_set_error(std::string(who) + ": bad arguments (need a candidate count > 0, d > 0, d % 4 == 0, n >= 0)");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * d * 4) + 4 * align_up(n * 4) + 256;
}

static int64_t transe_topk_bytes(const char* who, int32_t C, int32_t d, int64_t n, int32_t k) {
  if (k < 1 || k > 128 || !transe_sizes_ok(C, d, n, (int64_t)d * 4 + (int64_t)transe_topk_tiles(C) * k * 8)) {
    rgcn_set_error(std::string(who) + ": bad arguments (need a candidate count > 0, d > 0, d % 4 == 0, n >= 0, "
                   "1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  return align_up(n * d * 4) + align_up(n * transe_topk_tiles(C) * k * 8) + 256;
}

extern "C" int64_t rgcn_transe_rank_workspace_bytes(int32_t V, int32_t d, int64_t n) {
  return transe_rank_bytes("rgcn_transe_rank_workspace_bytes", V, d, n);
}

extern "C" int64_t rgcn_transe_topk_workspace_bytes(int32_t V, int32_t d, int64_t n, int32_t k) {
  return transe_topk_bytes("rgcn_transe_topk_workspace_bytes", V, d, n, k);
}

extern "C" int64_t rgcn_transe_relation_rank_workspace_bytes(int32_t R, int32_t d, int64_t n) {
  return transe_rank_bytes("rgcn_transe_relation_rank_workspace_bytes", R, d, n);
}

extern "C" int64_t rgcn_transe_relation_topk_workspace_bytes(int32_t R, int32_t d, int64_t n, int32_t k) {
  return transe_topk_bytes("rgcn_transe_relation_topk_workspace_bytes", R, d, n, k);
}

// The checks every TransE query entry point shares.  mode: 0 / 1 the entity side, TRANSE_RELATIONS relation queries
// against rel[0:C] (C = R, 1 <= R <= Vrel); out = raw_rank or ids (and energies, `out2`).
static int transe_query_checks(const std::string& who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                               int32_t C, int32_t d, const int32_t* X, int64_t n, int mode, const void* out,
                               const void* out2, const void* workspace) {
  if (!codes || !rel || !workspace || (n > 0 && (!X || !out || !out2))) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL || (mode != 0 && mode != 1 &&
                                                                                     mode != TRANSE_RELATIONS)) {
    rgcn_set_error(who + ": bad arguments (need V > 0, Vrel > 0, d % 4 == 0, 0 <= n < 2^31, side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  if (mode == TRANSE_RELATIONS && !relation_count_ok(who.c_str(), C, Vrel)) return RGCN_ERR_INVALID;
  return RGCN_OK;
}

static int transe_rank_body(const std::string& who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                            int32_t C, int32_t d, const int32_t* X, int64_t n, int mode, const uint32_t* known_mask,
                            int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                            cudaStream_t st) {
  int rc = transe_query_checks(who, codes, rel, V, Vrel, C, d, X, n, mode, raw_rank, raw_rank, workspace);
  if (rc) return rc;
  if (filtered_rank && !known_mask) {
    rgcn_set_error(who + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < transe_rank_bytes(who.c_str(), C, d, n)) {
    rgcn_set_error(who + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who.c_str());
  if (rc || n == 0) return rc;
  Carver ws(workspace, workspace_bytes);
  float* Q = ws.take<float>(n * d);
  float* gold_D = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (!rc) rc = launch_transe_prepare(codes, rel, d, X, n, mode, Q, gold_D, gold_col, st);
  if (!rc)
    rc = launch_transe_rank(Q, mode == TRANSE_RELATIONS ? rel : codes, C, d, n, gold_D, gold_col, known_mask, raw_cnt,
                            known_cnt, st);
  if (!rc) rc = launch_distmult_rank_finalize(raw_cnt, known_cnt, n, raw_rank, filtered_rank, st);
  return rc;
}

static int transe_topk_body(const std::string& who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                            int32_t C, int32_t d, const int32_t* X, int64_t n, int mode, int32_t k,
                            const uint32_t* exclude_mask, float gamma, int32_t* ids, float* energies, void* workspace,
                            int64_t workspace_bytes, cudaStream_t st) {
  int rc = transe_query_checks(who, codes, rel, V, Vrel, C, d, X, n, mode, ids, energies, workspace);
  if (rc) return rc;
  if (k < 1 || k > 128) {
    rgcn_set_error(who + ": k = " + std::to_string(k) + " is out of range (1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  if (!std::isfinite(gamma)) {
    rgcn_set_error(who + ": the margin gamma must be finite");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < transe_topk_bytes(who.c_str(), C, d, n, k)) {
    rgcn_set_error(who + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onen_device_checks(who.c_str());
  if (rc || n == 0) return rc;
  Carver ws(workspace, workspace_bytes);
  float* Q = ws.take<float>(n * d);
  uint2* cand = ws.take<uint2>(n * transe_topk_tiles(C) * k);
  rc = launch_transe_prepare(codes, rel, d, X, n, mode, Q, nullptr, nullptr, st);
  if (!rc)
    rc = launch_transe_topk(Q, mode == TRANSE_RELATIONS ? rel : codes, C, d, n, exclude_mask, k, gamma, cand, ids,
                            energies, st);
  return rc;
}

extern "C" int rgcn_transe_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                const int32_t* X, int64_t n, int side, const uint32_t* known_mask,
                                int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                                void* stream) {
  if (side != 0 && side != 1) side = -1;   // refused by the shared checks
  return transe_rank_body("rgcn_transe_rank", codes, rel, V, Vrel, V, d, X, n, side, known_mask, raw_rank,
                          filtered_rank, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_transe_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                                float gamma, int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes,
                                void* stream) {
  if (side != 0 && side != 1) side = -1;
  return transe_topk_body("rgcn_transe_topk", codes, rel, V, Vrel, V, d, X, n, side, k, exclude_mask, gamma, ids,
                          energies, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_transe_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                         int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                         int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  return transe_rank_body("rgcn_transe_relation_rank", codes, rel, V, Vrel, R, d, X, n, TRANSE_RELATIONS, known_mask,
                          raw_rank, filtered_rank, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_transe_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                         int32_t d, const int32_t* X, int64_t n, int32_t k,
                                         const uint32_t* exclude_mask, float gamma, int32_t* ids, float* energies,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
  return transe_topk_body("rgcn_transe_relation_topk", codes, rel, V, Vrel, R, d, X, n, TRANSE_RELATIONS, k,
                          exclude_mask, gamma, ids, energies, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// QuatE (quate.cu): scorer, backward, self-adversarial forward, and the DistMult scoring GEMMs behind QuatE's query
// rows: entity and relation ranks and top-k, 1-N training and the query rows of the score matrices.  Every argument is
// checked before any device work.
// ------------------------------------------------------------------------------------------------
static int quate_checks(const std::string& who, bool pointers_ok, int32_t V, int32_t Vrel, int32_t d, int64_t N) {
  if (!pointers_ok) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || N < 0) {
    rgcn_set_error(who + ": bad sizes (need V > 0, Vrel > 0, d > 0, d % 4 == 0, N >= 0)");
    return RGCN_ERR_INVALID;
  }
  return onen_device_checks(who.c_str());
}

extern "C" int rgcn_quate_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                  const int32_t* X, int64_t N, const float* Y, float* energies, float* loss_out,
                                  void* stream) {
  const int rc = quate_checks("rgcn_quate_forward", codes && rel && loss_out && (N <= 0 || (X && energies)), V, Vrel,
                              d, N);
  if (rc) return rc;
  return launch_quate_forward(codes, rel, d, X, N, Y, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int rgcn_quate_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                   const int32_t* X, int64_t N, const float* Y, const float* energies, float g_loss,
                                   float g_reg, const float* g_scale_dev, const float* g_energy, float* dcodes,
                                   float* drel, float* rel_slice_sumsq, void* stream) {
  const int rc = quate_checks("rgcn_quate_backward",
                              codes && rel && dcodes && drel && (N <= 0 || X) && (!Y || energies), V, Vrel, d, N);
  if (rc) return rc;
  return launch_quate_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev, g_energy, dcodes, drel,
                               rel_slice_sumsq, (cudaStream_t)stream);
}

extern "C" int rgcn_quate_self_adversarial_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                                   int32_t d, const int32_t* X, int64_t N, int32_t K, float alpha,
                                                   float* energies, float* coef, float* loss_out, void* workspace,
                                                   int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_quate_self_adversarial_forward";
  const int rc = self_adversarial_checks(
      who, codes && rel && loss_out && workspace && (N <= 0 || (X && energies && coef)), V, Vrel, d, N, K, alpha,
      workspace_bytes);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* parts = ws.take<float>(2 * (N / ((int64_t)K + 1)));
  return launch_self_adversarial_forward(SELFADV_QUATE, codes, rel, d, X, N, K, alpha, 0.f, energies, coef, loss_out,
                                         parts, (cudaStream_t)stream);
}

// Entity queries: rank_with_queries / topk_with_queries with QuatE's query rows, in the DistMult workspaces
// (distmult_rank_workspace_bytes, rgcn_topk_workspace_bytes), whose split of the codes is reused alike.
extern "C" int rgcn_quate_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                               const int32_t* X, int64_t n, int side, const uint32_t* known_mask, int reuse_split,
                               int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                               void* stream) {
  return rank_with_queries("rgcn_quate_rank", launch_quate_rank_prepare, codes, V, distmult_rank_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, known_mask, reuse_split, raw_rank, filtered_rank, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_quate_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                               const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                               int reuse_split, int32_t* ids, float* energies, void* workspace,
                               int64_t workspace_bytes, void* stream) {
  return topk_with_queries("rgcn_quate_topk", launch_quate_rank_prepare, codes, V, rgcn_topk_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, k, exclude_mask, reuse_split, ids, energies, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

// Relation queries: workspace [rh R*d | the workspace of rank_with_queries / topk_with_queries over rh].  Without
// reuse_split, rel[0:R] is normalised into rh and rh is split; with it, both are those of the previous call on the
// same workspace.
extern "C" int64_t rgcn_quate_relation_rank_workspace_bytes(int32_t R, int32_t d, int64_t n) {
  const int64_t rest = rgcn_relation_rank_workspace_bytes(R, d, n);
  return rest < 0 ? rest : align_up((int64_t)R * d * 4) + rest;
}

extern "C" int64_t rgcn_quate_relation_topk_workspace_bytes(int32_t R, int32_t d, int64_t n, int32_t k) {
  const int64_t rest = rgcn_relation_topk_workspace_bytes(R, d, n, k);
  return rest < 0 ? rest : align_up((int64_t)R * d * 4) + rest;
}

// The checks of the two relation entry points that must come before the normalisation; rank_with_queries /
// topk_with_queries then check the rest (all of them before their own device work).
static int quate_relation_checks(const char* who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                 int32_t R, int32_t d, const int32_t* X, int64_t n, const void* out, const void* out2,
                                 const void* workspace, int64_t need, int64_t workspace_bytes) {
  if (!codes || !rel || !workspace || (n > 0 && (!X || !out || !out2))) {
    rgcn_set_error(std::string(who) + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 || n < 0 || n > 0x7fffffffLL) {
    rgcn_set_error(std::string(who) + ": bad arguments (need V > 0, Vrel > 0, d % 4 == 0, 0 <= n < 2^31)");
    return RGCN_ERR_INVALID;
  }
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  return RGCN_OK;
}

static int quate_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int,
                                  float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  return launch_quate_relation_prepare(codes, rel, d, X, n, Q, gold_sig, gold_col, st);
}

extern "C" int rgcn_quate_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                        int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                        int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_quate_relation_rank";
  int rc = quate_relation_checks(who, codes, rel, V, Vrel, R, d, X, n, raw_rank, raw_rank, workspace,
                                 rgcn_quate_relation_rank_workspace_bytes(R, d, n), workspace_bytes);
  if (rc) return rc;
  if (filtered_rank && !known_mask) {
    rgcn_set_error(std::string(who) + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  Carver ws(workspace, workspace_bytes);
  float* rh = ws.take<float>((int64_t)R * d);
  if (!reuse_split) rc = launch_quate_normalize(rel, R, d, rh, st);
  if (rc) return rc;
  return rank_with_queries(who, quate_relation_prepare, rh, R, rgcn_relation_rank_workspace_bytes, codes, rel, V, Vrel,
                           d, X, n, 0, known_mask, reuse_split, raw_rank, filtered_rank, ws.base + ws.off,
                           workspace_bytes - ws.off, st);
}

extern "C" int rgcn_quate_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                        int32_t d, const int32_t* X, int64_t n, int32_t k,
                                        const uint32_t* exclude_mask, int reuse_split, int32_t* ids, float* energies,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_quate_relation_topk";
  if (k < 1 || k > 128) {
    rgcn_set_error(std::string(who) + ": k = " + std::to_string(k) + " is out of range (1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  int rc = quate_relation_checks(who, codes, rel, V, Vrel, R, d, X, n, ids, energies, workspace,
                                 rgcn_quate_relation_topk_workspace_bytes(R, d, n, k), workspace_bytes);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Carver ws(workspace, workspace_bytes);
  float* rh = ws.take<float>((int64_t)R * d);
  if (!reuse_split) rc = launch_quate_normalize(rel, R, d, rh, st);
  if (rc) return rc;
  return topk_with_queries(who, quate_relation_prepare, rh, R, rgcn_relation_topk_workspace_bytes, codes, rel, V, Vrel,
                           d, X, n, 0, k, exclude_mask, reuse_split, ids, energies, ws.base + ws.off,
                           workspace_bytes - ws.off, st);
}

// 1-N training: the one_to_n() body with QuatE's query rows and query backward, one launch per side run in a chunk.
// The workspace is rgcn_one_to_n_workspace_bytes, and the backward of a call made with g_scale = (1, 0) is
// rgcn_one_to_n_finish: the L2 term is DistMult's.
extern "C" int rgcn_quate_one_to_n(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                                   const int32_t* queries, int64_t n, const uint32_t* labels, float smoothing,
                                   const float* g_scale, float* loss, float* dcodes, float* drel, int64_t chunk,
                                   void* workspace, int64_t workspace_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const OnenStep prepare = [=](const OnenChunk& k, float* Q) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (!rc && b < e)
        rc = launch_quate_rank_prepare(codes, rel, d, k.X + 3 * b, e - b, run.side, Q + (b - k.c0) * d, nullptr,
                                       nullptr, st);
    }
    return rc;
  };
  const OnenStep query_bwd = [=](const OnenChunk& k, float* dQ) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (!rc && b < e)
        rc = launch_quate_query_bwd(codes, rel, d, k.X + 3 * b, e - b, run.side, dQ + (b - k.c0) * d, g_scale,
                                    k.c_reg, dcodes, drel, st);
    }
    return rc;
  };
  return one_to_n("rgcn_quate_one_to_n", prepare, query_bwd, false, codes, rel, V, Vrel, R, d, queries, n, labels,
                  smoothing, g_scale, loss, dcodes, drel, chunk, workspace, workspace_bytes, st);
}

// The query rows Q [n, d] of the triples X for one side (the rows the entity ranks score), for the [n, V] score
// matrices.
extern "C" int rgcn_quate_query_rows(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                     const int32_t* X, int64_t n, int side, float* Q, void* stream) {
  const std::string who = "rgcn_quate_query_rows";
  if (side != 0 && side != 1) {
    rgcn_set_error(who + ": bad arguments (side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  const int rc = quate_checks(who, codes && rel && (n <= 0 || (X && Q)), V, Vrel, d, n);
  if (rc) return rc;
  return launch_quate_rank_prepare(codes, rel, d, X, n, side, Q, nullptr, nullptr, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// HolE (hole.cu): the real Fourier basis and its transforms, and the QuatE-shaped surface over transformed tables:
// scorer, backward, self-adversarial forward, and the DistMult scoring GEMMs behind HolE's query rows (entity and
// relation ranks and top-k, 1-N training, the query rows of the score matrices).  Every argument is checked before any
// device work.
// ------------------------------------------------------------------------------------------------
extern "C" int64_t rgcn_hole_transform_workspace_bytes(int32_t d) {
  if (d <= 0 || d % 4 != 0) {
    rgcn_set_error("rgcn_hole_transform_workspace_bytes: bad arguments (need d > 0, d % 4 == 0)");
    return RGCN_ERR_INVALID;
  }
  return align_up(2 * (int64_t)d * d * 4);   // the hi / lo split of U (gemm_any)
}

// out = x U (inverse = 0) or x U^T (inverse = 1), one 3xTF32 GEMM; U is built into `basis` first unless basis_ready.
extern "C" int rgcn_hole_transform(const float* x, int64_t rows, int32_t d, int inverse, float* basis, int basis_ready,
                                   float* out, void* workspace, int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_hole_transform";
  if (!basis || !workspace || (rows > 0 && (!x || !out))) {
    rgcn_set_error(who + ": null pointer");
    return RGCN_ERR_INVALID;
  }
  if (d <= 0 || d % 4 != 0 || rows < 0 || rows > 0x7fffffffLL || (inverse != 0 && inverse != 1) ||
      (rows > 0 && x == out)) {
    rgcn_set_error(who + ": bad arguments (need d > 0, d % 4 == 0, 0 <= rows < 2^31, inverse in {0,1}, out != x)");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_hole_transform_workspace_bytes(d)) {
    rgcn_set_error(who + ": workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  int rc = onen_device_checks(who.c_str());
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (!basis_ready) rc = launch_hole_basis(d, basis, st);
  if (rc) return rc;
  return gemm_any(st, (float*)workspace, false, inverse != 0, rows, d, d, x, d, basis, d, 0.f, out, d);
}

extern "C" int rgcn_hole_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                 const int32_t* X, int64_t N, const float* Y, float* energies, float* loss_out,
                                 void* stream) {
  const int rc = quate_checks("rgcn_hole_forward", codes && rel && loss_out && (N <= 0 || (X && energies)), V, Vrel,
                              d, N);
  if (rc) return rc;
  return launch_hole_forward(codes, rel, d, X, N, Y, energies, loss_out, (cudaStream_t)stream);
}

extern "C" int rgcn_hole_backward(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                  const int32_t* X, int64_t N, const float* Y, const float* energies, float g_loss,
                                  float g_reg, const float* g_scale_dev, const float* g_energy, float* dcodes,
                                  float* drel, float* rel_slice_sumsq, void* stream) {
  const int rc = quate_checks("rgcn_hole_backward",
                              codes && rel && dcodes && drel && (N <= 0 || X) && (!Y || energies), V, Vrel, d, N);
  if (rc) return rc;
  return launch_hole_backward(codes, rel, d, X, N, Y, energies, g_loss, g_reg, g_scale_dev, g_energy, dcodes, drel,
                              rel_slice_sumsq, (cudaStream_t)stream);
}

extern "C" int rgcn_hole_self_adversarial_forward(const float* codes, const float* rel, int32_t V, int32_t Vrel,
                                                  int32_t d, const int32_t* X, int64_t N, int32_t K, float alpha,
                                                  float* energies, float* coef, float* loss_out, void* workspace,
                                                  int64_t workspace_bytes, void* stream) {
  const std::string who = "rgcn_hole_self_adversarial_forward";
  const int rc = self_adversarial_checks(
      who, codes && rel && loss_out && workspace && (N <= 0 || (X && energies && coef)), V, Vrel, d, N, K, alpha,
      workspace_bytes);
  if (rc) return rc;
  Carver ws(workspace, workspace_bytes);
  float* parts = ws.take<float>(2 * (N / ((int64_t)K + 1)));
  return launch_self_adversarial_forward(SELFADV_HOLE, codes, rel, d, X, N, K, alpha, 0.f, energies, coef, loss_out,
                                         parts, (cudaStream_t)stream);
}

// Entity queries: rank_with_queries / topk_with_queries with HolE's query rows, in the DistMult workspaces
// (distmult_rank_workspace_bytes, rgcn_topk_workspace_bytes), whose split of the codes is reused alike.
extern "C" int rgcn_hole_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                              const int32_t* X, int64_t n, int side, const uint32_t* known_mask, int reuse_split,
                              int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                              void* stream) {
  return rank_with_queries("rgcn_hole_rank", launch_hole_rank_prepare, codes, V, distmult_rank_workspace_bytes, codes,
                           rel, V, Vrel, d, X, n, side, known_mask, reuse_split, raw_rank, filtered_rank, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_hole_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                              const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                              int reuse_split, int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes,
                              void* stream) {
  return topk_with_queries("rgcn_hole_topk", launch_hole_rank_prepare, codes, V, rgcn_topk_workspace_bytes, codes, rel,
                           V, Vrel, d, X, n, side, k, exclude_mask, reuse_split, ids, energies, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

// Relation queries: the candidates are the transformed rel[0:R] themselves, so these are distmult_relation_rank /
// _topk with HolE's pair query rows, in the same workspaces (rgcn_relation_rank_workspace_bytes,
// rgcn_relation_topk_workspace_bytes).
static int hole_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int,
                                 float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  return launch_hole_relation_prepare(codes, rel, d, X, n, Q, gold_sig, gold_col, st);
}

extern "C" int rgcn_hole_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                       int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                       int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                       int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_hole_relation_rank";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return rank_with_queries(who, hole_relation_prepare, rel, R, rgcn_relation_rank_workspace_bytes, codes, rel, V, Vrel,
                           d, X, n, 0, known_mask, reuse_split, raw_rank, filtered_rank, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

extern "C" int rgcn_hole_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                       int32_t d, const int32_t* X, int64_t n, int32_t k, const uint32_t* exclude_mask,
                                       int reuse_split, int32_t* ids, float* energies, void* workspace,
                                       int64_t workspace_bytes, void* stream) {
  const char* who = "rgcn_hole_relation_topk";
  if (!relation_count_ok(who, R, Vrel)) return RGCN_ERR_INVALID;
  return topk_with_queries(who, hole_relation_prepare, rel, R, rgcn_relation_topk_workspace_bytes, codes, rel, V, Vrel,
                           d, X, n, 0, k, exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

// 1-N training: the one_to_n() body with HolE's query rows and query backward, one launch per side run in a chunk.
// The workspace is rgcn_one_to_n_workspace_bytes, and the backward of a call made with g_scale = (1, 0) is
// rgcn_one_to_n_finish: the L2 term is DistMult's.
extern "C" int rgcn_hole_one_to_n(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R, int32_t d,
                                  const int32_t* queries, int64_t n, const uint32_t* labels, float smoothing,
                                  const float* g_scale, float* loss, float* dcodes, float* drel, int64_t chunk,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const OnenStep prepare = [=](const OnenChunk& k, float* Q) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (!rc && b < e)
        rc = launch_hole_rank_prepare(codes, rel, d, k.X + 3 * b, e - b, run.side, Q + (b - k.c0) * d, nullptr,
                                      nullptr, st);
    }
    return rc;
  };
  const OnenStep query_bwd = [=](const OnenChunk& k, float* dQ) {
    int rc = RGCN_OK;
    for (const OnenRun& run : *k.runs) {
      const int64_t b = std::max(run.begin, k.c0), e = std::min(run.end, k.c1);
      if (!rc && b < e)
        rc = launch_hole_query_bwd(codes, rel, d, k.X + 3 * b, e - b, run.side, dQ + (b - k.c0) * d, g_scale,
                                   k.c_reg, dcodes, drel, st);
    }
    return rc;
  };
  return one_to_n("rgcn_hole_one_to_n", prepare, query_bwd, false, codes, rel, V, Vrel, R, d, queries, n, labels,
                  smoothing, g_scale, loss, dcodes, drel, chunk, workspace, workspace_bytes, st);
}

// The query rows Q [n, d] of the triples X for one side (the rows the entity ranks score), for the [n, V] score
// matrices.
extern "C" int rgcn_hole_query_rows(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                    const int32_t* X, int64_t n, int side, float* Q, void* stream) {
  const std::string who = "rgcn_hole_query_rows";
  if (side != 0 && side != 1) {
    rgcn_set_error(who + ": bad arguments (side in {0,1})");
    return RGCN_ERR_INVALID;
  }
  const int rc = quate_checks(who, codes && rel && (n <= 0 || (X && Q)), V, Vrel, d, n);
  if (rc) return rc;
  return launch_hole_rank_prepare(codes, rel, d, X, n, side, Q, nullptr, nullptr, (cudaStream_t)stream);
}
