// api.cu -- C-ABI entry points of librgcn_b200.so (see include/rgcn_b200.h).
// Orchestrates per-layer work on ONE stream: weight re-layout -> dense self-loop GEMM (own wgmma 3xTF32
// kernel, gemm_tf32x3.cu) -> warp-centric aggregation kernels.  No vendor-library compute anywhere.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>

#include "kernels.cuh"

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

int common_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
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

int layer_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
  int rc = common_checks(g, d, B, who);
  if (rc) return rc;
  if (g->V_src < g->V_dst) {  // the self-loop term reads H rows [0, V_dst)
    rgcn_set_error(std::string(who) + ": layer entry points need V_src >= V_dst (messages-only graphs go through rgcn_block_aggregate)");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
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

// 3 = weight-id-major with TMA-staged gathers (block_staged.cu) where the block size supports it
static bool use_staged(int d, int s) {
  int algo = g_block_algo;
  if (const char* e = std::getenv("RGCN_BLOCK_ALGO")) algo = std::atoi(e);
  return (algo == 3 || algo == -1) && block_stg_supported(d, s);
}

static int launch_block_relmajor(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                                 const float* r_norm, const float* X, int ldx, int d, int s, const float* Wt,
                                 float* out, const float* Hrow, int ldh, float* dWt, cudaStream_t st) {
  if (use_staged(d, s))
    return launch_block_stg(items, n_items, r_row, r_nbr, r_norm, X, ldx, d, s, Wt, out, Hrow, ldh, dWt, st);
  return launch_block_rel(items, n_items, r_row, r_nbr, r_norm, X, ldx, d, s, Wt, out, Hrow, ldh, dWt, st);
}

static bool use_rel_major(int d, int s) {
  int algo = g_block_algo;
  if (const char* e = std::getenv("RGCN_BLOCK_ALGO")) algo = std::atoi(e);
  if (algo == 0) return false;
  return block_rel_supported(d, s);
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
  int rc = layer_checks(g, d, B, "rgcn_block_forward");
  if (rc) return rc;
  if (d % B != 0) {
    rgcn_set_error("rgcn_block_forward: d must be a multiple of B (gcn_basis_concat.py:15)");
    return RGCN_ERR_INVALID;
  }
  if (!H || !Wf || !Wb || !Wself || !out || !workspace || keep <= 0.f) {
    rgcn_set_error("rgcn_block_forward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_block_workspace_bytes(g, d, B, 0)) {
    rgcn_set_error("rgcn_block_forward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  {
    const bool relm = use_rel_major(d, s);
    rc = need_views(g, !relm, relm, "rgcn_block_forward");
    if (rc) return rc;
  }
  const int slabs = slabs_for(d);
  const int64_t n_split = g->by_dst.n_split;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* Wt = ws.take<float>((int64_t)g->n_relw * s * d);
  float* scratch = ws.take<float>(n_split * d);
  int* counters = ws.take<int>(n_split * slabs);

  MARK("start");
  rc = launch_block_relayout(Wf, Wb, R, B, s, /*transpose=*/0, Wt, st);
  if (rc) return rc;
  MARK("block_relayout");
  if (n_split > 0) {
    rc = rgcn_check_cuda(
        cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
        "memset(scratch)");
    if (rc) return rc;
  }
  // self-loop term S = H[0:V_dst] @ W_self written straight into `out` (gcn_basis_concat.py:65-66)
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, d, H, d, Wself, d, 0.f, out, d);
  if (rc) return rc;
  MARK("gemm_self_loop");
  if (use_rel_major(d, s)) {
    // out = dropout(S);  out[dst] += W_r . sum(norm x)  (L2 vector reductions);  out = relu(out)
    rc = launch_mask_relu(out, drop_mask, 1.0f / keep, 0, (int64_t)g->V_dst * d, st);
    if (rc) return rc;
    rc = launch_block_relmajor(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row,
                          g->by_rel.d_nbr, g->by_rel.d_norm, H, d, d, s, Wt, out, nullptr, 0, nullptr,
                          st);
    if (rc) return rc;
    MARK("block_agg_fwd");
    rc = launch_mask_relu(out, nullptr, 1.f, relu, (int64_t)g->V_dst * d, st);
    MARK("relu_epilogue");
    return rc;
  }
  AggLaunch a = make_agg(g->by_dst, H, d, d, scratch, counters);
  rc = launch_block_agg(a, s, Wt, out, drop_mask, 1.0f / keep, relu, st);
  MARK("block_agg_fwd");
  return rc;
}

extern "C" int rgcn_block_backward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                   const float* Wf, const float* Wb, const float* Wself,
                                   const uint8_t* drop_mask, float keep, int relu, const float* out,
                                   const float* dOut, float* dH, float* dWf, float* dWb,
                                   float* dWself, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  int rc = layer_checks(g, d, B, "rgcn_block_backward");
  if (rc) return rc;
  if (d % B != 0) {
    rgcn_set_error("rgcn_block_backward: d must be a multiple of B");
    return RGCN_ERR_INVALID;
  }
  if (!H || !Wf || !Wb || !Wself || !dOut || !dH || !dWf || !dWb || !dWself || !workspace ||
      (relu && !out) || keep <= 0.f) {
    rgcn_set_error("rgcn_block_backward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_block_workspace_bytes(g, d, B, 1)) {
    rgcn_set_error("rgcn_block_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  {
    const bool relm = use_rel_major(d, s);
    rc = need_views(g, !relm, true, "rgcn_block_backward");
    if (rc) return rc;
  }
  const int slabs = slabs_for(d);
  const int64_t n_split = g->by_src.n_split;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* Wtt = ws.take<float>(wt);
  float* dWt = ws.take<float>(wt);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);
  float* scratch = ws.take<float>(n_split * d);
  int* counters = ws.take<int>(n_split * slabs);
  if (!drop_mask) dS = G;

  // G = dOut * relu'(out);  dS = G * mask / keep   (message_gcn.py:64 dropout is on the self loop only)
  MARK("start");
  if (!relu && !drop_mask) {
    // nothing to apply (the node-sharded layers pass the already masked gradient): read dOut in place instead of
    // copying it into the workspace (20 GB read + 20 GB written at the full benchmark size)
    G = dS = const_cast<float*>(dOut);
  } else {
    rc = launch_grad_prologue(dOut, out, drop_mask, 1.0f / keep, relu, (int64_t)g->V_dst * d, G, dS, st);
    if (rc) return rc;
  }
  MARK("grad_prologue");
  // dW_self = H[0:V_dst]^T dS
  rc = gemm_any(st, split_ws, true, false, d, d, g->V_dst, H, d, dS, d, 0.f, dWself, d);
  if (rc) return rc;
  MARK("gemm_dWself");
  // dH[0:V_dst] = dS W_self^T ; halo rows start at zero
  rc = gemm_any(st, split_ws, false, true, g->V_dst, d, d, dS, d, Wself, d, 0.f, dH, d);
  if (rc) return rc;
  if (g->V_src > g->V_dst) {
    rc = rgcn_check_cuda(cudaMemsetAsync(dH + (size_t)g->V_dst * d, 0,
                                         (size_t)(g->V_src - g->V_dst) * d * sizeof(float), st),
                         "memset(dH halo)");
    if (rc) return rc;
  }
  MARK("gemm_dH_self");
  // dH[u] += sum_{m: src_m = u} norm_m W[relw_m]^T G[dst_m]   (same kernel, transposed table)
  rc = launch_block_relayout(Wf, Wb, R, B, s, /*transpose=*/1, Wtt, st);
  if (rc) return rc;
  MARK("block_relayout_T");
  if (n_split > 0) {
    rc = rgcn_check_cuda(
        cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
        "memset(scratch)");
    if (rc) return rc;
  }
  // dW accumulates in the j-major layout (zeroed first); when the block size allows, the dH pass
  // produces it in the same walk (one round of gathers for the whole backward of the messages)
  rc = rgcn_check_cuda(cudaMemsetAsync(dWt, 0, wt * sizeof(float), st), "memset(dWt)");
  if (rc) return rc;
  const bool rel = use_rel_major(d, s);
  const bool fused = rel && block_rel_fuse_dw_supported(d, s) && !std::getenv("RGCN_NO_FUSE_DW");
  if (rel) {
    rc = launch_block_relmajor(g->by_rel_src.d_items, (int)g->by_rel_src.n_items, g->by_rel_src.d_row,
                          g->by_rel_src.d_nbr, g->by_rel_src.d_norm, G, d, d, s, Wtt, dH,
                          fused ? H : nullptr, d, fused ? dWt : nullptr, st);
  } else {
    AggLaunch a = make_agg(g->by_src, G, d, d, scratch, counters);
    rc = launch_block_agg(a, s, Wtt, dH, nullptr, 1.f, 0, st);
  }
  if (rc) return rc;
  MARK("block_agg_dH");
  // dW[w] = sum_{m: relw_m = w} norm_m G[dst_m] (x)_block H[src_m]
  if (!fused) {
    rc = launch_block_dw(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row,
                         g->by_rel.d_nbr, g->by_rel.d_norm, H, d, G, d, d, s, dWt, st);
    if (rc) return rc;
  }
  MARK("block_dW");
  rc = launch_block_unlayout(dWt, R, B, s, dWf, dWb, 0, fused ? 1 : 0, st);
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
  int rc = common_checks(g, d, B, "rgcn_block_aggregate");
  if (rc) return rc;
  if (d % B != 0 || !X || !Wf || !Wb || !out || !workspace) {
    rgcn_set_error("rgcn_block_aggregate: bad arguments");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_block_aggregate_workspace_bytes(g, d, B, 0)) {
    rgcn_set_error("rgcn_block_aggregate: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  {
    const bool relm = use_rel_major(d, s);
    rc = need_views(g, !relm, relm, "rgcn_block_aggregate");
    if (rc) return rc;
  }
  const int slabs = slabs_for(d);
  const int64_t n_split = g->by_dst.n_split;
  Carver ws(workspace, workspace_bytes);
  float* Wt = ws.take<float>((int64_t)g->n_relw * s * d);
  float* scratch = ws.take<float>(n_split * d);
  int* counters = ws.take<int>(n_split * slabs);
  MARK("start");
  rc = launch_block_relayout(Wf, Wb, R, B, s, 0, Wt, st);
  if (rc) return rc;
  if (use_rel_major(d, s)) {
    rc = launch_block_relmajor(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row, g->by_rel.d_nbr,
                          g->by_rel.d_norm, X, d, d, s, Wt, out, nullptr, 0, nullptr, st);
  } else {
    if (n_split > 0) {
      rc = rgcn_check_cuda(
          cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
          "memset(scratch)");
      if (rc) return rc;
    }
    AggLaunch a = make_agg(g->by_dst, X, d, d, scratch, counters);
    rc = launch_block_agg(a, s, Wt, out, nullptr, 1.f, 0, st);  // out = out + sum (in-place epilogue)
  }
  MARK("block_aggregate");
  return rc;
}

extern "C" int rgcn_block_aggregate_backward(const rgcn_graph_t* g, int32_t d, int32_t B,
                                             const float* X, const float* Wf, const float* Wb,
                                             const float* G, float* dX, float* dWf, float* dWb,
                                             int accumulate_dW, void* workspace,
                                             int64_t workspace_bytes, void* stream) {
  int rc = common_checks(g, d, B, "rgcn_block_aggregate_backward");
  if (rc) return rc;
  if (d % B != 0 || !X || !Wf || !Wb || !G || !dX || !dWf || !dWb || !workspace) {
    rgcn_set_error("rgcn_block_aggregate_backward: bad arguments");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_block_aggregate_workspace_bytes(g, d, B, 1)) {
    rgcn_set_error("rgcn_block_aggregate_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int s = d / B, R = g->n_relw / 2;
  {
    const bool relm = use_rel_major(d, s);
    rc = need_views(g, !relm, true, "rgcn_block_aggregate_backward");
    if (rc) return rc;
  }
  const int slabs = slabs_for(d);
  const int64_t n_split = g->by_src.n_split;
  const int64_t wt = (int64_t)g->n_relw * s * d;
  Carver ws(workspace, workspace_bytes);
  float* Wtt = ws.take<float>(wt);
  float* dWt = ws.take<float>(wt);
  float* scratch = ws.take<float>(n_split * d);
  int* counters = ws.take<int>(n_split * slabs);
  MARK("start");
  rc = launch_block_relayout(Wf, Wb, R, B, s, 1, Wtt, st);
  if (rc) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(dX, 0, (size_t)g->V_src * d * sizeof(float), st), "memset(dX)");
  if (rc) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(dWt, 0, wt * sizeof(float), st), "memset(dWt)");
  if (rc) return rc;
  const bool rel = use_rel_major(d, s);
  const bool fused = rel && block_rel_fuse_dw_supported(d, s) && !std::getenv("RGCN_NO_FUSE_DW");
  if (rel) {
    rc = launch_block_relmajor(g->by_rel_src.d_items, (int)g->by_rel_src.n_items, g->by_rel_src.d_row,
                          g->by_rel_src.d_nbr, g->by_rel_src.d_norm, G, d, d, s, Wtt, dX,
                          fused ? X : nullptr, d, fused ? dWt : nullptr, st);
  } else {
    if (n_split > 0) {
      rc = rgcn_check_cuda(
          cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
          "memset(scratch)");
      if (rc) return rc;
    }
    AggLaunch a = make_agg(g->by_src, G, d, d, scratch, counters);
    rc = launch_block_agg(a, s, Wtt, dX, nullptr, 1.f, 0, st);
  }
  if (rc) return rc;
  if (!fused) {
    rc = launch_block_dw(g->by_rel.d_items, (int)g->by_rel.n_items, g->by_rel.d_row, g->by_rel.d_nbr,
                         g->by_rel.d_norm, X, d, G, d, d, s, dWt, st);
    if (rc) return rc;
  }
  MARK("block_aggregate_bwd");
  return launch_block_unlayout(dWt, R, B, s, dWf, dWb, accumulate_dW, fused ? 1 : 0, st);
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
  int rc = layer_checks(g, d, B, "rgcn_basis_forward");
  if (rc) return rc;
  rc = need_views(g, true, false, "rgcn_basis_forward");
  if (rc) return rc;
  if (!H || !Vf || !Vb || !Cf || !Cb || !Wself || !out || !saved || !workspace || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_forward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_workspace_bytes(g, d, B, 0)) {
    rgcn_set_error("rgcn_basis_forward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t dB = (int64_t)d * B;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  float* split_ws = ws.take<float>((int64_t)2 * d * d * B);
  rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat, Cf, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cf");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat + (size_t)R * B, Cb, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cb");
  if (rc) return rc;
  MARK("start");
  // Agg[v][dir][k*B+b] = sum_m norm_m C[relw_m,b] H[src_m,k]
  rc = launch_zero_rows(saved, 2 * dB, g->by_dst.d_split_rows, (int)g->by_dst.n_split, st);
  if (rc) return rc;
  AggLaunch a = make_agg(g->by_dst, H, d, d, nullptr, nullptr);
  rc = launch_basis_agg(a, Ccat, B, g->n_relw, /*layout=*/0, saved, st);
  if (rc) return rc;
  MARK("basis_agg_fwd");
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, d, H, d, Wself, d, 0.f, out, d);
  if (rc) return rc;
  rc = launch_mask_relu(out, drop_mask, 1.0f / keep, 0, (int64_t)g->V_dst * d, st);
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
  int rc = layer_checks(g, d, B, "rgcn_basis_backward");
  if (rc) return rc;
  rc = need_views(g, true, false, "rgcn_basis_backward");
  if (rc) return rc;
  if (!H || !Vf || !Vb || !Cf || !Cb || !Wself || !saved || !dOut || !dH || !dVf || !dVb || !dCf ||
      !dCb || !dWself || !workspace || (relu && !out) || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_backward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_workspace_bytes(g, d, B, 1)) {
    rgcn_set_error("rgcn_basis_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
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
  if (!drop_mask) dS = G;
  rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat, Cf, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cf");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat + (size_t)R * B, Cb, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cb");
  if (rc) return rc;

  MARK("start");
  rc = launch_grad_prologue(dOut, out, drop_mask, 1.0f / keep, relu, (int64_t)g->V_dst * d, G, dS, st);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, true, false, d, d, g->V_dst, H, d, dS, d, 0.f, dWself, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, true, g->V_dst, d, d, dS, d, Wself, d, 0.f, dH, d);
  if (rc) return rc;
  if (g->V_src > g->V_dst) {
    rc = rgcn_check_cuda(cudaMemsetAsync(dH + (size_t)g->V_dst * d, 0,
                                         (size_t)(g->V_src - g->V_dst) * d * sizeof(float), st),
                         "memset(dH halo)");
    if (rc) return rc;
  }
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
  rc = rgcn_check_cuda(cudaMemcpyAsync(dCf, dCcat, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy dCf");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(dCb, dCcat + (size_t)R * B, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy dCb");
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

// argument validation runs before anything touches the device: bad shapes, null pointers and short workspaces are
// RGCN_ERR_INVALID / RGCN_ERR_WORKSPACE even for a host-only graph
static int onehot_shape_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
  if (!g || d <= 0 || d % 4 != 0 || B <= 0) {
    rgcn_set_error(std::string(who) + ": need a graph, d > 0, d % 4 == 0, B > 0");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}

static int onehot_graph_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
  int rc = layer_checks(g, d, B, who);
  if (rc) return rc;
  return need_views(g, true, false, who);
}

static int concat_coefficients(const float* Cf, const float* Cb, int R, int B, float* Ccat, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat, Cf, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cf");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(Ccat + (size_t)R * B, Cb, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy Cb");
  return rc;
}

extern "C" int rgcn_basis_onehot_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* Wf,
                                         const float* Wb, const float* Cf, const float* Cb, const float* Wself,
                                         const uint8_t* drop_mask, float keep, int relu, float* out, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  int rc = onehot_shape_checks(g, d, B, "rgcn_basis_onehot_forward");
  if (rc) return rc;
  if (!Wf || !Wb || !Cf || !Cb || !Wself || !out || !workspace || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_onehot_forward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_onehot_workspace_bytes(g, d, B, 0)) {
    rgcn_set_error("rgcn_basis_onehot_forward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onehot_graph_checks(g, d, B, "rgcn_basis_onehot_forward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  const int64_t n = (int64_t)g->V_dst * d;
  Carver ws(workspace, workspace_bytes);
  float* Ccat = ws.take<float>((int64_t)g->n_relw * B);
  rc = concat_coefficients(Cf, Cb, R, B, Ccat, st);
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
  int rc = onehot_shape_checks(g, d, B, "rgcn_basis_onehot_backward");
  if (rc) return rc;
  if (!Wf || !Wb || !Cf || !Cb || !dOut || !dWf || !dWb || !dCf || !dCb || !dWself || !workspace ||
      (relu && !out) || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_onehot_backward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_onehot_workspace_bytes(g, d, B, 1)) {
    rgcn_set_error("rgcn_basis_onehot_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = onehot_graph_checks(g, d, B, "rgcn_basis_onehot_backward");
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
  rc = concat_coefficients(Cf, Cb, R, B, Ccat, st);
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
  rc = rgcn_check_cuda(cudaMemcpyAsync(dCf, dCcat, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy dCf");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(dCb, dCcat + (size_t)R * B, (size_t)R * B * 4, cudaMemcpyDeviceToDevice, st), "copy dCb");
  return rc;
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

// shape, pointer and workspace checks first, then the graph (device, views) -- nothing touches the device before
static int diagcoef_graph_checks(const rgcn_graph_t* g, int32_t d, int32_t B, const char* who) {
  int rc = layer_checks(g, d, B, who);
  if (rc) return rc;
  return need_views(g, true, true, who);
}

extern "C" int rgcn_basis_diagcoef_forward(const rgcn_graph_t* g, int32_t d, int32_t B, const float* H,
                                           const float* Vf, const float* Vb, const float* Cf, const float* Cb,
                                           const float* Wself, const float* b, const uint8_t* drop_mask, float keep,
                                           int relu, float* out, float* saved, void* workspace,
                                           int64_t workspace_bytes, void* stream) {
  int rc = onehot_shape_checks(g, d, B, "rgcn_basis_diagcoef_forward");
  if (rc) return rc;
  if (!H || !Vf || !Vb || !Cf || !Cb || !Wself || !b || !out || !saved || !workspace || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_diagcoef_forward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_diagcoef_workspace_bytes(g, d, B, 0)) {
    rgcn_set_error("rgcn_basis_diagcoef_forward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = diagcoef_graph_checks(g, d, B, "rgcn_basis_diagcoef_forward");
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
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, d, H, d, Wself, d, 0.f, out, d);
  if (!rc) rc = launch_mask_relu(out, drop_mask, 1.0f / keep, 0, (int64_t)g->V_dst * d, st);
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
  int rc = onehot_shape_checks(g, d, B, "rgcn_basis_diagcoef_backward");
  if (rc) return rc;
  if (!H || !Vf || !Vb || !Cf || !Cb || !Wself || !saved || !dOut || !dH || !dVf || !dVb || !dCf || !dCb ||
      !dWself || !db || !workspace || (relu && !out) || keep <= 0.f) {
    rgcn_set_error("rgcn_basis_diagcoef_backward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_basis_diagcoef_workspace_bytes(g, d, B, 1)) {
    rgcn_set_error("rgcn_basis_diagcoef_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = diagcoef_graph_checks(g, d, B, "rgcn_basis_diagcoef_backward");
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
  if (!drop_mask) dS = G;

  MARK("start");
  rc = launch_diagcoef_sigmoid(Cf, Cb, (int64_t)R * dB, sig, st);
  if (rc) return rc;
  // G = dOut * relu'(out);  dS = G * mask / keep   (dropout is on the self loop only)
  if (!relu && !drop_mask) {
    G = dS = const_cast<float*>(dOut);
  } else {
    rc = launch_grad_prologue(dOut, out, drop_mask, 1.0f / keep, relu, (int64_t)g->V_dst * d, G, dS, st);
    if (rc) return rc;
  }
  rc = launch_diagcoef_colsum(G, g->V_dst, d, db, st);
  if (rc) return rc;
  MARK("grad_prologue_db");
  rc = gemm_any(st, split_ws, true, false, d, d, g->V_dst, H, d, dS, d, 0.f, dWself, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, true, g->V_dst, d, d, dS, d, Wself, d, 0.f, dH, d);
  if (rc) return rc;
  if (g->V_src > g->V_dst) {
    rc = rgcn_check_cuda(cudaMemsetAsync(dH + (size_t)g->V_dst * d, 0,
                                         (size_t)(g->V_src - g->V_dst) * d * sizeof(float), st),
                         "memset(dH halo)");
    if (rc) return rc;
  }
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

// shape, pointer and workspace checks come first (they need no device), then the graph: device, V_src >= V_dst, CSR
static int diag_graph_checks(const rgcn_graph_t* g, int32_t d, const char* who) {
  int rc = layer_checks(g, d, 1, who);
  if (rc) return rc;
  return need_views(g, true, false, who);
}

extern "C" int rgcn_diag_forward(const rgcn_graph_t* g, int32_t d, const float* H, const float* Df, const float* Db,
                                 const float* Wself, const float* b, const uint8_t* drop_mask, float keep, int relu,
                                 float* out, void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = onehot_shape_checks(g, d, 1, "rgcn_diag_forward");
  if (rc) return rc;
  if (!H || !Df || !Db || !Wself || !b || !out || !workspace || keep <= 0.f) {
    rgcn_set_error("rgcn_diag_forward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_diag_workspace_bytes(g, d, 0)) {
    rgcn_set_error("rgcn_diag_forward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = diag_graph_checks(g, d, "rgcn_diag_forward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int64_t n_split = g->by_dst.n_split;
  const int slabs = slabs_for(d);
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* scratch = ws.take<float>(n_split * d);
  int* counters = ws.take<int>(n_split * slabs);
  MARK("start");
  if (n_split > 0) {
    rc = rgcn_check_cuda(cudaMemsetAsync(scratch, 0, (char*)(counters + n_split * slabs) - (char*)scratch, st),
                         "memset(scratch)");
    if (rc) return rc;
  }
  // self-loop term H[0:V_dst] W_self written straight into `out`; the walk applies the dropout mask (gcn_diag.py:39-40)
  rc = gemm_any(st, split_ws, false, false, g->V_dst, d, d, H, d, Wself, d, 0.f, out, d);
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
  int rc = onehot_shape_checks(g, d, 1, "rgcn_diag_backward");
  if (rc) return rc;
  if (!H || !Df || !Db || !Wself || !dOut || !dH || !dDf || !dDb || !dWself || !db || !workspace ||
      (relu && !out) || keep <= 0.f) {
    rgcn_set_error("rgcn_diag_backward: null pointer or keep <= 0");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_diag_workspace_bytes(g, d, 1)) {
    rgcn_set_error("rgcn_diag_backward: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  rc = diag_graph_checks(g, d, "rgcn_diag_backward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = rgcn_check_cuda(cudaSetDevice(g->device), "cudaSetDevice");
  if (rc) return rc;
  const int R = g->n_relw / 2;
  Carver ws(workspace, workspace_bytes);
  float* split_ws = ws.take<float>((int64_t)2 * d * d);
  float* G = ws.take<float>((int64_t)g->V_dst * d);
  float* dS = ws.take<float>((int64_t)g->V_dst * d);
  if (!drop_mask) dS = G;

  MARK("start");
  // G = dOut * relu'(out);  dS = G * mask / keep   (dropout is on the self loop only)
  if (!relu && !drop_mask) {
    G = dS = const_cast<float*>(dOut);
  } else {
    rc = launch_grad_prologue(dOut, out, drop_mask, 1.0f / keep, relu, (int64_t)g->V_dst * d, G, dS, st);
    if (rc) return rc;
  }
  rc = launch_diagcoef_colsum(G, g->V_dst, d, db, st);
  if (rc) return rc;
  MARK("grad_prologue_db");
  rc = gemm_any(st, split_ws, true, false, d, d, g->V_dst, H, d, dS, d, 0.f, dWself, d);
  if (rc) return rc;
  rc = gemm_any(st, split_ws, false, true, g->V_dst, d, d, dS, d, Wself, d, 0.f, dH, d);
  if (rc) return rc;
  if (g->V_src > g->V_dst) {
    rc = rgcn_check_cuda(cudaMemsetAsync(dH + (size_t)g->V_dst * d, 0,
                                         (size_t)(g->V_src - g->V_dst) * d * sizeof(float), st),
                         "memset(dH halo)");
    if (rc) return rc;
  }
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
  int rc = common_checks(g, d, B, "rgcn_block_slice_sumsq");
  if (rc) return rc;
  if (d % B != 0 || !H || !G || !sumsq2 || !workspace) {
    rgcn_set_error("rgcn_block_slice_sumsq: bad arguments");
    return RGCN_ERR_INVALID;
  }
  rc = need_views(g, false, true, "rgcn_block_slice_sumsq");
  if (rc) return rc;
  if (workspace_bytes < rgcn_block_slice_sumsq_workspace_bytes(g, d, B)) {
    rgcn_set_error("rgcn_block_slice_sumsq: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
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
// The decoder-independent body of distmult_rank / rgcn_complex_rank: hi/lo split of `codes` (unless reused), the
// decoder's query rows + gold scores, the scoring GEMM with its rank-counting epilogue, raw/filtered ranks.
// Workspace layout: [hi V*d | lo V*d | Q n*d | gold_sig n | gold_col n | raw_cnt n | known_cnt n].
typedef int (*RankPrepareFn)(const float*, const float*, int, const int32_t*, int64_t, int, float*, float*, int32_t*,
                             cudaStream_t);

static int rank_with_queries(RankPrepareFn prepare, const float* codes, const float* rel, int32_t V, int32_t d,
                             const int32_t* X, int64_t n, int side, const uint32_t* known_mask, int reuse_split,
                             int32_t* raw_rank, int32_t* filtered_rank, void* workspace, int64_t workspace_bytes,
                             cudaStream_t st) {
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)V * d);
  float* lo = ws.take<float>((int64_t)V * d);
  float* Q = ws.take<float>(n * d);
  float* gold_sig = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(codes, d, V, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (rc) return rc;
  rc = prepare(codes, rel, d, X, n, side, Q, gold_sig, gold_col, st);
  if (rc) return rc;
  rc = launch_gemm_rank_tf32x3(Q, d, hi, lo, d, (int)n, V, d, gold_sig, gold_col, known_mask, (V + 31) / 32, raw_cnt,
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
  if (!codes || !rel || (n > 0 && (!X || !raw_rank)) || !workspace || V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 ||
      n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1) || (filtered_rank && !known_mask)) {
    rgcn_set_error("distmult_rank: bad arguments (need d % 4 == 0, side in {0,1}, a known mask when filtered ranks are requested)");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < distmult_rank_workspace_bytes(V, d, n)) {
    rgcn_set_error("distmult_rank: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  return rank_with_queries(launch_distmult_rank_prepare, codes, rel, V, d, X, n, side, known_mask, reuse_split,
                           raw_rank, filtered_rank, workspace, workspace_bytes, (cudaStream_t)stream);
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
  if (!codes || !rel || (n > 0 && (!X || !raw_rank)) || !workspace || V <= 0 || Vrel <= 0 || d <= 0 || d % 4 != 0 ||
      n < 0 || n > 0x7fffffffLL || (side != 0 && side != 1) || (filtered_rank && !known_mask)) {
    rgcn_set_error("rgcn_complex_rank: bad arguments (need d % 4 == 0, side in {0,1}, a known mask when filtered "
                   "ranks are requested)");
    return RGCN_ERR_INVALID;
  }
  if (workspace_bytes < rgcn_complex_rank_workspace_bytes(V, d, n)) {
    rgcn_set_error("rgcn_complex_rank: workspace too small");
    return RGCN_ERR_WORKSPACE;
  }
  return rank_with_queries(launch_complex_rank_prepare, codes, rel, V, d, X, n, side, known_mask, reuse_split,
                           raw_rank, filtered_rank, workspace, workspace_bytes, (cudaStream_t)stream);
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

static int topk_with_queries(RankPrepareFn prepare, const char* who, const float* codes, const float* rel, int32_t V,
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
  const int64_t need = rgcn_topk_workspace_bytes(V, d, n, k);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_topk_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  const int tn = (V + 127) / 128;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)V * d);
  float* lo = ws.take<float>((int64_t)V * d);
  float* Q = ws.take<float>(n * d);
  uint2* cand = ws.take<uint2>(n * tn * k);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(codes, d, V, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = prepare(codes, rel, d, X, n, side, Q, nullptr, nullptr, st);
  if (rc) return rc;
  rc = launch_gemm_topk_tf32x3(Q, d, hi, lo, d, (int)n, V, d, exclude_mask, (V + 31) / 32, k, cand, st);
  if (rc) return rc;
  return launch_topk_merge(cand, n, tn * k, k, ids, energies, st);
}

extern "C" int distmult_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                             const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                             int reuse_split, int32_t* ids, float* energies, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  return topk_with_queries(launch_distmult_rank_prepare, "distmult_topk", codes, rel, V, Vrel, d, X, n, side, k,
                           exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t d,
                                 const int32_t* X, int64_t n, int side, int32_t k, const uint32_t* exclude_mask,
                                 int reuse_split, int32_t* ids, float* energies, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  return topk_with_queries(launch_complex_rank_prepare, "rgcn_complex_topk", codes, rel, V, Vrel, d, X, n, side, k,
                           exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// Relation prediction over all relations, fused (DistMult and ComplEx): queries (h, ?, t)
// ------------------------------------------------------------------------------------------------
// Both decoders' energies are linear in the relation row, so a pair query is one row Q[t] (the decoder's relation
// prepare kernel) and the energies of all relations are Q @ rel[0:R]^T: the entity-side scoring GEMM with its rank or
// top-k epilogue, run with Bt = the hi/lo split of the first R relation rows and N = R.  Rows R..Vrel-1 of `rel` (the
// R-GCN encoders keep a [V, d] relation table) are never split, scored, counted or returned.
// Workspace layouts: rank [hi R*d | lo R*d | Q n*d | gold_sig n | gold_col n | raw_cnt n | known_cnt n] (that of
// rank_with_queries with V = R), top-k [hi R*d | lo R*d | Q n*d | cand n*ceil(R/128)*k] (that of topk_with_queries);
// one relation workspace with its split serves both, never the entity split.
typedef int (*RelationPrepareFn)(const float*, const float*, int, const int32_t*, int64_t, float*, float*, int32_t*,
                                 cudaStream_t);

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

// the argument checks shared by the four relation entry points (before any device work)
static bool relation_args_ok(const char* who, const float* codes, const float* rel, int32_t V, int32_t Vrel,
                             int32_t R, int32_t d, const int32_t* X, int64_t n, const void* out1, const void* out2,
                             const void* workspace) {
  if (!codes || !rel || (n > 0 && (!X || !out1 || !out2)) || !workspace || V <= 0 || d <= 0 || d % 4 != 0 || n < 0 ||
      n > 0x7fffffffLL) {
    rgcn_set_error(std::string(who) + ": bad arguments (need non-null pointers, V > 0, d % 4 == 0)");
    return false;
  }
  if (R < 1 || R > Vrel) {
    rgcn_set_error(std::string(who) + ": R = " + std::to_string(R) + " relations, need 1 <= R <= Vrel = " +
                   std::to_string(Vrel));
    return false;
  }
  return true;
}

static int relation_rank(RelationPrepareFn prepare, const char* who, const float* codes, const float* rel, int32_t V,
                         int32_t Vrel, int32_t R, int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                         int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                         int64_t workspace_bytes, cudaStream_t st) {
  if (!relation_args_ok(who, codes, rel, V, Vrel, R, d, X, n, raw_rank, raw_rank, workspace)) return RGCN_ERR_INVALID;
  if (filtered_rank && !known_mask) {
    rgcn_set_error(std::string(who) + ": bad arguments (filtered ranks need a known mask)");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = rgcn_relation_rank_workspace_bytes(R, d, n);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_relation_rank_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)R * d);
  float* lo = ws.take<float>((int64_t)R * d);
  float* Q = ws.take<float>(n * d);
  float* gold_sig = ws.take<float>(n);
  int32_t* gold_col = ws.take<int32_t>(n);
  int32_t* raw_cnt = ws.take<int32_t>(n);
  int32_t* known_cnt = ws.take<int32_t>(n);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(rel, d, R, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = rgcn_check_cuda(cudaMemsetAsync(raw_cnt, 0, (char*)(known_cnt + n) - (char*)raw_cnt, st), "memset(rank counts)");
  if (rc) return rc;
  rc = prepare(codes, rel, d, X, n, Q, gold_sig, gold_col, st);
  if (rc) return rc;
  rc = launch_gemm_rank_tf32x3(Q, d, hi, lo, d, (int)n, R, d, gold_sig, gold_col, known_mask, (R + 31) / 32, raw_cnt,
                               known_cnt, st);
  if (rc) return rc;
  return launch_distmult_rank_finalize(raw_cnt, known_cnt, n, raw_rank, filtered_rank, st);
}

static int relation_topk(RelationPrepareFn prepare, const char* who, const float* codes, const float* rel, int32_t V,
                         int32_t Vrel, int32_t R, int32_t d, const int32_t* X, int64_t n, int32_t k,
                         const uint32_t* exclude_mask, int reuse_split, int32_t* ids, float* energies, void* workspace,
                         int64_t workspace_bytes, cudaStream_t st) {
  if (!relation_args_ok(who, codes, rel, V, Vrel, R, d, X, n, ids, energies, workspace)) return RGCN_ERR_INVALID;
  if (k < 1 || k > 128) {
    rgcn_set_error(std::string(who) + ": k = " + std::to_string(k) + " is out of range (1 <= k <= 128)");
    return RGCN_ERR_INVALID;
  }
  const int64_t need = rgcn_relation_topk_workspace_bytes(R, d, n, k);
  if (need < 0) return (int)need;
  if (workspace_bytes < need) {
    rgcn_set_error(std::string(who) + ": workspace too small (rgcn_relation_topk_workspace_bytes)");
    return RGCN_ERR_WORKSPACE;
  }
  const int tn = (R + 127) / 128;
  Carver ws(workspace, workspace_bytes);
  float* hi = ws.take<float>((int64_t)R * d);
  float* lo = ws.take<float>((int64_t)R * d);
  float* Q = ws.take<float>(n * d);
  uint2* cand = ws.take<uint2>(n * tn * k);
  int rc = RGCN_OK;
  if (!reuse_split) rc = launch_gemm_split_b(rel, d, R, d, /*transposed=*/0, hi, lo, st);
  if (rc || n == 0) return rc;
  rc = prepare(codes, rel, d, X, n, Q, nullptr, nullptr, st);
  if (rc) return rc;
  rc = launch_gemm_topk_tf32x3(Q, d, hi, lo, d, (int)n, R, d, exclude_mask, (R + 31) / 32, k, cand, st);
  if (rc) return rc;
  return launch_topk_merge(cand, n, tn * k, k, ids, energies, st);
}

extern "C" int distmult_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                      int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                      int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                      int64_t workspace_bytes, void* stream) {
  return relation_rank(launch_distmult_relation_prepare, "distmult_relation_rank", codes, rel, V, Vrel, R, d, X, n,
                       known_mask, reuse_split, raw_rank, filtered_rank, workspace, workspace_bytes,
                       (cudaStream_t)stream);
}

extern "C" int rgcn_complex_relation_rank(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                          int32_t d, const int32_t* X, int64_t n, const uint32_t* known_mask,
                                          int reuse_split, int32_t* raw_rank, int32_t* filtered_rank, void* workspace,
                                          int64_t workspace_bytes, void* stream) {
  return relation_rank(launch_complex_relation_prepare, "rgcn_complex_relation_rank", codes, rel, V, Vrel, R, d, X, n,
                       known_mask, reuse_split, raw_rank, filtered_rank, workspace, workspace_bytes,
                       (cudaStream_t)stream);
}

extern "C" int distmult_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                      int32_t d, const int32_t* X, int64_t n, int32_t k, const uint32_t* exclude_mask,
                                      int reuse_split, int32_t* ids, float* energies, void* workspace,
                                      int64_t workspace_bytes, void* stream) {
  return relation_topk(launch_distmult_relation_prepare, "distmult_relation_topk", codes, rel, V, Vrel, R, d, X, n, k,
                       exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int rgcn_complex_relation_topk(const float* codes, const float* rel, int32_t V, int32_t Vrel, int32_t R,
                                          int32_t d, const int32_t* X, int64_t n, int32_t k,
                                          const uint32_t* exclude_mask, int reuse_split, int32_t* ids,
                                          float* energies, void* workspace, int64_t workspace_bytes, void* stream) {
  return relation_topk(launch_complex_relation_prepare, "rgcn_complex_relation_topk", codes, rel, V, Vrel, R, d, X, n,
                       k, exclude_mask, reuse_split, ids, energies, workspace, workspace_bytes, (cudaStream_t)stream);
}
