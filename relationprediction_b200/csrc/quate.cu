// quate.cu -- QuatE (Zhang, Tay, Yao, Liu; NeurIPS 2019) triple scorer, loss and backward, and the query rows and
// query backward that put QuatE on the DistMult scoring GEMMs (ranks, top-k, 1-N), for sm_90a.  Semantics in DESIGN.md
// section 1.  Quaternion k of a row is the float4 at column 4k; with h = codes[s], r = rel[r], t = codes[o] and
// rh_k = r_k / max(|r_k|, eps):
//   E = sum_k <h_k (x) rh_k, t_k> = sum_k <h_k, t_k (x) conj(rh_k)> = sum_k <rh_k, conj(h_k) (x) t_k>.
// The energy is linear in each of the three rows, so every all-candidate query is one query row against a table:
// h (x) rh against the objects, t (x) conj(rh) against the subjects, conj(h) (x) t against the normalised relations.
// The scorer and its backward have the DistMult shape: a warp owns a triple, a lane whole quaternions.
#include <cuda_runtime.h>

#include <algorithm>

#include "kernels.cuh"
#include "triple_rows.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

__device__ __forceinline__ void red4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

__device__ __forceinline__ float4 axpy4(float a, float4 x, float4 y) {   // a x + y
  return make_float4(fmaf(a, x.x, y.x), fmaf(a, x.y, y.y), fmaf(a, x.z, y.z), fmaf(a, x.w, y.w));
}

__device__ __forceinline__ float4 scale4(float a, float4 x) { return make_float4(a * x.x, a * x.y, a * x.z, a * x.w); }

__device__ __forceinline__ float sumsq4(float4 x) { return x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w; }

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the three raw rows
__global__ void __launch_bounds__(256)
    k_quate_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                int64_t N, const float* __restrict__ Y, float* __restrict__ energies, float* __restrict__ loss_acc) {
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh_l[warp] = sh_q[warp] = 0.0;
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float e = 0.f, q = 0.f;
    QuatERows::partial(codes, rel, d, s, r, o, lane, e, q);
    e = warp_sum(e);
    q = warp_sum(q);
    if (lane == 0) {
      energies[n] = e;
      if (Y) {
        const float y = __ldg(Y + n);
        // the reference's sigmoid cross-entropy (pos_weight 1): (1 - y) x + log1p(exp(-|x|)) + max(-x, 0)
        sh_l[warp] += (double)((1.f - y) * e + log1pf(expf(-fabsf(e))) + fmaxf(-e, 0.f));
      }
      sh_q[warp] += (double)q;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double L = 0.0, Q = 0.0;
    for (int w = 0; w < 8; ++w) {
      L += sh_l[w];
      Q += sh_q[w];
    }
    atomicAdd(loss_acc + 0, (float)L);
    atomicAdd(loss_acc + 1, (float)Q);
  }
}

__global__ void k_quate_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// With g = dL/dE, per quaternion:  dh = g t (x) conj(rh),  dt = g h (x) rh,  drh = g conj(h) (x) t, taken back to r
// through the normalisation; plus c_reg x on the three raw rows (the L2 term).
__global__ void __launch_bounds__(256)
    k_quate_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                int64_t N, const float* __restrict__ Y, const float* __restrict__ energies, float g_loss_over_n,
                float c_reg, const float* __restrict__ g_scale, const float* __restrict__ g_energy,
                float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      gx += g_loss_over_n * (1.f / (1.f + expf(-e)) - __ldg(Y + n));
    }
    const float4* e1 = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* e2 = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(e1 + i), b = __ldg(rr + i), c = __ldg(e2 + i);
      float m;
      const float4 bh = quat_normalize(b, m);
      const float4 da = axpy4(gx, quat_mul(c, quat_conj(bh)), scale4(c_reg, a));
      const float4 dc = axpy4(gx, quat_mul(a, bh), scale4(c_reg, c));
      const float4 db = axpy4(1.f, quat_normalize_bwd(bh, m, scale4(gx, quat_mul(quat_conj(a), c))),
                              scale4(c_reg, b));
      red4(g1 + 4 * i, da);
      red4(gr + 4 * i, db);
      red4(g2 + 4 * i, dc);
      slice_sq += sumsq4(db);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- query rows for the scoring GEMMs ------------------------------------------------------------------------------
// One warp per query t = (s, r, o).  side 1 (objects corrupted): Q = h (x) rh, kept s, gold o; side 0 (subjects
// corrupted): Q = t (x) conj(rh), kept o, gold s.  With gold_sig, also gold_sig[t] = sigmoid(<Q, codes[gold]>) from
// the float32 Q just stored (k_rank_prepare's rule) and gold_col[t] = gold; gold_sig == nullptr: Q only, the predicted
// column of X is not read.
__global__ void __launch_bounds__(256)
    k_quate_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                         const int32_t* __restrict__ X, int64_t n, int side, float* __restrict__ Q,
                         float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const int kept = side == 0 ? o : s, gold = side == 0 ? s : o;
    const float4* ek = reinterpret_cast<const float4*>(codes + (size_t)kept * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* eg = reinterpret_cast<const float4*>(codes + (size_t)gold * d);
    float4* q = reinterpret_cast<float4*>(Q + (size_t)t * d);
    float e = 0.f;
    for (int i = lane; i < d4; i += 32) {
      float m;
      const float4 bh = quat_normalize(__ldg(rr + i), m);
      const float4 p = quat_mul(__ldg(ek + i), side == 0 ? quat_conj(bh) : bh);
      q[i] = p;
      if (gold_sig) e = quat_dot(p, __ldg(eg + i), e);
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = gold;
    }
  }
}

// rh[j] = the normalised quaternion j of rel, j < count (the first R rows of the relation table, R d / 4 quaternions)
__global__ void __launch_bounds__(256)
    k_quate_normalize(const float4* __restrict__ rel, int64_t count, float4* __restrict__ rh) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < count; j += (int64_t)gridDim.x * blockDim.x) {
    float m;
    rh[j] = quat_normalize(__ldg(rel + j), m);
  }
}

// Pair queries (h, ?, t): Q = conj(h) (x) t, scored against the normalised relation rows.  gold_sig[t] =
// sigmoid(<Q, rh[r]>) with rh[r] formed by quat_normalize, as k_quate_normalize writes it, gold_col[t] = r
// (gold_sig == nullptr: Q only; the relation column of X is then not read).
__global__ void __launch_bounds__(256)
    k_quate_relation_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                             const int32_t* __restrict__ X, int64_t n, float* __restrict__ Q,
                             float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), o = __ldg(X + 3 * t + 2);
    const int r = gold_sig ? __ldg(X + 3 * t + 1) : 0;
    const float4* eh = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* et = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    float4* q = reinterpret_cast<float4*>(Q + (size_t)t * d);
    float e = 0.f;
    for (int i = lane; i < d4; i += 32) {
      const float4 p = quat_mul(quat_conj(__ldg(eh + i)), __ldg(et + i));
      q[i] = p;
      if (gold_sig) {
        float m;
        e = quat_dot(p, quat_normalize(__ldg(rr + i), m), e);
      }
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = r;
    }
  }
}

// 1-N query backward, queries (anchor k, r, anchor) of one side, dQ [n, d]:
//   side 1: Q = k (x) rh        ->  dk = dQ (x) conj(rh),  drh = conj(k) (x) dQ
//   side 0: Q = k (x) conj(rh)  ->  dk = dQ (x) rh,        drh = conj(dQ) (x) k
// drh goes back to r through the normalisation; each + c k (c r), the L2 term of the raw rows.
__global__ void __launch_bounds__(256)
    k_quate_query_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                      const int32_t* __restrict__ X, int64_t n, int side, const float* __restrict__ dQ,
                      const float* __restrict__ g_scale, float c_reg, float* __restrict__ dcodes,
                      float* __restrict__ drel) {
  if (g_scale) c_reg *= __ldg(g_scale + 1);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int a = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    const float4* ek = reinterpret_cast<const float4*>(codes + (size_t)a * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* gq = reinterpret_cast<const float4*>(dQ + (size_t)t * d);
    float* gk = dcodes + (size_t)a * d;
    float* gr = drel + (size_t)r * d;
    for (int i = lane; i < d4; i += 32) {
      const float4 k = __ldg(ek + i), b = __ldg(rr + i), g = __ldg(gq + i);
      float m;
      const float4 bh = quat_normalize(b, m);
      const float4 dk = side == 0 ? quat_mul(g, bh) : quat_mul(g, quat_conj(bh));
      const float4 dbh = side == 0 ? quat_mul(quat_conj(g), k) : quat_mul(quat_conj(k), g);
      red4(gk + 4 * i, axpy4(c_reg, k, dk));
      red4(gr + 4 * i, axpy4(c_reg, b, quat_normalize_bwd(bh, m, dbh)));
    }
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) { return (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, 132 * 8)); }

}  // namespace

int launch_quate_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                         float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc || N == 0) return rc;
  k_quate_fwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, loss_out);
  rc = check_launch("k_quate_fwd");
  if (rc) return rc;
  k_quate_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_quate_finalize");
}

int launch_quate_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                          const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  k_quate_bwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                     g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_quate_bwd");
}

int launch_quate_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                              float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_quate_rank_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_sig, gold_col);
  return check_launch("k_quate_rank_prepare");
}

int launch_quate_normalize(const float* rel, int R, int d, float* rh, cudaStream_t st) {
  const int64_t count = (int64_t)R * (d / 4);
  if (count == 0) return RGCN_OK;
  const int blocks = (int)std::min<int64_t>((count + 255) / 256, 132 * 8);
  k_quate_normalize<<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(rel), count,
                                            reinterpret_cast<float4*>(rh));
  return check_launch("k_quate_normalize");
}

int launch_quate_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* Q,
                                  float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_quate_relation_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, Q, gold_sig, gold_col);
  return check_launch("k_quate_relation_prepare");
}

int launch_quate_query_bwd(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                           const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                           cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_quate_query_bwd<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, dQ, g_scale, c_reg, dcodes,
                                                           drel);
  return check_launch("k_quate_query_bwd");
}
