// distmult.cu -- DistMult ("BilinearDiag") triple scorer, loss and backward for sm_90a.
// Reference: decoders/bilinear_diag.py:14-34 (gathers, energy, sigmoid cross-entropy with
// pos_weight forced to 1) and :63-69 (L2 regulariser over the gathered rows).
// Bandwidth-bound: a warp owns one triple = three row gathers with 128-bit loads; the loss terms
// are reduced warp -> block -> one atomic per block.
#include <cuda_runtime.h>

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
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares
__global__ void __launch_bounds__(256)
    k_distmult_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                   const int32_t* __restrict__ X, int64_t N, const float* __restrict__ Y,
                   float* __restrict__ energies, float* __restrict__ loss_acc) {
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wid0 = (int64_t)blockIdx.x * 8 + warp;
  const int64_t wstride = (int64_t)gridDim.x * 8;
  double lsum = 0.0, qsum = 0.0;
  for (int64_t n = wid0; n < N; n += wstride) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float e = 0.f, q = 0.f;
    DistMultRows::partial(codes, rel, d, s, r, o, lane, e, q);
    e = warp_sum(e);
    q = warp_sum(q);
    if (lane == 0) {
      energies[n] = e;
      if (Y) {
        const float y = __ldg(Y + n);
        // weighted_cross_entropy_with_logits, pos_weight = 1 (bilinear_diag.py:32-34):
        // (1 - y) * x + log1p(exp(-|x|)) + max(-x, 0)
        const float l = (1.f - y) * e + log1pf(expf(-fabsf(e))) + fmaxf(-e, 0.f);
        lsum += (double)l;
      }
      qsum += (double)q;
    }
  }
  if (lane == 0) {
    sh_l[warp] = lsum;
    sh_q[warp] = qsum;
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

__global__ void k_distmult_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

__global__ void __launch_bounds__(256)
    k_distmult_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                   const int32_t* __restrict__ X, int64_t N, const float* __restrict__ Y,
                   const float* __restrict__ energies, float g_loss_over_n, float c_reg,
                   const float* __restrict__ g_scale, const float* __restrict__ g_energy,
                   float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wid0 = (int64_t)blockIdx.x * 8 + warp;
  const int64_t wstride = (int64_t)gridDim.x * 8;
  const int d4 = d >> 2;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = wid0; n < N; n += wstride) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      const float sg = 1.f / (1.f + expf(-e));
      gx += g_loss_over_n * (sg - __ldg(Y + n));
    }
    const float4* e1 = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* e2 = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(e1 + i), b = __ldg(rr + i), c = __ldg(e2 + i);
      float4 da, db, dc;
      da.x = fmaf(gx, b.x * c.x, c_reg * a.x);
      da.y = fmaf(gx, b.y * c.y, c_reg * a.y);
      da.z = fmaf(gx, b.z * c.z, c_reg * a.z);
      da.w = fmaf(gx, b.w * c.w, c_reg * a.w);
      db.x = fmaf(gx, a.x * c.x, c_reg * b.x);
      db.y = fmaf(gx, a.y * c.y, c_reg * b.y);
      db.z = fmaf(gx, a.z * c.z, c_reg * b.z);
      db.w = fmaf(gx, a.w * c.w, c_reg * b.w);
      dc.x = fmaf(gx, a.x * b.x, c_reg * c.x);
      dc.y = fmaf(gx, a.y * b.y, c_reg * c.y);
      dc.z = fmaf(gx, a.z * b.z, c_reg * c.z);
      dc.w = fmaf(gx, a.w * b.w, c_reg * c.w);
      red4(g1 + 4 * i, da);
      red4(gr + 4 * i, db);
      red4(g2 + 4 * i, dc);
      slice_sq += db.x * db.x + db.y * db.y + db.z * db.z + db.w * db.w;
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- fused all-entity scoring + ranking (next row N3): query rows and gold scores --------------------------------
__global__ void __launch_bounds__(256)
    k_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                   int64_t n, int side, float* __restrict__ Q, float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
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
      const float4 a = __ldg(ek + i), b = __ldg(rr + i);
      const float4 p = make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
      q[i] = p;
      if (gold_sig) {   // the top-k path asks for the query rows only: the predicted column of X is not read
        const float4 c = __ldg(eg + i);
        e = fmaf(p.x, c.x, e);
        e = fmaf(p.y, c.y, e);
        e = fmaf(p.z, c.z, e);
        e = fmaf(p.w, c.w, e);
      }
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = gold;
    }
  }
}

// ---- fused all-relation scoring + ranking / top-k: pair queries (h, ?, t) ----------------------------------------
// The energy is linear in the relation row: e(h, r, t) = <codes[h] * codes[t], rel[r]>, so Q[t] = codes[h] * codes[t]
// is scored against every relation row by the same GEMM.  gold_sig[t] = sigmoid(<Q[t], rel[r]>), gold_col[t] = r
// (gold_sig == nullptr: Q only; the relation column of X is then not read).
__global__ void __launch_bounds__(256)
    k_relation_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                       const int32_t* __restrict__ X, int64_t n, float* __restrict__ Q, float* __restrict__ gold_sig,
                       int32_t* __restrict__ gold_col) {
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
      const float4 a = __ldg(eh + i), b = __ldg(et + i);
      const float4 p = make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
      q[i] = p;
      if (gold_sig) {
        const float4 c = __ldg(rr + i);
        e = fmaf(p.x, c.x, e);
        e = fmaf(p.y, c.y, e);
        e = fmaf(p.z, c.z, e);
        e = fmaf(p.w, c.w, e);
      }
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = r;
    }
  }
}

// raw rank = #{score >= gold}; filtered rank = raw - #{known with score >= gold} + 1 (common/evaluation.py:148-152)
__global__ void k_rank_finalize(const int32_t* __restrict__ raw_cnt, const int32_t* __restrict__ known_cnt, int64_t n,
                                int32_t* __restrict__ raw_rank, int32_t* __restrict__ filtered_rank) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    raw_rank[t] = raw_cnt[t];
    if (filtered_rank) filtered_rank[t] = raw_cnt[t] - known_cnt[t] + 1;
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) {
  int64_t b = (N + 7) / 8;
  const int64_t cap = 132 * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

int launch_distmult_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N,
                            const float* Y, float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc) return rc;
  if (N == 0) return RGCN_OK;
  k_distmult_fwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, loss_out);
  rc = check_launch("k_distmult_fwd");
  if (rc) return rc;
  k_distmult_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_distmult_finalize");
}

int launch_distmult_backward(const float* codes, const float* rel, int d, const int32_t* X,
                             int64_t N, const float* Y, const float* energies, float g_loss,
                             float g_reg, const float* g_scale_dev, const float* g_energy,
                             float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  k_distmult_bwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies,
                                                        g_loss_over_n, c_reg, g_scale_dev, g_energy,
                                                        dcodes, drel, rel_slice_sumsq);
  return check_launch("k_distmult_bwd");
}

int launch_distmult_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                                 float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_rank_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_sig, gold_col);
  return check_launch("k_rank_prepare");
}

int launch_distmult_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                                     float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_relation_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, Q, gold_sig, gold_col);
  return check_launch("k_relation_prepare");
}

int launch_distmult_rank_finalize(const int32_t* raw_cnt, const int32_t* known_cnt, int64_t n, int32_t* raw_rank,
                                  int32_t* filtered_rank, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  int64_t b = (n + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  k_rank_finalize<<<(int)b, 256, 0, st>>>(raw_cnt, known_cnt, n, raw_rank, filtered_rank);
  return check_launch("k_rank_finalize");
}
