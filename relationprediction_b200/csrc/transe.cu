// transe.cu -- TransE (Bordes et al., NIPS 2013) triple scorer, loss, backward, and all-entity and all-relation ranking
// and top-k by L1 distance for sm_90a.  Semantics in DESIGN.md section 1.  Entity and relation rows are plain real
// vectors of d columns, and with h = codes[s], r = rel[r], t = codes[o]:
//   u_k = (h_k + r_k) - t_k,   D = sum_k |u_k|,   E = gamma - D.
// The scorer and its backward have the DistMult shape (a warp owns a triple, a lane 4 consecutive columns).  Every
// query is "rank the rows of a table by L1 distance to one query row": |h + r - t| = |v - q| with q = h + r against the
// objects, q = t - r against the subjects and q = t - h against the relations.  So the four inference paths are
// k_dist_tile (dist_tile.cuh) with TransE's per-pair term and the rank or top-k epilogue.
#include <cuda_runtime.h>

#include <algorithm>

#include "dist_tile.cuh"
#include "kernels.cuh"
#include "triple_rows.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the three rows
__global__ void __launch_bounds__(256)
    k_transe_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, float gamma, float* __restrict__ energies,
                 float* __restrict__ loss_acc) {
  // per-warp sums, kept by lane 0 in shared memory, as k_rotate_fwd does
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TransERows<4> rows{gamma};
  if (lane == 0) sh_l[warp] = sh_q[warp] = 0.0;
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float e = 0.f, q = 0.f;
    rows.partial(codes, rel, d, s, r, o, lane, e, q);
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

__global__ void k_transe_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// With g = dL/dE and s = sign(u) (0 where u = 0, the subgradient):  dh = dr = -g s,  dt = g s,  plus c_reg x on all
// three rows (the L2 term).
__global__ void __launch_bounds__(256)
    k_transe_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, const float* __restrict__ energies, float g_loss_over_n,
                 float c_reg, const float* __restrict__ g_scale, const float* __restrict__ g_energy,
                 float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      gx += g_loss_over_n * (1.f / (1.f + expf(-e)) - __ldg(Y + n));
    }
    const float* e1 = codes + (size_t)s * d;
    const float* rr = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int k = lane * 4; k < d; k += 32 * 4) {
      float a[4], b[4], c[4];
      Vec<4>::load(e1 + k, a), Vec<4>::load(rr + k, b), Vec<4>::load(e2 + k, c);
      float da[4], db[4], dc[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float u = transe_residual(a[j], b[j], c[j]);
        const float gs = u > 0.f ? gx : (u < 0.f ? -gx : 0.f);   // g sign(u)
        da[j] = fmaf(c_reg, a[j], -gs);
        db[j] = fmaf(c_reg, b[j], -gs);
        dc[j] = fmaf(c_reg, c[j], gs);
        slice_sq += db[j] * db[j];
      }
      Vec<4>::red(g1 + k, da), Vec<4>::red(gr + k, db), Vec<4>::red(g2 + k, dc);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- ranking and top-k by distance (the tile kernel and its fixed summation order: dist_tile.cuh) ---------------
__device__ __forceinline__ float transe_dist_step(float qr, float qi, float vr, float vi, float acc) {
  return __fadd_rn(__fadd_rn(acc, fabsf(__fsub_rn(qr, vr))), fabsf(__fsub_rn(qi, vi)));
}

struct TransEStep {
  __device__ __forceinline__ static float step(float qr, float qi, float vr, float vi, float acc) {
    return transe_dist_step(qr, qi, vr, vi, acc);
  }
};

// One warp per query t = (s, r, o).  mode 1 (objects corrupted): q = codes[s] + rel[r], gold o; mode 0 (subjects
// corrupted): q = codes[o] - rel[r], gold s; TRANSE_RELATIONS: q = codes[o] - codes[s], gold r, candidates rel.  With
// gold_D, lane 0 then sums the gold's distance sequentially from the float32 q just stored, in k_dist_tile's order.
__global__ void __launch_bounds__(256)
    k_transe_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                     const int32_t* __restrict__ X, int64_t n, int mode, float* __restrict__ Q,
                     float* __restrict__ gold_D, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const float* a = mode == 1 ? codes + (size_t)s * d : codes + (size_t)o * d;
    const float* b = mode == TRANSE_RELATIONS ? codes + (size_t)s * d : rel + (size_t)r * d;
    float* q = Q + (size_t)t * d;
    for (int k = lane * 4; k < d; k += 32 * 4) {
      float x[4], y[4], z[4];
      Vec<4>::load(a + k, x), Vec<4>::load(b + k, y);
#pragma unroll
      for (int j = 0; j < 4; ++j) z[j] = mode == 1 ? __fadd_rn(x[j], y[j]) : __fsub_rn(x[j], y[j]);
      Vec<4>::store(q + k, z);
    }
    if (gold_D) {
      __syncwarp();   // the warp's stores of q are visible to lane 0
      if (lane == 0) {
        const int gold = mode == TRANSE_RELATIONS ? r : mode == 0 ? s : o;
        const float* g = (mode == TRANSE_RELATIONS ? rel : codes) + (size_t)gold * d;
        float D = 0.f;
        for (int k0 = 0; k0 < h; k0 += RK_KC) {
          float part = 0.f;
          for (int k = k0; k < min(k0 + RK_KC, h); ++k)
            part = transe_dist_step(q[k], q[h + k], __ldg(g + k), __ldg(g + h + k), part);
          D = __fadd_rn(D, part);
        }
        gold_D[t] = D;
        gold_col[t] = gold;
      }
      __syncwarp();
    }
  }
}

// energies = gamma - D from the merged -D, rounded once; the (-1, -inf) tail stays -inf
__global__ void k_transe_margin(float* __restrict__ energies, int64_t count, float gamma) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    energies[i] = __fadd_rn(gamma, energies[i]);
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) { return (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, 132 * 8)); }

}  // namespace

int launch_transe_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          float gamma, float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc || N == 0) return rc;
  k_transe_fwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, gamma, energies, loss_out);
  rc = check_launch("k_transe_fwd");
  if (rc) return rc;
  k_transe_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_transe_finalize");
}

int launch_transe_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                           const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  k_transe_bwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                      g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_transe_bwd");
}

int launch_transe_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int mode,
                          float* Q, float* gold_D, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_transe_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, mode, Q, gold_D, gold_col);
  return check_launch("k_transe_prepare");
}

int launch_transe_rank(const float* Q, const float* table, int V, int d, int64_t n, const float* gold_D,
                       const int32_t* gold_col, const uint32_t* known, int32_t* raw_cnt, int32_t* known_cnt,
                       cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_dist_tile<TransEStep, DistRankEpi><<<dist_tile_grid(V, n), 256, 0, st>>>(Q, table, V, d, n, gold_D, gold_col, known,
                                                                            (V + 31) / 32, raw_cnt, known_cnt);
  return check_launch("k_dist_tile<transe, rank>");
}

int launch_transe_topk(const float* Q, const float* table, int V, int d, int64_t n, const uint32_t* excl, int k,
                       float gamma, uint2* cand, int32_t* ids, float* energies, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_dist_tile<TransEStep, DistTopKEpi><<<dist_tile_grid(V, n), 256, 0, st>>>(Q, table, V, d, n, excl, (V + 31) / 32, k,
                                                                            cand);
  int rc = check_launch("k_dist_tile<transe, topk>");
  if (!rc) rc = launch_topk_merge(cand, n, transe_topk_tiles(V) * k, k, ids, energies, st);
  if (rc) return rc;
  const int64_t count = n * k;
  k_transe_margin<<<(unsigned)std::min<int64_t>((count + 255) / 256, 132 * 16), 256, 0, st>>>(energies, count, gamma);
  return check_launch("k_transe_margin");
}
