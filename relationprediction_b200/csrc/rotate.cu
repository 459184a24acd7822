// rotate.cu -- RotatE (Sun et al., ICLR 2019) triple scorer, loss, backward and all-entity ranking for sm_90a.
// Semantics in DESIGN.md section 1.  Entity rows are [re | im] (h = d / 2 columns each), the phases theta of relation r
// are the first h columns of its row, and with a = codes[s], c = codes[o]:
//   u_k = a_k e^{i theta_k} - c_k,   D = sum_{k<h} |u_k|,   E = gamma - D.
// The scorer and its backward have the ComplEx shape (a warp owns a triple, a lane the column pairs (k, k + h)).  The
// ranking cannot be a GEMM -- a modulus is not a product -- so k_rotate_rank is a tiled all-pairs distance kernel on
// the CUDA cores: k_dist_tile (dist_tile.cuh) with RotatE's per-pair modulus.
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

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the two entity rows
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, float gamma, float* __restrict__ energies,
                 float* __restrict__ loss_acc) {
  // per-warp sums, kept by lane 0 in shared memory: as registers live across the whole loop, ptxas spills them
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const RotateRows<W> rows{gamma};
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

__global__ void k_rotate_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// With g = dL/dE, m = |u|, w = u / m (0 where m = 0), p = a e^{i theta} and dE = -dD:
//   dc = g w,   da = -g [w_re cos + w_im sin, -w_re sin + w_im cos],   dtheta = -g (w_im p_re - w_re p_im)
// plus c_reg x on the entity rows (the L2 term).  Columns h..d-1 of the relation row get nothing.
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, const float* __restrict__ energies, float g_loss_over_n,
                 float c_reg, const float* __restrict__ g_scale, const float* __restrict__ g_energy,
                 float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      gx += g_loss_over_n * (1.f / (1.f + expf(-e)) - __ldg(Y + n));
    }
    const float* e1 = codes + (size_t)s * d;
    const float* th = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float ar[W], ai[W], t[W], cr[W], ci[W];
      Vec<W>::load(e1 + k, ar), Vec<W>::load(e1 + h + k, ai);
      Vec<W>::load(th + k, t);
      Vec<W>::load(e2 + k, cr), Vec<W>::load(e2 + h + k, ci);
      float dar[W], dai[W], dt[W], dcr[W], dci[W];
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float ur, ui, sn, cs;
        rotate_residual(ar[j], ai[j], t[j], cr[j], ci[j], ur, ui, sn, cs);
        const float m = rotate_modulus(ur, ui);
        const float gm = m > 0.f ? gx / m : 0.f;   // g / m: the subgradient 0 where u = 0
        const float wr = gm * ur, wi = gm * ui;     // g w
        const float pr = fmaf(ar[j], cs, -ai[j] * sn), pi = fmaf(ar[j], sn, ai[j] * cs);
        dcr[j] = fmaf(c_reg, cr[j], wr);
        dci[j] = fmaf(c_reg, ci[j], wi);
        dar[j] = fmaf(c_reg, ar[j], -fmaf(wr, cs, wi * sn));
        dai[j] = fmaf(c_reg, ai[j], -fmaf(wi, cs, -wr * sn));
        dt[j] = fmaf(wr, pi, -wi * pr);
        slice_sq += dt[j] * dt[j];
      }
      Vec<W>::red(g1 + k, dar), Vec<W>::red(g1 + h + k, dai);
      Vec<W>::red(gr + k, dt);
      Vec<W>::red(g2 + k, dcr), Vec<W>::red(g2 + h + k, dci);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- all-entity ranking by distance (the tile kernel and its fixed summation order: dist_tile.cuh) -------------
__device__ __forceinline__ float rotate_dist_step(float qr, float qi, float vr, float vi, float acc) {
  return __fadd_rn(acc, rotate_modulus(__fsub_rn(qr, vr), __fsub_rn(qi, vi)));
}

struct RotateStep {
  __device__ __forceinline__ static float step(float qr, float qi, float vr, float vi, float acc) {
    return rotate_dist_step(qr, qi, vr, vi, acc);
  }
};

// One warp per query t.  side 1 (objects corrupted): q = codes[s] e^{i theta}, gold o; side 0 (subjects corrupted):
// q = codes[o] e^{-i theta}, gold s -- |a e^{i theta} - c| = |a - c e^{-i theta}|.  Lane 0 then sums the gold's
// distance sequentially from the float32 q just stored, as k_rotate_rank will.
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                          const int32_t* __restrict__ X, int64_t n, int side, float* __restrict__ Q,
                          float* __restrict__ gold_D, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const int kept = side == 0 ? o : s, gold = side == 0 ? s : o;
    const float* ek = codes + (size_t)kept * d;
    const float* th = rel + (size_t)r * d;
    float* q = Q + (size_t)t * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float kr[W], ki[W], tt[W], qr[W], qi[W];
      Vec<W>::load(ek + k, kr), Vec<W>::load(ek + h + k, ki);
      Vec<W>::load(th + k, tt);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float sn, cs;
        sincosf(tt[j], &sn, &cs);
        if (side == 0) sn = -sn;
        qr[j] = fmaf(kr[j], cs, -ki[j] * sn);
        qi[j] = fmaf(kr[j], sn, ki[j] * cs);
      }
      Vec<W>::store(q + k, qr), Vec<W>::store(q + h + k, qi);
    }
    __syncwarp();   // the warp's stores of q are visible to lane 0
    if (lane == 0) {
      const float* g = codes + (size_t)gold * d;
      float D = 0.f;
      for (int k0 = 0; k0 < h; k0 += RK_KC) {
        float part = 0.f;
        for (int k = k0; k < min(k0 + RK_KC, h); ++k)
          part = rotate_dist_step(q[k], q[h + k], __ldg(g + k), __ldg(g + h + k), part);
        D = __fadd_rn(D, part);
      }
      gold_D[t] = D;
      gold_col[t] = gold;
    }
    __syncwarp();
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) { return (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, 132 * 8)); }

}  // namespace

int launch_rotate_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          float gamma, float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc || N == 0) return rc;
  if (d % 8 == 0)
    k_rotate_fwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, gamma, energies, loss_out);
  else
    k_rotate_fwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, gamma, energies, loss_out);
  rc = check_launch("k_rotate_fwd");
  if (rc) return rc;
  k_rotate_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_rotate_finalize");
}

int launch_rotate_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                           const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  if (d % 8 == 0)
    k_rotate_bwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                           g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  else
    k_rotate_bwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                           g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_rotate_bwd");
}

int launch_rotate_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                               float* Q, float* gold_D, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  if (d % 8 == 0)
    k_rotate_rank_prepare<4><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_D, gold_col);
  else
    k_rotate_rank_prepare<2><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_D, gold_col);
  return check_launch("k_rotate_rank_prepare");
}

int launch_rotate_rank(const float* Q, const float* codes, int V, int d, int64_t n, const float* gold_D,
                       const int32_t* gold_col, const uint32_t* known, int32_t* raw_cnt, int32_t* known_cnt,
                       cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_dist_tile<RotateStep, DistRankEpi><<<dist_tile_grid(V, n), 256, 0, st>>>(Q, codes, V, d, n, gold_D, gold_col, known,
                                                                            (V + 31) / 32, raw_cnt, known_cnt);
  return check_launch("k_dist_tile<rotate, rank>");
}
