// complex.cu -- ComplEx triple scorer, loss, backward and rank queries for sm_90a.
// Reference: decoders/complex.py:18-45 (gathers, energy, sigmoid cross-entropy with pos_weight forced to 1),
// :71-75 (a row of width d is [real | imaginary], h = d/2 columns each), :77-106 (all-entity scoring) and
// :108-114 (L2 regulariser over the gathered rows, all d columns).
// Same memory-bound shape as DistMult: a warp owns one triple = three row gathers; a lane owns the column pairs
// (k, k+h) of all three rows, so every complex product is formed in registers.  The imaginary half starts h floats
// into the row: 16-byte aligned when d % 8 == 0 (float4 path), only 8-byte aligned when d % 8 == 4 (float2 path,
// e.g. d = 500).  The loss terms are reduced warp -> block -> one atomic per block.
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

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the gathered rows
template <int W>
__global__ void __launch_bounds__(256)
    k_complex_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
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
    ComplexRows<W>::partial(codes, rel, d, s, r, o, lane, e, q);   // complex.py:38-41
    e = warp_sum(e);
    q = warp_sum(q);
    if (lane == 0) {
      energies[n] = e;
      if (Y) {
        const float y = __ldg(Y + n);
        // weighted_cross_entropy_with_logits, pos_weight = 1 (complex.py:43-45):
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

__global__ void k_complex_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// with g = dL/dE:  de1 = g [rr e2r + ri e2i, rr e2i - ri e2r],  dr = g [e1r e2r + e1i e2i, e1r e2i - e1i e2r],
//                  de2 = g [e1r rr - e1i ri, e1i rr + e1r ri];  each + c_reg * x (the L2 term)
template <int W>
__global__ void __launch_bounds__(256)
    k_complex_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
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
  const int h = d >> 1;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = wid0; n < N; n += wstride) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      const float sg = 1.f / (1.f + expf(-e));
      gx += g_loss_over_n * (sg - __ldg(Y + n));
    }
    const float* e1 = codes + (size_t)s * d;
    const float* rr = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float ar[W], ai[W], br[W], bi[W], cr[W], ci[W];
      Vec<W>::load(e1 + k, ar), Vec<W>::load(e1 + h + k, ai);
      Vec<W>::load(rr + k, br), Vec<W>::load(rr + h + k, bi);
      Vec<W>::load(e2 + k, cr), Vec<W>::load(e2 + h + k, ci);
      float dar[W], dai[W], dbr[W], dbi[W], dcr[W], dci[W];
#pragma unroll
      for (int j = 0; j < W; ++j) {
        dar[j] = fmaf(gx, fmaf(br[j], cr[j], bi[j] * ci[j]), c_reg * ar[j]);
        dai[j] = fmaf(gx, fmaf(br[j], ci[j], -bi[j] * cr[j]), c_reg * ai[j]);
        dbr[j] = fmaf(gx, fmaf(ar[j], cr[j], ai[j] * ci[j]), c_reg * br[j]);
        dbi[j] = fmaf(gx, fmaf(ar[j], ci[j], -ai[j] * cr[j]), c_reg * bi[j]);
        dcr[j] = fmaf(gx, fmaf(ar[j], br[j], -ai[j] * bi[j]), c_reg * cr[j]);
        dci[j] = fmaf(gx, fmaf(ai[j], br[j], ar[j] * bi[j]), c_reg * ci[j]);
        slice_sq += dbr[j] * dbr[j] + dbi[j] * dbi[j];
      }
      Vec<W>::red(g1 + k, dar), Vec<W>::red(g1 + h + k, dai);
      Vec<W>::red(gr + k, dbr), Vec<W>::red(gr + h + k, dbi);
      Vec<W>::red(g2 + k, dcr), Vec<W>::red(g2 + h + k, dci);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- fused all-entity scoring + ranking: query rows and gold scores (complex.py:77-106) --------------------------
// side 0 (subjects corrupted): Q = [rr e2r + ri e2i, rr e2i - ri e2r], gold = s
// side 1 (objects corrupted):  Q = [e1r rr - e1i ri, e1i rr + e1r ri], gold = o
template <int W>
__global__ void __launch_bounds__(256)
    k_complex_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                           const int32_t* __restrict__ X, int64_t n, int side, float* __restrict__ Q,
                           float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const int kept = side == 0 ? o : s, gold = side == 0 ? s : o;
    const float* ek = codes + (size_t)kept * d;
    const float* rr = rel + (size_t)r * d;
    const float* eg = codes + (size_t)gold * d;
    float* q = Q + (size_t)t * d;
    float e = 0.f;
    for (int k = lane * W; k < h; k += 32 * W) {
      float kr[W], ki[W], br[W], bi[W], gr[W], gi[W], qr[W], qi[W];
      Vec<W>::load(ek + k, kr), Vec<W>::load(ek + h + k, ki);
      Vec<W>::load(rr + k, br), Vec<W>::load(rr + h + k, bi);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        if (side == 0) {
          qr[j] = fmaf(br[j], kr[j], bi[j] * ki[j]);
          qi[j] = fmaf(br[j], ki[j], -bi[j] * kr[j]);
        } else {
          qr[j] = fmaf(kr[j], br[j], -ki[j] * bi[j]);
          qi[j] = fmaf(ki[j], br[j], kr[j] * bi[j]);
        }
      }
      Vec<W>::store(q + k, qr), Vec<W>::store(q + h + k, qi);
      if (gold_sig) {   // the top-k path asks for the query rows only: the predicted column of X is not read
        Vec<W>::load(eg + k, gr), Vec<W>::load(eg + h + k, gi);
#pragma unroll
        for (int j = 0; j < W; ++j) {
          e = fmaf(qr[j], gr[j], e);
          e = fmaf(qi[j], gi[j], e);
        }
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
// The energy of complex.py:38-41, (hr rr) . tr + (hi rr) . ti + (hr ri) . ti - (hi ri) . tr, is linear in the
// relation row [rr | ri]:  e = rr . (hr tr + hi ti) + ri . (hr ti - hi tr),  so
//   Q = [hr tr + hi ti, hr ti - hi tr],  gold = r,  gold_sig[t] = sigmoid(<Q[t], rel[r]>)
// (gold_sig == nullptr: Q only; the relation column of X is then not read).
template <int W>
__global__ void __launch_bounds__(256)
    k_complex_relation_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                               const int32_t* __restrict__ X, int64_t n, float* __restrict__ Q,
                               float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), o = __ldg(X + 3 * t + 2);
    const int r = gold_sig ? __ldg(X + 3 * t + 1) : 0;
    const float* eh = codes + (size_t)s * d;
    const float* et = codes + (size_t)o * d;
    const float* rr = rel + (size_t)r * d;
    float* q = Q + (size_t)t * d;
    float e = 0.f;
    for (int k = lane * W; k < h; k += 32 * W) {
      float hr[W], hi[W], tr[W], ti[W], br[W], bi[W], qr[W], qi[W];
      Vec<W>::load(eh + k, hr), Vec<W>::load(eh + h + k, hi);
      Vec<W>::load(et + k, tr), Vec<W>::load(et + h + k, ti);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        qr[j] = fmaf(hr[j], tr[j], hi[j] * ti[j]);
        qi[j] = fmaf(hr[j], ti[j], -hi[j] * tr[j]);
      }
      Vec<W>::store(q + k, qr), Vec<W>::store(q + h + k, qi);
      if (gold_sig) {
        Vec<W>::load(rr + k, br), Vec<W>::load(rr + h + k, bi);
#pragma unroll
        for (int j = 0; j < W; ++j) {
          e = fmaf(qr[j], br[j], e);
          e = fmaf(qi[j], bi[j], e);
        }
      }
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = r;
    }
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

int launch_complex_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc) return rc;
  if (N == 0) return RGCN_OK;
  if (d % 8 == 0)
    k_complex_fwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, loss_out);
  else
    k_complex_fwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, loss_out);
  rc = check_launch("k_complex_fwd");
  if (rc) return rc;
  k_complex_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_complex_finalize");
}

int launch_complex_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                            const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                            const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq,
                            cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  if (d % 8 == 0)
    k_complex_bwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                            g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  else
    k_complex_bwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                            g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_complex_bwd");
}

int launch_complex_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                                float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  if (d % 8 == 0)
    k_complex_rank_prepare<4><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_sig,
                                                                     gold_col);
  else
    k_complex_rank_prepare<2><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_sig,
                                                                     gold_col);
  return check_launch("k_complex_rank_prepare");
}

int launch_complex_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                                    float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  if (d % 8 == 0)
    k_complex_relation_prepare<4><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, Q, gold_sig, gold_col);
  else
    k_complex_relation_prepare<2><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, Q, gold_sig, gold_col);
  return check_launch("k_complex_relation_prepare");
}
