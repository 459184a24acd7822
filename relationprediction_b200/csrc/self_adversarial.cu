// self_adversarial.cu -- self-adversarial negative sampling (Sun et al., RotatE, ICLR 2019) for the DistMult, ComplEx,
// RotatE, TransE, QuatE and HolE decoders, sm_90a: the forward of the objective, which also writes each triple's energy
// gradient.
//
// The fed triples follow the negative sampler's layout (auxilliaries.py:13-33): for N = n (K + 1) rows, rows 0..n-1
// are the positives and row i + n j (j = 1..K) is the j-th corruption of positive i.  With s_i the positive's energy
// and s_ij its corruptions',
//   p_ij = exp(alpha s_ij) / sum_j' exp(alpha s_ij')        (constants: no gradient flows through p)
//   L    = 1 / (2n) sum_i [ softplus(-s_i) + sum_j p_ij softplus(s_ij) ]
// so dL/ds_i = -sigmoid(-s_i) / (2n) and dL/ds_ij = p_ij sigmoid(s_ij) / (2n): the per-triple coefficients the
// existing scorer backward (distmult.cu / complex.cu) takes as its upstream energy gradient.  No scatter kernel here.
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

// max(x, 0) + log1p(exp(-|x|)): finite for any finite x
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// One warp owns one group i: the positive (row i) and its K corruptions (rows i + n j).  Pass 1 scores the K + 1
// triples in order with the decoder's row arithmetic (Rows) and keeps a running max m and sum S of exp(alpha s - m)
// over the corruptions; lane j % 32 stores energy j.  Pass 2 walks the group in strides of 32 -- so any K works -- and
// every lane reads back only the energies it stored itself, forms p, the coefficient and its loss terms.  The loss and
// the squared norms of the group's rows go to one part each per group, for a reduction in a fixed order.  `rows` is
// the decoder's functor (RotateRows and TransERows carry gamma); it comes last so the other parameters keep their
// offsets.
template <class Rows>
__global__ void __launch_bounds__(256)
    k_selfadv_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                  int64_t n, int K, float alpha, float inv_2n, float* energies, float* __restrict__ coef,
                  float* __restrict__ loss_part, float* __restrict__ reg_part, Rows rows) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * 8 + warp; i < n; i += (int64_t)gridDim.x * 8) {
    float m = -INFINITY, S = 0.f, q = 0.f;
    for (int j = 0; j <= K; ++j) {
      const int64_t t = i + n * j;
      const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
      float e = 0.f;
      rows.partial(codes, rel, d, s, r, o, lane, e, q);
      e = warp_sum(e);   // the xor butterfly leaves the same sum in every lane
      if (lane == (j & 31)) energies[t] = e;
      if (j > 0) {
        const float a = alpha * e;
        const float m_new = fmaxf(m, a);
        S = S * expf(m - m_new) + expf(a - m_new);
        m = m_new;
      }
    }
    const float inv_S = 1.f / S;   // S >= 1: the largest corruption contributes exp(0)
    float l = 0.f;
    for (int j = lane; j <= K; j += 32) {
      const int64_t t = i + n * j;
      const float e = energies[t];   // stored by this lane in pass 1
      float c;
      if (j == 0) {
        c = -sigmoid(-e) * inv_2n;
        l += softplus(-e);
      } else {
        const float p = expf(alpha * e - m) * inv_S;
        c = p * sigmoid(e) * inv_2n;
        l += p * softplus(e);
      }
      coef[t] = c;
    }
    l = warp_sum(l);
    const float qg = warp_sum(q);
    if (lane == 0) {
      loss_part[i] = l;
      reg_part[i] = qg;
    }
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

}  // namespace

int launch_self_adversarial_forward(int decoder, const float* codes, const float* rel, int d, const int32_t* X,
                                    int64_t N, int K, float alpha, float gamma, float* energies, float* coef,
                                    float* loss_out, float* parts, cudaStream_t st) {
  if (N == 0) return rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  const int64_t n = N / (K + 1);
  float* loss_part = parts;
  float* reg_part = parts + n;
  const int blocks = (int)std::min<int64_t>((n + 7) / 8, 132 * 8);
  const float inv_2n = (float)(0.5 / (double)n);
  if (decoder == SELFADV_DISTMULT)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          DistMultRows{});
  else if (decoder == SELFADV_COMPLEX && d % 8 == 0)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          ComplexRows<4>{});
  else if (decoder == SELFADV_COMPLEX)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          ComplexRows<2>{});
  else if (decoder == SELFADV_QUATE)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          QuatERows{});
  else if (decoder == SELFADV_HOLE)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          HolERows{});
  else if (decoder == SELFADV_TRANSE)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          TransERows<4>{gamma});
  else if (d % 8 == 0)
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          RotateRows<4>{gamma});
  else
    k_selfadv_fwd<<<blocks, 256, 0, st>>>(codes, rel, d, X, n, K, alpha, inv_2n, energies, coef, loss_part, reg_part,
                                          RotateRows<2>{gamma});
  int rc = check_launch("k_selfadv_fwd");
  if (rc) return rc;
  // loss[0] = (sum of the loss parts) / (2n), loss[1] = (sum of the squared norms) / (N d): the NegativeSampling L2 term
  return launch_onen_loss_reduce(loss_part, n, reg_part, n, 0.5 / (double)n, 1.0 / ((double)N * (double)d), loss_out,
                                 st);
}
