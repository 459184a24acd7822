// variational.cu -- the reparameterised code of the variational encoders (extras/variational_encoding.py:14-31):
//
//   z = mu + exp(l) eps,   KL = -0.0005 sum over all V x w elements of (1 + 2 l - mu^2 - exp(2 l))
//
// with l = log sigma and eps ~ N(0, 1) drawn by the caller.  Two variants:
//   embedding  mu = W_mu, l = W_sigma ([V, w] free tables, model_builder.py:43-69): forward and backward are one
//              element-wise pass each (k_var_emb_fwd, k_var_emb_bwd).
//   gcn        mu = H W_mu + b_mu, l = H W_sigma + b_sigma (model_builder.py:219-238): the forward is one 3xTF32 GEMM
//              with the interleaved weight W_int and the variational epilogue (k_gemm_tf32x3<3>, gemm_tf32x3.cu),
//              which also keeps P = (mu, l) interleaved [V, 2w] for the backward.  The backward turns dz, g = dKL
//              and P into dP (k_var_prologue), then dW_int = H^T dP and dH = dP W_int^T on the GEMM kernels.
// Gradients, g the incoming gradient of the KL term:
//   dmu = dz + 0.001 g mu,   dl = dz exp(l) eps + 0.001 g (exp(2 l) - 1).
// g is read from device memory, so the backward needs no host synchronisation.  Every sum (the KL, db_mu, db_sigma)
// is formed in a fixed order from per-block parts, so it is bitwise repeatable.  expf is not clamped (neither is the
// reference's tf.exp).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.cuh"

namespace {

constexpr int EMB_THREADS = 256;
constexpr int64_t EMB_MAX_BLOCKS = 528;   // fixed part count (4 x 132): the KL does not depend on the device
constexpr int PRO_TX = 32;                // column quads (4 elements = 8 P columns) per CTA
constexpr int PRO_TY = 8;                 // row lanes per CTA
constexpr int64_t PRO_MAX_PARTS = 256;    // row blocks of the prologue = parts of the db column sums

__device__ __forceinline__ float kl_term(float mu, float l) { return 1.f + 2.f * l - mu * mu - expf(2.f * l); }

// one float per block: the warp sums (shuffle tree), then warp 0 adds the warps in order
__device__ __forceinline__ void block_part(float s, float* part) {
  __shared__ float warp_sum[EMB_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < EMB_THREADS / 32; ++k) t += warp_sum[k];
    part[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(EMB_THREADS)
    k_var_emb_fwd(const float4* __restrict__ mu, const float4* __restrict__ ls, const float4* __restrict__ eps,
                  int64_t n4, float4* __restrict__ z, float* __restrict__ kl_part) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)EMB_THREADS + threadIdx.x; i < n4; i += (int64_t)gridDim.x * EMB_THREADS) {
    const float4 m = __ldg(mu + i), l = __ldg(ls + i), e = __ldg(eps + i);
    z[i] = make_float4(m.x + expf(l.x) * e.x, m.y + expf(l.y) * e.y, m.z + expf(l.z) * e.z, m.w + expf(l.w) * e.w);
    s += kl_term(m.x, l.x) + kl_term(m.y, l.y) + kl_term(m.z, l.z) + kl_term(m.w, l.w);
  }
  block_part(s, kl_part);
}

// kl = -0.0005 * sum of the parts: each thread sums a strided set in double, then a shared-memory tree
__global__ void __launch_bounds__(256) k_var_kl_reduce(const float* __restrict__ part, int64_t n, float* __restrict__ kl) {
  __shared__ double s[256];
  double t = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += 256) t += (double)part[i];
  s[threadIdx.x] = t;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) kl[0] = (float)(-0.0005 * s[0]);
}

__global__ void __launch_bounds__(256)
    k_var_emb_bwd(const float4* __restrict__ mu, const float4* __restrict__ ls, const float4* __restrict__ eps,
                  const float4* __restrict__ dz, const float* __restrict__ g_kl, int64_t n4, float4* __restrict__ dmu,
                  float4* __restrict__ dls) {
  const float g = 0.001f * __ldg(g_kl);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 m = __ldg(mu + i), l = __ldg(ls + i), e = __ldg(eps + i), y = __ldg(dz + i);
    __stcs(dmu + i, make_float4(y.x + g * m.x, y.y + g * m.y, y.z + g * m.z, y.w + g * m.w));
    __stcs(dls + i, make_float4(y.x * expf(l.x) * e.x + g * (expf(2.f * l.x) - 1.f),
                                y.y * expf(l.y) * e.y + g * (expf(2.f * l.y) - 1.f),
                                y.z * expf(l.z) * e.z + g * (expf(2.f * l.z) - 1.f),
                                y.w * expf(l.w) * e.w + g * (expf(2.f * l.w) - 1.f)));
  }
}

// gcn backward prologue.  CTA (x, y): element quads q = 32 x + tx (P columns 8q .. 8q + 7), rows y * 8 + ty stepping
// by gridDim.y * 8.  Writes dP and keeps its column sums in registers; the CTA folds its 8 row lanes in order and
// writes one part row col_part[y, :].
__global__ void __launch_bounds__(PRO_TX* PRO_TY)
    k_var_prologue(const float4* __restrict__ P, const float4* __restrict__ eps, const float4* __restrict__ dz,
                   const float* __restrict__ g_kl, int64_t V, int w4, float4* __restrict__ dP,
                   float* __restrict__ col_part) {
  __shared__ float4 part[PRO_TY][PRO_TX][2];
  const int tx = threadIdx.x % PRO_TX, ty = threadIdx.x / PRO_TX;
  const int q = blockIdx.x * PRO_TX + tx;
  const float g = 0.001f * __ldg(g_kl);
  float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
  if (q < w4) {
    for (int64_t r = (int64_t)blockIdx.y * PRO_TY + ty; r < V; r += (int64_t)gridDim.y * PRO_TY) {
      const int64_t i = r * w4 + q;
      const float4 p0 = __ldg(P + 2 * i), p1 = __ldg(P + 2 * i + 1);   // (mu, l) of elements 4q .. 4q + 3
      const float4 e = __ldg(eps + i), y = __ldg(dz + i);
      float4 o0, o1;
      o0.x = y.x + g * p0.x;  o0.y = y.x * expf(p0.y) * e.x + g * (expf(2.f * p0.y) - 1.f);
      o0.z = y.y + g * p0.z;  o0.w = y.y * expf(p0.w) * e.y + g * (expf(2.f * p0.w) - 1.f);
      o1.x = y.z + g * p1.x;  o1.y = y.z * expf(p1.y) * e.z + g * (expf(2.f * p1.y) - 1.f);
      o1.z = y.w + g * p1.z;  o1.w = y.w * expf(p1.w) * e.w + g * (expf(2.f * p1.w) - 1.f);
      dP[2 * i] = o0;         // read again by both GEMMs that follow: plain stores
      dP[2 * i + 1] = o1;
      s0.x += o0.x; s0.y += o0.y; s0.z += o0.z; s0.w += o0.w;
      s1.x += o1.x; s1.y += o1.y; s1.z += o1.z; s1.w += o1.w;
    }
  }
  part[ty][tx][0] = s0;
  part[ty][tx][1] = s1;
  __syncthreads();
  if (ty == 0 && q < w4) {
#pragma unroll
    for (int k = 1; k < PRO_TY; ++k) {
      const float4 a = part[k][tx][0], b = part[k][tx][1];
      s0.x += a.x; s0.y += a.y; s0.z += a.z; s0.w += a.w;
      s1.x += b.x; s1.y += b.y; s1.z += b.z; s1.w += b.w;
    }
    float4* o = reinterpret_cast<float4*>(col_part + (size_t)blockIdx.y * 8 * w4) + 2 * q;
    o[0] = s0;
    o[1] = s1;
  }
}

__global__ void k_var_colsum_finish(const float* __restrict__ col_part, int64_t parts, int w,
                                    float* __restrict__ db_mu, float* __restrict__ db_sigma) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * w) return;
  float s = 0.f;
  for (int64_t p = 0; p < parts; ++p) s += col_part[p * 2 * w + c];
  ((c & 1) ? db_sigma : db_mu)[c >> 1] = s;
}

__global__ void k_var_deinterleave(const float2* __restrict__ dWint, int64_t n, float* __restrict__ dWmu,
                                   float* __restrict__ dWsig) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float2 v = __ldg(dWint + i);
    dWmu[i] = v.x;
    dWsig[i] = v.y;
  }
}

unsigned grid_for(int64_t n, int threads) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 132 * 8));
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

}  // namespace

int64_t var_emb_kl_parts(int64_t V, int w) {
  const int64_t n4 = V * w / 4;
  return std::max<int64_t>(1, std::min<int64_t>((n4 + EMB_THREADS - 1) / EMB_THREADS, EMB_MAX_BLOCKS));
}

int launch_var_emb_forward(const float* Wmu, const float* Wsig, const float* eps, int64_t V, int w, float* z,
                           float* kl_part, cudaStream_t st) {
  const int64_t n4 = V * w / 4;
  k_var_emb_fwd<<<(unsigned)var_emb_kl_parts(V, w), EMB_THREADS, 0, st>>>(
      reinterpret_cast<const float4*>(Wmu), reinterpret_cast<const float4*>(Wsig),
      reinterpret_cast<const float4*>(eps), n4, reinterpret_cast<float4*>(z), kl_part);
  return check_launch("k_var_emb_fwd");
}

int launch_var_kl_reduce(const float* kl_part, int64_t n, float* kl, cudaStream_t st) {
  k_var_kl_reduce<<<1, 256, 0, st>>>(kl_part, n, kl);
  return check_launch("k_var_kl_reduce");
}

int launch_var_emb_backward(const float* Wmu, const float* Wsig, const float* eps, const float* dz, const float* g_kl,
                            int64_t V, int w, float* dWmu, float* dWsig, cudaStream_t st) {
  const int64_t n4 = V * w / 4;
  if (n4 == 0) return RGCN_OK;
  k_var_emb_bwd<<<grid_for(n4, 256), 256, 0, st>>>(
      reinterpret_cast<const float4*>(Wmu), reinterpret_cast<const float4*>(Wsig),
      reinterpret_cast<const float4*>(eps), reinterpret_cast<const float4*>(dz), g_kl, n4,
      reinterpret_cast<float4*>(dWmu), reinterpret_cast<float4*>(dWsig));
  return check_launch("k_var_emb_bwd");
}

int64_t var_colsum_parts(int64_t V) {
  return std::max<int64_t>(1, std::min<int64_t>((V + PRO_TY - 1) / PRO_TY, PRO_MAX_PARTS));
}

int launch_var_prologue(const float* P, const float* eps, const float* dz, const float* g_kl, int64_t V, int w,
                        float* dP, float* col_part, cudaStream_t st) {
  const int w4 = w / 4;
  const dim3 grid((unsigned)((w4 + PRO_TX - 1) / PRO_TX), (unsigned)var_colsum_parts(V));
  k_var_prologue<<<grid, PRO_TX * PRO_TY, 0, st>>>(
      reinterpret_cast<const float4*>(P), reinterpret_cast<const float4*>(eps), reinterpret_cast<const float4*>(dz),
      g_kl, V, w4, reinterpret_cast<float4*>(dP), col_part);
  return check_launch("k_var_prologue");
}

int launch_var_colsum_finish(const float* col_part, int64_t parts, int w, float* db_mu, float* db_sigma,
                             cudaStream_t st) {
  k_var_colsum_finish<<<(unsigned)((2 * w + 255) / 256), 256, 0, st>>>(col_part, parts, w, db_mu, db_sigma);
  return check_launch("k_var_colsum_finish");
}

int launch_var_deinterleave(const float* dWint, int d, int w, float* dWmu, float* dWsig, cudaStream_t st) {
  const int64_t n = (int64_t)d * w;
  k_var_deinterleave<<<grid_for(n, 256), 256, 0, st>>>(reinterpret_cast<const float2*>(dWint), n, dWmu, dWsig);
  return check_launch("k_var_deinterleave");
}
