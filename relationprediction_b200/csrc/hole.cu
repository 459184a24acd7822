// hole.cu -- HolE (Nickel, Rosasco, Poggio; AAAI 2016) on the real Fourier basis, for sm_90a: the basis, the triple
// scorer, loss and backward, and the query rows and query backward that put HolE on the DistMult scoring GEMMs (ranks,
// top-k, 1-N).  Semantics in DESIGN.md section 1.  The energy of (s, r, o) is
//   E = sum_k r_k [h * t]_k,   [h * t]_k = sum_i h_i t_{(i + k) mod d},
// O(d^2) per triple written out.  In the orthonormal real DFT basis x~ = x U (columns: DC, Nyquist, then (cos, -sin)
// pairs of frequencies 1 .. d/2 - 1) it is a ComplEx-type product, O(d) per triple:
//   E = sqrt(d) (h~0 r~0 t~0 + h~1 r~1 t~1) + sqrt(d/2) sum_f Re(conj(h~f r~f) t~f).
// Every kernel here except k_hole_basis works on transformed tables; the transforms x U and g U^T are GEMMs on the
// library's 3xTF32 kernels (api.cu, rgcn_hole_transform).  The energy is linear in each row, so every all-candidate
// query is one query row against a table: w (h r) against the objects, w conj(r) t against the subjects, w conj(h) t
// against the relations (triple_rows.cuh: hole_mul, hole_cmul).
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

// U [d, d] row-major, U[k][c]: column 0 = 1/sqrt(d), column 1 = (-1)^k / sqrt(d), columns 2f and 2f+1 =
// sqrt(2/d) (cos, -sin)(2 pi f k / d).  Formed in double precision and rounded once; the angle's argument f k is
// reduced mod d exactly first.
__global__ void __launch_bounds__(256) k_hole_basis(int d, float* __restrict__ U) {
  const int64_t count = (int64_t)d * d;
  const double s0 = 1.0 / sqrt((double)d), s1 = sqrt(2.0 / (double)d);
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < count; j += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(j / d), c = (int)(j % d);
    double v;
    if (c == 0) {
      v = s0;
    } else if (c == 1) {
      v = (k & 1) ? -s0 : s0;
    } else {
      const int64_t m = (int64_t)(c >> 1) * k % d;
      double sn, cs;
      sincospi(2.0 * (double)m / (double)d, &sn, &cs);
      v = (c & 1) ? -s1 * sn : s1 * cs;
    }
    U[j] = (float)v;
  }
}

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the three rows
__global__ void __launch_bounds__(256)
    k_hole_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
               int64_t N, const float* __restrict__ Y, float* __restrict__ energies, float* __restrict__ loss_acc) {
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh_l[warp] = sh_q[warp] = 0.0;
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float e = 0.f, q = 0.f;
    HolERows::partial(codes, rel, d, s, r, o, lane, e, q);
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

__global__ void k_hole_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// With g = dL/dE:  dh = g w conj(r) t,  dt = g w (h r),  dr = g w conj(h) t;  plus c_reg x on the three rows (the L2
// term).
__global__ void __launch_bounds__(256)
    k_hole_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
               int64_t N, const float* __restrict__ Y, const float* __restrict__ energies, float g_loss_over_n,
               float c_reg, const float* __restrict__ g_scale, const float* __restrict__ g_energy,
               float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  float w0, w1;
  hole_weights(d, w0, w1);
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
      const bool first = i == 0;
      const float4 da = axpy4(gx, hole_cmul(b, c, first, w0, w1), scale4(c_reg, a));
      const float4 dc = axpy4(gx, hole_mul(a, b, first, w0, w1), scale4(c_reg, c));
      const float4 db = axpy4(gx, hole_cmul(a, c, first, w0, w1), scale4(c_reg, b));
      red4(g1 + 4 * i, da);
      red4(gr + 4 * i, db);
      red4(g2 + 4 * i, dc);
      slice_sq += hole_dot(db, db, 0.f);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- query rows for the scoring GEMMs ------------------------------------------------------------------------------
// One warp per query t = (s, r, o).  side 1 (objects corrupted): Q = w (h r), kept s, gold o; side 0 (subjects
// corrupted): Q = w conj(r) t, kept o, gold s.  With gold_sig, also gold_sig[t] = sigmoid(<Q, codes[gold]>) from the
// float32 Q just stored (k_rank_prepare's rule) and gold_col[t] = gold; gold_sig == nullptr: Q only, the predicted
// column of X is not read.
__global__ void __launch_bounds__(256)
    k_hole_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                        const int32_t* __restrict__ X, int64_t n, int side, float* __restrict__ Q,
                        float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  float w0, w1;
  hole_weights(d, w0, w1);
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const int kept = side == 0 ? o : s, gold = side == 0 ? s : o;
    const float4* ek = reinterpret_cast<const float4*>(codes + (size_t)kept * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* eg = reinterpret_cast<const float4*>(codes + (size_t)gold * d);
    float4* q = reinterpret_cast<float4*>(Q + (size_t)t * d);
    float e = 0.f;
    for (int i = lane; i < d4; i += 32) {
      const float4 k = __ldg(ek + i), b = __ldg(rr + i);
      const float4 p = side == 0 ? hole_cmul(b, k, i == 0, w0, w1) : hole_mul(k, b, i == 0, w0, w1);
      q[i] = p;
      if (gold_sig) e = hole_dot(p, __ldg(eg + i), e);
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = gold;
    }
  }
}

// Pair queries (h, ?, t): Q = w conj(h) t, scored against the relation rows.  gold_sig[t] = sigmoid(<Q, rel[r]>),
// gold_col[t] = r (gold_sig == nullptr: Q only; the relation column of X is then not read).
__global__ void __launch_bounds__(256)
    k_hole_relation_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                            const int32_t* __restrict__ X, int64_t n, float* __restrict__ Q,
                            float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  float w0, w1;
  hole_weights(d, w0, w1);
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), o = __ldg(X + 3 * t + 2);
    const int r = gold_sig ? __ldg(X + 3 * t + 1) : 0;
    const float4* eh = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* et = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    float4* q = reinterpret_cast<float4*>(Q + (size_t)t * d);
    float e = 0.f;
    for (int i = lane; i < d4; i += 32) {
      const float4 p = hole_cmul(__ldg(eh + i), __ldg(et + i), i == 0, w0, w1);
      q[i] = p;
      if (gold_sig) e = hole_dot(p, __ldg(rr + i), e);
    }
    e = warp_sum(e);
    if (lane == 0 && gold_sig) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = r;
    }
  }
}

// 1-N query backward, queries (anchor k, r, side) of one side, dQ [n, d]:
//   side 1: Q = w (k r)        ->  dk = w conj(r) dQ,  dr = w conj(k) dQ
//   side 0: Q = w conj(r) k    ->  dk = w (r dQ),      dr = w conj(dQ) k
// each + c k (c r), the L2 term.
__global__ void __launch_bounds__(256)
    k_hole_query_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                     const int32_t* __restrict__ X, int64_t n, int side, const float* __restrict__ dQ,
                     const float* __restrict__ g_scale, float c_reg, float* __restrict__ dcodes,
                     float* __restrict__ drel) {
  if (g_scale) c_reg *= __ldg(g_scale + 1);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  float w0, w1;
  hole_weights(d, w0, w1);
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int a = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    const float4* ek = reinterpret_cast<const float4*>(codes + (size_t)a * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* gq = reinterpret_cast<const float4*>(dQ + (size_t)t * d);
    float* gk = dcodes + (size_t)a * d;
    float* gr = drel + (size_t)r * d;
    for (int i = lane; i < d4; i += 32) {
      const float4 k = __ldg(ek + i), b = __ldg(rr + i), g = __ldg(gq + i);
      const bool first = i == 0;
      const float4 dk = side == 0 ? hole_mul(b, g, first, w0, w1) : hole_cmul(b, g, first, w0, w1);
      const float4 db = side == 0 ? hole_cmul(g, k, first, w0, w1) : hole_cmul(k, g, first, w0, w1);
      red4(gk + 4 * i, axpy4(c_reg, k, dk));
      red4(gr + 4 * i, axpy4(c_reg, b, db));
    }
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) { return (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, 132 * 8)); }

}  // namespace

int launch_hole_basis(int d, float* U, cudaStream_t st) {
  const int64_t count = (int64_t)d * d;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((count + 255) / 256, 132 * 8));
  k_hole_basis<<<blocks, 256, 0, st>>>(d, U);
  return check_launch("k_hole_basis");
}

int launch_hole_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                        float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc || N == 0) return rc;
  k_hole_fwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, loss_out);
  rc = check_launch("k_hole_fwd");
  if (rc) return rc;
  k_hole_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_hole_finalize");
}

int launch_hole_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                         const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                         const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  k_hole_bwd<<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                    g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_hole_bwd");
}

int launch_hole_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                             float* Q, float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_hole_rank_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_sig, gold_col);
  return check_launch("k_hole_rank_prepare");
}

int launch_hole_relation_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* Q,
                                 float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_hole_relation_prepare<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, Q, gold_sig, gold_col);
  return check_launch("k_hole_relation_prepare");
}

int launch_hole_query_bwd(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                          const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                          cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_hole_query_bwd<<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, dQ, g_scale, c_reg, dcodes,
                                                          drel);
  return check_launch("k_hole_query_bwd");
}
