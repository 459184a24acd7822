// onen.cu -- 1-N training of the DistMult and ComplEx decoders, sm_90a: the label rows, the L2 term, the fixed-order
// loss reduction and the query backward.  The energies, loss terms and energy gradients come from the scoring GEMM's
// BCE epilogue (k_gemm_tf32x3<5>), the query rows from the rank prepare kernels (distmult.cu / complex.cu).
//
// The queries of one launch are triples X[t] = (anchor, r, anchor) that share one side: side 1 (object queries,
// (anchor, r, ?)) and side 0 (subject queries, (?, r, anchor)).  This is the form the rank prepare kernels read: they
// take the kept entity from column 0 (side 1) or column 2 (side 0).
#include <cuda_runtime.h>

#include <algorithm>

#include "kernels.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

// One warp per query: zero its bit row, find its key in the sorted CSR keys, set the bits of its entities.
__global__ void __launch_bounds__(256)
    k_onen_labels(const int64_t* __restrict__ keys, const int64_t* __restrict__ offsets,
                  const int32_t* __restrict__ entities, int64_t n_keys, const int32_t* __restrict__ X, int64_t n,
                  int side, int V, int words, uint32_t* __restrict__ bits) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    uint32_t* row = bits + (size_t)t * words;
    for (int w = lane; w < words; w += 32) row[w] = 0u;
    __syncwarp();
    const int anchor = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    const int64_t key = ((int64_t)2 * r + side) * V + anchor;
    int64_t lo = 0, hi = n_keys;   // first index with keys[i] >= key
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(keys + mid) < key) lo = mid + 1; else hi = mid;
    }
    if (lo < n_keys && __ldg(keys + lo) == key) {
      for (int64_t i = __ldg(offsets + lo) + lane; i < __ldg(offsets + lo + 1); i += 32) {
        const int e = __ldg(entities + i);
        atomicOr(row + (e >> 5), 1u << (e & 31));
      }
    }
  }
}

constexpr int64_t REG_MAX_PARTS = 132 * 8;

// reg_part[block] = sum over the block's queries of |codes[anchor]|^2 + |rel[r]|^2 (a fixed assignment of queries to
// blocks for a given n, so the parts are repeatable)
__global__ void __launch_bounds__(256)
    k_onen_reg(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
               int64_t n, float* __restrict__ reg_part) {
  __shared__ double sh[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  double acc = 0.0;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const float4* ea = reinterpret_cast<const float4*>(codes + (size_t)__ldg(X + 3 * t) * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)__ldg(X + 3 * t + 1) * d);
    float q = 0.f;
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(ea + i), b = __ldg(rr + i);
      q += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
      q += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
    }
    acc += (double)warp_sum(q);
  }
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += sh[w];
    reg_part[blockIdx.x] = (float)s;
  }
}

__global__ void __launch_bounds__(256)
    k_onen_loss_reduce(const float* __restrict__ loss_part, int64_t n_loss, const float* __restrict__ reg_part,
                       int64_t n_reg, double inv_nv, double inv_nd, float* __restrict__ loss) {
  __shared__ double s[2][256];
  double a = 0.0, b = 0.0;
  for (int64_t i = threadIdx.x; i < n_loss; i += 256) a += (double)loss_part[i];
  for (int64_t i = threadIdx.x; i < n_reg; i += 256) b += (double)reg_part[i];
  s[0][threadIdx.x] = a;
  s[1][threadIdx.x] = b;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) {
      s[0][threadIdx.x] += s[0][threadIdx.x + h];
      s[1][threadIdx.x] += s[1][threadIdx.x + h];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    loss[0] = (float)(inv_nv * s[0][0]);
    loss[1] = (float)(inv_nd * s[1][0]);
  }
}

__device__ __forceinline__ void red4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// DistMult: Q = k (.) r  ->  dk = dQ (.) r + c k,  dr = dQ (.) k + c r.  dQ null: the L2 term only (any decoder).
__global__ void __launch_bounds__(256)
    k_onen_query_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                     const int32_t* __restrict__ X, int64_t n, const float* __restrict__ dQ,
                     const float* __restrict__ g_scale, float c_reg, float* __restrict__ dcodes,
                     float* __restrict__ drel) {
  if (g_scale) c_reg *= __ldg(g_scale + 1);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int a = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    const float4* ek = reinterpret_cast<const float4*>(codes + (size_t)a * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* gq = dQ ? reinterpret_cast<const float4*>(dQ + (size_t)t * d) : nullptr;
    float* gk = dcodes + (size_t)a * d;
    float* gr = drel + (size_t)r * d;
    for (int i = lane; i < d4; i += 32) {
      const float4 k = __ldg(ek + i), b = __ldg(rr + i), g = gq ? __ldg(gq + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      red4(gk + 4 * i, make_float4(fmaf(g.x, b.x, c_reg * k.x), fmaf(g.y, b.y, c_reg * k.y),
                                   fmaf(g.z, b.z, c_reg * k.z), fmaf(g.w, b.w, c_reg * k.w)));
      red4(gr + 4 * i, make_float4(fmaf(g.x, k.x, c_reg * b.x), fmaf(g.y, k.y, c_reg * b.y),
                                   fmaf(g.z, k.z, c_reg * b.z), fmaf(g.w, k.w, c_reg * b.w)));
    }
  }
}

template <int W>
struct Vec;
template <>
struct Vec<4> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  }
  __device__ __forceinline__ static void red(float* p, const float (&v)[4]) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]),
                 "f"(v[3])
                 : "memory");
  }
};
template <>
struct Vec<2> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[2]) {
    const float2 t = __ldg(reinterpret_cast<const float2*>(p));
    v[0] = t.x, v[1] = t.y;
  }
  __device__ __forceinline__ static void red(float* p, const float (&v)[2]) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
  }
};

// ComplEx, rows [real | imaginary], kept entity k, relation b, dQ = (gr, gi):
//   side 1: Q = [kr br - ki bi, ki br + kr bi]  ->  dk = [gr br + gi bi, gi br - gr bi],  db = [gr kr + gi ki, gi kr - gr ki]
//   side 0: Q = [br kr + bi ki, br ki - bi kr]  ->  dk = [gr br - gi bi, gr bi + gi br],  db = [gr kr + gi ki, gr ki - gi kr]
// each + c k (c b), the L2 term.  W = 4: d % 8 == 0 (float4 halves), W = 2: d % 8 == 4.
template <int W>
__global__ void __launch_bounds__(256)
    k_onen_complex_query_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                             const int32_t* __restrict__ X, int64_t n, int side, const float* __restrict__ dQ,
                             const float* __restrict__ g_scale, float c_reg, float* __restrict__ dcodes,
                             float* __restrict__ drel) {
  if (g_scale) c_reg *= __ldg(g_scale + 1);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  const float sg = side == 0 ? -1.f : 1.f;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int a = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    const float* ek = codes + (size_t)a * d;
    const float* rr = rel + (size_t)r * d;
    const float* gq = dQ + (size_t)t * d;
    float* gk = dcodes + (size_t)a * d;
    float* gb = drel + (size_t)r * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float kr[W], ki[W], br[W], bi[W], gr[W], gi[W];
      Vec<W>::load(ek + k, kr), Vec<W>::load(ek + h + k, ki);
      Vec<W>::load(rr + k, br), Vec<W>::load(rr + h + k, bi);
      Vec<W>::load(gq + k, gr), Vec<W>::load(gq + h + k, gi);
      float dkr[W], dki[W], dbr[W], dbi[W];
#pragma unroll
      for (int j = 0; j < W; ++j) {
        // side 1: bi enters Q with sign +, side 0 with sign - (Q is conj(b) k instead of k b)
        const float sbi = sg * bi[j];
        dkr[j] = fmaf(gr[j], br[j], fmaf(gi[j], sbi, c_reg * kr[j]));
        dki[j] = fmaf(gi[j], br[j], fmaf(-gr[j], sbi, c_reg * ki[j]));
        dbr[j] = fmaf(gr[j], kr[j], fmaf(gi[j], ki[j], c_reg * br[j]));
        dbi[j] = fmaf(sg, fmaf(gi[j], kr[j], -gr[j] * ki[j]), c_reg * bi[j]);
      }
      Vec<W>::red(gk + k, dkr), Vec<W>::red(gk + h + k, dki);
      Vec<W>::red(gb + k, dbr), Vec<W>::red(gb + h + k, dbi);
    }
  }
}

// dst = g_scale[0] * src over count4 float4s
__global__ void __launch_bounds__(256)
    k_onen_scale(const float4* __restrict__ src, const float* __restrict__ g_scale, int64_t count4,
                 float4* __restrict__ dst) {
  const float g = __ldg(g_scale);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(src + i);
    dst[i] = make_float4(g * v.x, g * v.y, g * v.z, g * v.w);
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_rows(int64_t n) {
  int64_t b = (n + 7) / 8;
  if (b > REG_MAX_PARTS) b = REG_MAX_PARTS;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

int launch_onen_labels(const int64_t* keys, const int64_t* offsets, const int32_t* entities, int64_t n_keys,
                       const int32_t* X, int64_t n, int side, int V, int words, uint32_t* bits, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_onen_labels<<<blocks_for_rows(n), 256, 0, st>>>(keys, offsets, entities, n_keys, X, n, side, V, words, bits);
  return check_launch("k_onen_labels");
}

int64_t onen_reg_parts(int64_t n) { return blocks_for_rows(n); }

int launch_onen_reg(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, float* reg_part,
                    cudaStream_t st) {
  k_onen_reg<<<blocks_for_rows(n), 256, 0, st>>>(codes, rel, d, X, n, reg_part);
  return check_launch("k_onen_reg");
}

int launch_onen_loss_reduce(const float* loss_part, int64_t n_loss, const float* reg_part, int64_t n_reg,
                            double inv_nv, double inv_nd, float* loss, cudaStream_t st) {
  k_onen_loss_reduce<<<1, 256, 0, st>>>(loss_part, n_loss, reg_part, n_reg, inv_nv, inv_nd, loss);
  return check_launch("k_onen_loss_reduce");
}

int launch_onen_scale(const float* src, const float* g_scale, int64_t count, float* dst, cudaStream_t st) {
  const int64_t count4 = count / 4;
  if (count4 == 0) return RGCN_OK;
  const int blocks = (int)std::min<int64_t>((count4 + 255) / 256, REG_MAX_PARTS);
  k_onen_scale<<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(src), g_scale, count4,
                                       reinterpret_cast<float4*>(dst));
  return check_launch("k_onen_scale");
}

int launch_onen_query_bwd(int complex, const float* codes, const float* rel, int d, const int32_t* X, int64_t n,
                          int side, const float* dQ, const float* g_scale, float c_reg, float* dcodes, float* drel,
                          cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  if (!complex) {
    k_onen_query_bwd<<<blocks_for_rows(n), 256, 0, st>>>(codes, rel, d, X, n, dQ, g_scale, c_reg, dcodes, drel);
    return check_launch("k_onen_query_bwd");
  }
  if (d % 8 == 0)
    k_onen_complex_query_bwd<4><<<blocks_for_rows(n), 256, 0, st>>>(codes, rel, d, X, n, side, dQ, g_scale, c_reg,
                                                                      dcodes, drel);
  else
    k_onen_complex_query_bwd<2><<<blocks_for_rows(n), 256, 0, st>>>(codes, rel, d, X, n, side, dQ, g_scale, c_reg,
                                                                      dcodes, drel);
  return check_launch("k_onen_complex_query_bwd");
}
