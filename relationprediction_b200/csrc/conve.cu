// conve.cu -- the ConvE query network (DESIGN.md section 1), sm_90a: the 3x3 convolution over the stacked
// [anchor ; relation] image and its backward, the FC layer's bias / hidden-dropout / ReLU pass and the element-wise
// steps of its backward.  The FC products themselves are the 3xTF32 GEMMs of gemm_tf32x3.cu.
//
// A query t gathers the anchor row codes[X[3t + acol]] and the relation row rel[X[3t + 1]] ([d] each, d = h w), stacks
// them row-major into a 2h x w image (anchor on top), and the C filters (valid 3x3, stride 1) give C planes of
// P = (2h - 2)(w - 2) outputs: the feature row of F = C P columns, channel-major, stored with leading dimension Fp
// (F rounded up to 4, the padding columns zero) so that it is the A operand of the FC GEMM.
// Masks are uint8 keep-masks (1 keep, 0 drop), scaled by 1/keep; a null mask is no dropout.
#include <cuda_runtime.h>

#include <algorithm>
#include <string>

#include "kernels.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}

// the image of query t (input dropout applied) into img[2d]
__device__ __forceinline__ void load_image(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                                           int a, int r, const uint8_t* __restrict__ in_mask, float inv_in,
                                           int64_t t, float* img) {
  for (int i = threadIdx.x; i < 2 * d; i += blockDim.x) {
    float v = i < d ? __ldg(codes + (size_t)a * d + i) : __ldg(rel + (size_t)r * d + (i - d));
    if (in_mask) v *= (float)__ldg(in_mask + (size_t)t * 2 * d + i) * inv_in;
    img[i] = v;
  }
}

// Forward: one CTA walks queries t = blockIdx.x, + gridDim.x, ...; smem img [2d] | filt [9C] | bias [C].
// Feat[t][c P + p] = relu(bias[c] + sum_k filt[c][k] img[...]) * featmask[t][c] / keep_f; columns F..Fp-1 zero.
__global__ void __launch_bounds__(256)
    k_conve_conv_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, int h, int w, int C,
                     const int32_t* __restrict__ X, int acol, int64_t n, const float* __restrict__ filt,
                     const float* __restrict__ cbias, const uint8_t* __restrict__ in_mask, float inv_in,
                     const uint8_t* __restrict__ feat_mask, float inv_feat, int Fp, float* __restrict__ Feat) {
  extern __shared__ float sm[];
  float* img = sm;
  float* sf = img + 2 * d;
  float* sb = sf + 9 * C;
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) sf[i] = __ldg(filt + i);
  for (int i = threadIdx.x; i < C; i += blockDim.x) sb[i] = __ldg(cbias + i);
  const int ow = w - 2, P = (2 * h - 2) * ow, F = C * P;
  for (int64_t t = blockIdx.x; t < n; t += gridDim.x) {
    __syncthreads();   // the previous query's readers of img are done
    load_image(codes, rel, d, __ldg(X + 3 * t + acol), __ldg(X + 3 * t + 1), in_mask, inv_in, t, img);
    __syncthreads();
    float* out = Feat + (size_t)t * Fp;
    for (int o = threadIdx.x; o < Fp; o += blockDim.x) {
      float v = 0.f;
      if (o < F) {
        const int c = o / P, p = o - c * P, y = p / ow, x = p - y * ow;
        const float* f = sf + 9 * c;
        const float* im = img + y * w + x;
        v = sb[c];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) v = fmaf(f[3 * ky + kx], im[ky * w + kx], v);
        v = fmaxf(v, 0.f);
        if (feat_mask) v *= (float)__ldg(feat_mask + (size_t)t * C + c) * inv_feat;
      }
      out[o] = v;
    }
  }
}

// Q [n, d] holds Z = Feat W_fc; Q = relu((Z + b) * hidmask / keep_h) in place
__global__ void __launch_bounds__(256)
    k_conve_fc_act(float* __restrict__ Q, int64_t n, int d, const float* __restrict__ b,
                   const uint8_t* __restrict__ hid_mask, float inv_hid) {
  const int64_t total = n * d;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float v = Q[i] + __ldg(b + i % d);
    if (hid_mask) v *= (float)__ldg(hid_mask + i) * inv_hid;
    Q[i] = fmaxf(v, 0.f);
  }
}

// dZ = dQ * [Q > 0] * hidmask / keep_h, written row-major dZ [m, d] and transposed dZt [d, ldt] (columns m..ldt-1
// zero); 32 x 32 tiles through shared memory so that both stores are coalesced
__global__ void __launch_bounds__(256)
    k_conve_dz(const float* __restrict__ Q, const float* __restrict__ dQ, int64_t m, int d,
               const uint8_t* __restrict__ hid_mask, float inv_hid, float* __restrict__ dZ, float* __restrict__ dZt,
               int64_t ldt) {
  __shared__ float tile[32][33];
  const int64_t t0 = (int64_t)blockIdx.y * 32;
  const int j0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int64_t t = t0 + i;
    const int j = j0 + threadIdx.x;
    float g = 0.f;
    if (t < m && j < d) {
      const size_t k = (size_t)t * d + j;
      if (__ldg(Q + k) > 0.f) g = __ldg(dQ + k) * (hid_mask ? (float)__ldg(hid_mask + k) * inv_hid : 1.f);
      dZ[k] = g;
    }
    tile[i][threadIdx.x] = g;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int j = j0 + i;
    const int64_t t = t0 + threadIdx.x;
    if (j < d && t < ldt) dZt[(size_t)j * ldt + t] = tile[threadIdx.x][i];
  }
}

// db[j] (+)= sum over t < m of dZt[j][t], one warp per j, lanes in a fixed order
__global__ void __launch_bounds__(256)
    k_conve_rowsum(const float* __restrict__ dZt, int d, int64_t m, int64_t ldt, float* __restrict__ db,
                   int accumulate) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = blockIdx.x * 8 + warp; j < d; j += gridDim.x * 8) {
    float s = 0.f;
    for (int64_t t = lane; t < m; t += 32) s += dZt[(size_t)j * ldt + t];
    s = warp_sum(s);
    if (lane == 0) db[j] = accumulate ? db[j] + s : s;
  }
}

// Backward of the convolution for the queries of one launch.  dF [m, Fp] is the gradient of the feature rows; the
// pre-activation gradient is dF / keep_f where Feat > 0 (a dropped channel or an inactive ReLU has Feat = 0) and 0
// elsewhere.  Per CTA (queries t = blockIdx.x, + gridDim.x, ...): the filter and bias gradients of its queries in
// acc [10C] (entry c*10 + k: tap k < 9, bias k = 9; each entry one warp's, summed in a fixed order), written to
// part[blockIdx.x]; the image gradient, input-dropout masked, red.add into dcodes[anchor] and drel[r].
// smem: img [2d] | dimg [2d] | filt [9C] | acc [10C] | dpre [cg P] (cg channels at a time).
__global__ void __launch_bounds__(256)
    k_conve_conv_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, int h, int w, int C,
                     int cg, const int32_t* __restrict__ X, int64_t m, const float* __restrict__ filt,
                     const uint8_t* __restrict__ in_mask, float inv_in, const float* __restrict__ Feat,
                     const float* __restrict__ dF, float inv_feat, int Fp, float* __restrict__ part,
                     float* __restrict__ dcodes, float* __restrict__ drel) {
  extern __shared__ float sm[];
  float* img = sm;
  float* dimg = img + 2 * d;
  float* sf = dimg + 2 * d;
  float* acc = sf + 9 * C;
  float* dpre = acc + 10 * C;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) sf[i] = __ldg(filt + i);
  for (int i = threadIdx.x; i < 10 * C; i += blockDim.x) acc[i] = 0.f;
  const int ow = w - 2, oh = 2 * h - 2, P = oh * ow;
  for (int64_t t = blockIdx.x; t < m; t += gridDim.x) {
    const int a = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1);
    __syncthreads();
    load_image(codes, rel, d, a, r, in_mask, inv_in, t, img);
    for (int i = threadIdx.x; i < 2 * d; i += blockDim.x) dimg[i] = 0.f;
    const float* ft = Feat + (size_t)t * Fp;
    const float* gt = dF + (size_t)t * Fp;
    for (int c0 = 0; c0 < C; c0 += cg) {
      const int cn = min(cg, C - c0);
      __syncthreads();   // img loaded; the previous group's readers of dpre are done
      for (int i = threadIdx.x; i < cn * P; i += blockDim.x) {
        const int o = c0 * P + i;
        dpre[i] = __ldg(ft + o) > 0.f ? __ldg(gt + o) * inv_feat : 0.f;
      }
      __syncthreads();
      for (int e = warp; e < cn * 10; e += nwarps) {
        const int cl = e / 10, k = e - cl * 10, ky = k / 3, kx = k - 3 * ky;
        const float* dp = dpre + cl * P;
        float s = 0.f;
        for (int p = lane; p < P; p += 32) {
          const int y = p / ow, x = p - y * ow;
          s = fmaf(dp[p], k < 9 ? img[(y + ky) * w + x + kx] : 1.f, s);
        }
        s = warp_sum(s);
        if (lane == 0) acc[(c0 + cl) * 10 + k] += s;
      }
      for (int q = threadIdx.x; q < 2 * d; q += blockDim.x) {
        const int iy = q / w, ix = q - iy * w;
        float s = 0.f;
        for (int cl = 0; cl < cn; ++cl) {
          const float* f = sf + 9 * (c0 + cl);
          const float* dp = dpre + cl * P;
#pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const int y = iy - ky;
            if (y < 0 || y >= oh) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int x = ix - kx;
              if (x >= 0 && x < ow) s = fmaf(dp[y * ow + x], f[3 * ky + kx], s);
            }
          }
        }
        dimg[q] += s;
      }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < 2 * d; q += blockDim.x) {
      float g = dimg[q];
      if (in_mask) g *= (float)__ldg(in_mask + (size_t)t * 2 * d + q) * inv_in;
      if (q < d)
        atomicAdd(dcodes + (size_t)a * d + q, g);
      else
        atomicAdd(drel + (size_t)r * d + (q - d), g);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 10 * C; i += blockDim.x) part[(size_t)blockIdx.x * 10 * C + i] = acc[i];
}

// dfilt[c][k] / dbias[c] (+)= the sum of the parts in part order
__global__ void __launch_bounds__(256)
    k_conve_filter_reduce(const float* __restrict__ part, int parts, int C, float* __restrict__ dfilt,
                          float* __restrict__ dbias, int accumulate) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < 10 * C; e += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int g = 0; g < parts; ++g) s += part[(size_t)g * 10 * C + e];
    const int c = e / 10, k = e - 10 * c;
    float* dst = k < 9 ? dfilt + 9 * c + k : dbias + c;
    *dst = accumulate ? *dst + s : s;
  }
}

__device__ __forceinline__ void split_rna(float a, float& hi, float& lo) {
  uint32_t hb, lb;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(a));
  hi = __uint_as_float(hb);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(a - hi));
  lo = __uint_as_float(lb);
}

// The pre-split FC weight W [F, d], zero-padded to Fp rows: transposed = 1 gives Bt = W^T [d, Fp] (the forward,
// Z = Feat W), 0 gives Bt = W [Fp, d] (the backward, dF = dZ W^T).  The split rounds as k_split_b does.
__global__ void k_conve_split_w(const float* __restrict__ W, int F, int d, int Fp, int transposed,
                                float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t total = (int64_t)Fp * d;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = transposed ? (int)(i % Fp) : (int)(i / d), j = transposed ? (int)(i / Fp) : (int)(i % d);
    float hv = 0.f, lv = 0.f;
    if (k < F) split_rna(__ldg(W + (size_t)k * d + j), hv, lv);
    hi[i] = hv;
    lo[i] = lv;
  }
}

// dW [F, d] = the first F columns of dWt [d, Fp], transposed (32 x 32 tiles)
__global__ void __launch_bounds__(256)
    k_conve_transpose(const float* __restrict__ dWt, int F, int d, int Fp, float* __restrict__ dW) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int j = j0 + i, k = k0 + threadIdx.x;
    if (j < d && k < F) tile[i][threadIdx.x] = dWt[(size_t)j * Fp + k];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int k = k0 + i, j = j0 + threadIdx.x;
    if (k < F && j < d) dW[(size_t)k * d + j] = tile[threadIdx.x][i];
  }
}

// gold_sig[t] = sigmoid(<Q[t], codes[gold]>), gold = X[t][0] (side 0) or X[t][2] (side 1); one warp per query,
// summed as k_rank_prepare does
__global__ void __launch_bounds__(256)
    k_conve_gold(const float* __restrict__ Q, const float* __restrict__ codes, int d, const int32_t* __restrict__ X,
                 int64_t n, int side, float* __restrict__ gold_sig, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d4 = d >> 2, gcol = side == 0 ? 0 : 2;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int gold = __ldg(X + 3 * t + gcol);
    const float4* q = reinterpret_cast<const float4*>(Q + (size_t)t * d);
    const float4* eg = reinterpret_cast<const float4*>(codes + (size_t)gold * d);
    float e = 0.f;
#pragma unroll 1
    for (int i = lane; i < d4; i += 32) {
      const float4 p = __ldg(q + i), c = __ldg(eg + i);
      e = fmaf(p.x, c.x, e);
      e = fmaf(p.y, c.y, e);
      e = fmaf(p.z, c.z, e);
      e = fmaf(p.w, c.w, e);
    }
    e = warp_sum(e);
    if (lane == 0) {
      gold_sig[t] = 1.0f / (1.0f + expf(-e));
      gold_col[t] = gold;
    }
  }
}

// dst = g_scale[0] src over `count` floats (any count)
__global__ void __launch_bounds__(256)
    k_conve_scale(const float* __restrict__ src, const float* __restrict__ g_scale, int64_t count,
                  float* __restrict__ dst) {
  const float g = __ldg(g_scale);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = g * __ldg(src + i);
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int grid_for(int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>((items + 255) / 256, 132 * 8)); }

// raises the kernel's dynamic shared memory limit when `bytes` needs more than the default 48 KB
template <class K>
int smem_limit(K kernel, int64_t bytes, const char* label) {
  if (bytes > 227 * 1024) {
    rgcn_set_error(std::string(label) + ": the shape needs more shared memory than a block has");
    return RGCN_ERR_INVALID;
  }
  if (bytes <= 48 * 1024) return RGCN_OK;
  return rgcn_check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
                         (std::string("cudaFuncSetAttribute(") + label + ")").c_str());
}

constexpr int CONV_CTAS = 132 * 2;   // CTAs of the convolution kernels: a fixed count, so the parts are repeatable

}  // namespace

int64_t conve_conv_parts(int64_t m) { return std::max<int64_t>(1, std::min<int64_t>(m, CONV_CTAS)); }

// channels of one dpre group of k_conve_conv_bwd: as many as keep its shared memory within 48 KB, at least one
static int conve_bwd_group(int d, int h, int w, int C) {
  const int64_t P = (int64_t)(2 * h - 2) * (w - 2), base = (4LL * d + 19LL * C) * 4;
  const int64_t cg = (48 * 1024 - base) / (P * 4);
  return (int)std::max<int64_t>(1, std::min<int64_t>(cg, C));
}

int64_t conve_smem_bytes(int d, int h, int w, int C) {
  const int64_t P = (int64_t)(2 * h - 2) * (w - 2);
  const int64_t fwd = (2LL * d + 10LL * C) * 4, bwd = (4LL * d + 19LL * C) * 4 + conve_bwd_group(d, h, w, C) * P * 4;
  return std::max(fwd, bwd);
}

int launch_conve_conv_fwd(const float* codes, const float* rel, int d, int h, int C, const int32_t* X, int acol,
                          int64_t n, const float* filt, const float* cbias, const uint8_t* in_mask, float inv_in,
                          const uint8_t* feat_mask, float inv_feat, int Fp, float* Feat, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  const int w = d / h;
  const int64_t smem = (2LL * d + 10LL * C) * 4;
  int rc = smem_limit(k_conve_conv_fwd, smem, "k_conve_conv_fwd");
  if (rc) return rc;
  k_conve_conv_fwd<<<(int)conve_conv_parts(n), 256, smem, st>>>(codes, rel, d, h, w, C, X, acol, n, filt, cbias,
                                                                in_mask, inv_in, feat_mask, inv_feat, Fp, Feat);
  return check_launch("k_conve_conv_fwd");
}

int launch_conve_fc_act(float* Q, int64_t n, int d, const float* b, const uint8_t* hid_mask, float inv_hid,
                        cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_conve_fc_act<<<grid_for(n * d), 256, 0, st>>>(Q, n, d, b, hid_mask, inv_hid);
  return check_launch("k_conve_fc_act");
}

int launch_conve_dz(const float* Q, const float* dQ, int64_t m, int d, const uint8_t* hid_mask, float inv_hid,
                    float* dZ, float* dZt, int64_t ldt, cudaStream_t st) {
  if (ldt == 0) return RGCN_OK;
  const dim3 grid((d + 31) / 32, (unsigned)((ldt + 31) / 32)), block(32, 8);
  k_conve_dz<<<grid, block, 0, st>>>(Q, dQ, m, d, hid_mask, inv_hid, dZ, dZt, ldt);
  return check_launch("k_conve_dz");
}

int launch_conve_rowsum(const float* dZt, int d, int64_t m, int64_t ldt, float* db, int accumulate, cudaStream_t st) {
  k_conve_rowsum<<<(d + 7) / 8, 256, 0, st>>>(dZt, d, m, ldt, db, accumulate);
  return check_launch("k_conve_rowsum");
}

int launch_conve_conv_bwd(const float* codes, const float* rel, int d, int h, int C, const int32_t* X, int64_t m,
                          const float* filt, const uint8_t* in_mask, float inv_in, const float* Feat, const float* dF,
                          float inv_feat, int Fp, float* part, float* dcodes, float* drel, cudaStream_t st) {
  if (m == 0) return RGCN_OK;
  const int w = d / h, cg = conve_bwd_group(d, h, w, C);
  const int64_t smem = (4LL * d + 19LL * C) * 4 + (int64_t)cg * (2 * h - 2) * (w - 2) * 4;
  int rc = smem_limit(k_conve_conv_bwd, smem, "k_conve_conv_bwd");
  if (rc) return rc;
  k_conve_conv_bwd<<<(int)conve_conv_parts(m), 256, smem, st>>>(codes, rel, d, h, w, C, cg, X, m, filt, in_mask,
                                                                inv_in, Feat, dF, inv_feat, Fp, part, dcodes, drel);
  return check_launch("k_conve_conv_bwd");
}

int launch_conve_filter_reduce(const float* part, int parts, int C, float* dfilt, float* dbias, int accumulate,
                               cudaStream_t st) {
  k_conve_filter_reduce<<<grid_for(10LL * C), 256, 0, st>>>(part, parts, C, dfilt, dbias, accumulate);
  return check_launch("k_conve_filter_reduce");
}

int launch_conve_split_w(const float* W, int F, int d, int Fp, int transposed, float* hi, float* lo,
                         cudaStream_t st) {
  k_conve_split_w<<<grid_for((int64_t)Fp * d), 256, 0, st>>>(W, F, d, Fp, transposed, hi, lo);
  return check_launch("k_conve_split_w");
}

int launch_conve_transpose(const float* dWt, int F, int d, int Fp, float* dW, cudaStream_t st) {
  const dim3 grid((F + 31) / 32, (d + 31) / 32), block(32, 8);
  k_conve_transpose<<<grid, block, 0, st>>>(dWt, F, d, Fp, dW);
  return check_launch("k_conve_transpose");
}

int launch_conve_gold(const float* Q, const float* codes, int d, const int32_t* X, int64_t n, int side,
                      float* gold_sig, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  k_conve_gold<<<(int)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, 132 * 8)), 256, 0, st>>>(
      Q, codes, d, X, n, side, gold_sig, gold_col);
  return check_launch("k_conve_gold");
}

int launch_conve_scale(const float* src, const float* g_scale, int64_t count, float* dst, cudaStream_t st) {
  if (count == 0) return RGCN_OK;
  k_conve_scale<<<grid_for(count), 256, 0, st>>>(src, g_scale, count, dst);
  return check_launch("k_conve_scale");
}
