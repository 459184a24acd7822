// highway.cu -- backward prologue of the highway gate (extras/highway_layer.py:19-38).
//
// Forward (the gate GEMM with its blend epilogue, k_gemm_tf32x3<2> in gemm_tf32x3.cu):
//   z = c2 W + b,  g = sigmoid(z),  out = g c1 + (1 - g) c2.
// Backward, given dY = d out and the saved g, one pass over the seven [V, d] streams:
//   dc1 = g dY,   dc2 = (1 - g) dY,   dz = dY (c1 - c2) g (1 - g),   db += column sums of dz.
// The two GEMMs that follow (dc2 += dz W^T, dW = c2^T dz) run on the tensor-core kernels of gemm_tf32x3.cu.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "kernels.cuh"

namespace {

constexpr int HW_TX = 32;   // float4 columns per CTA (128 floats)
constexpr int HW_TY = 8;    // row lanes per CTA

// CTA (x, y): float4 columns 32 x .. 32 x + 31, rows y * 8 + ty, stepping by gridDim.y * 8.  Each thread keeps its
// column's partial sum of dz in registers; the CTA folds its 8 row lanes in shared memory and adds one value per
// column into db (zeroed by the caller).
__global__ void __launch_bounds__(HW_TX* HW_TY)
    k_highway_prologue(const float4* __restrict__ c1, const float4* __restrict__ c2, const float4* __restrict__ g,
                       const float4* __restrict__ dY, int64_t V, int d4, float4* __restrict__ dc1,
                       float4* __restrict__ dz, float4* __restrict__ dc2, float* __restrict__ db) {
  __shared__ float4 part[HW_TY][HW_TX];
  const int tx = threadIdx.x % HW_TX, ty = threadIdx.x / HW_TX;
  const int col = blockIdx.x * HW_TX + tx;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < d4) {
    for (int64_t r = (int64_t)blockIdx.y * HW_TY + ty; r < V; r += (int64_t)gridDim.y * HW_TY) {
      const int64_t i = r * d4 + col;
      const float4 a = __ldg(c1 + i), b = __ldg(c2 + i), gg = __ldg(g + i), y = __ldg(dY + i);
      float4 o1, oz, o2;
      o1.x = gg.x * y.x; o2.x = (1.f - gg.x) * y.x; oz.x = o1.x * (a.x - b.x) * (1.f - gg.x);
      o1.y = gg.y * y.y; o2.y = (1.f - gg.y) * y.y; oz.y = o1.y * (a.y - b.y) * (1.f - gg.y);
      o1.z = gg.z * y.z; o2.z = (1.f - gg.z) * y.z; oz.z = o1.z * (a.z - b.z) * (1.f - gg.z);
      o1.w = gg.w * y.w; o2.w = (1.f - gg.w) * y.w; oz.w = o1.w * (a.w - b.w) * (1.f - gg.w);
      __stcs(dc1 + i, o1);
      dz[i] = oz;        // dz and dc2 are read again by the GEMMs that follow: plain stores
      dc2[i] = o2;
      s.x += oz.x; s.y += oz.y; s.z += oz.z; s.w += oz.w;
    }
  }
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && col < d4) {
#pragma unroll
    for (int k = 1; k < HW_TY; ++k) {
      const float4 p = part[k][tx];
      s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
    }
    float* o = db + 4 * col;
    atomicAdd(o + 0, s.x);
    atomicAdd(o + 1, s.y);
    atomicAdd(o + 2, s.z);
    atomicAdd(o + 3, s.w);
  }
}

}  // namespace

int launch_highway_prologue(const float* c1, const float* c2, const float* g, const float* dY, int64_t V, int d,
                            float* dc1, float* dz, float* dc2, float* db, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(db, 0, (size_t)d * sizeof(float), st), "memset(db)");
  if (rc || V == 0) return rc;
  const int d4 = d / 4;
  const int gx = (d4 + HW_TX - 1) / HW_TX;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // about 8 CTAs of 256 threads per SM in all (full occupancy), fewer when V has fewer row groups
  const int64_t gy = std::max<int64_t>(1, std::min<int64_t>((V + HW_TY - 1) / HW_TY, (int64_t)sms * 8 / gx));
  k_highway_prologue<<<dim3(gx, (unsigned)gy), HW_TX * HW_TY, 0, st>>>(
      reinterpret_cast<const float4*>(c1), reinterpret_cast<const float4*>(c2), reinterpret_cast<const float4*>(g),
      reinterpret_cast<const float4*>(dY), V, d4, reinterpret_cast<float4*>(dc1), reinterpret_cast<float4*>(dz),
      reinterpret_cast<float4*>(dc2), db);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_highway_prologue");
}
