// basis_onehot.cu -- forward of the featureless (one-hot input) first basis layer for sm_90a.
// Reference: gcn_basis.py:15-71 with onehot_input=True (dot_or_lookup = embedding_lookup, shared_functions.py:5-9),
// message_gcn.py:28-79.  With one-hot input the basis terms of a message are rows of the tables themselves:
//   m = sum_b C_dir[r, b] * W_dir[u, b, :]       (u = the message's source, W_dir : [V, B, d])
// so there is nothing to aggregate before a transform.  The kernel walks the source-major view (messages of one
// source sorted by weight id): a run of messages with one (source, weight id) forms m ONCE from the source's table
// row (B*d floats, read once per run and from L1/L2 by later runs of the same source), then PUSHES norm * m into
// every destination row with 128-bit vector reductions (red.global.add.v4.f32) that resolve in L2.  A
// destination-major pull would gather a different B*d table row per message instead.
// The summation order across sources is not deterministic (fp32 reductions).
#include <cuda_runtime.h>

#include "kernels.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void red4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// A warp owns one work item of the source-major view (<= item_max messages of one source) and one column slab of
// NV*128 columns; a lane owns NV float4 quads of the row.
template <int NV>
__global__ void __launch_bounds__(RGCN_THREADS)
    k_basis_onehot_push(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                        const int32_t* __restrict__ relw, const float* __restrict__ norm,
                        const float* __restrict__ Wf, const float* __restrict__ Wb, const float* __restrict__ C,
                        int B, int d, int half, float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, u = itv.z;
  const size_t dB = (size_t)d * B;
  bool ok[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) ok[k] = c0 + 4 * (lane + 32 * k) < d;

  float4 m[NV];
  int cur = -1;
  for (int base = beg; base < end; base += 32) {
    const int n = min(32, end - base);
    int my_v = 0, my_rw = 0;
    float my_nm = 0.f;
    if (lane < n) {
      my_v = __ldg(nbr + base + lane);
      my_rw = __ldg(relw + base + lane);
      my_nm = __ldg(norm + base + lane);
    }
    for (int t = 0; t < n; ++t) {
      const int rw = __shfl_sync(FULL, my_rw, t);
      const int v = __shfl_sync(FULL, my_v, t);
      const float nm = __shfl_sync(FULL, my_nm, t);
      if (rw != cur) {  // warp-uniform: a new run, form its message row m
        cur = rw;
        const float* wr = (rw >= half ? Wb : Wf) + (size_t)u * dB + c0;
        const float* cr = C + (size_t)rw * B;
#pragma unroll
        for (int k = 0; k < NV; ++k) m[k] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
        for (int b = 0; b < B; ++b) {
          const float cb = __ldg(cr + b);
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            if (ok[k]) {
              const float4 w = ldg4(wr + (size_t)b * d + 4 * (lane + 32 * k));
              m[k].x = fmaf(cb, w.x, m[k].x);
              m[k].y = fmaf(cb, w.y, m[k].y);
              m[k].z = fmaf(cb, w.z, m[k].z);
              m[k].w = fmaf(cb, w.w, m[k].w);
            }
          }
        }
      }
      float* po = out + (size_t)v * d + c0;
#pragma unroll
      for (int k = 0; k < NV; ++k)
        if (ok[k]) red4(po + 4 * (lane + 32 * k), make_float4(nm * m[k].x, nm * m[k].y, nm * m[k].z, nm * m[k].w));
    }
  }
}

}  // namespace

int launch_basis_onehot_push(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                             const float* norm, const float* Wf, const float* Wb, const float* C, int B, int d,
                             int n_relw, float* out, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  int nv = (d + 127) / 128;
  if (nv > 4) nv = 4;
  const int slabs = (d + nv * 128 - 1) / (nv * 128);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, slabs);
  const int half = n_relw / 2;
#define PUSH(NV_) \
  k_basis_onehot_push<NV_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, Wf, Wb, C, B, d, half, out)
  switch (nv) {
    case 1: PUSH(1); break;
    case 2: PUSH(2); break;
    case 3: PUSH(3); break;
    default: PUSH(4); break;
  }
#undef PUSH
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_basis_onehot_push");
}
