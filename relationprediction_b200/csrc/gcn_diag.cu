// gcn_diag.cu -- message walks of the diagonal R-GCN layer (Name=gcn_diag) for sm_90a.  Reference:
// encoders/message_gcns/gcn_diag.py with message_gcn.py:49-79.  One message s -> o of weight id w is
//   m = norm * D[w] (.) H[s]          D = [D_forward; D_backward] as a [2R][d] table (16 KB per 8 relations at d = 512,
//                                     resident in L2)
// The weight is diagonal, so a run of messages of one (row, weight id) sums norm * H first and applies D[w] once.
//   forward   k_diaggcn_fwd  destination-major pull with the epilogue fused: out = act(dropout(out) + agg + b), where
//                            `out` holds the self-loop GEMM's H W_self.  Split rows reduce into an L2 scratch row and
//                            the last arriving item applies the epilogue (as k_block_agg does).
//   backward  k_diaggcn_bwd  ONE source-major walk.  Per row u it loads H[u] once and per message gathers G[dst] once;
//                            a run of one weight id sums S = sum norm G[dst], then
//                              dH[u]  += D[w] (.) S                       (read-modify-write after the dS W_self^T GEMM)
//                              dD[w]  += H[u] (.) S                       (one red.global.add.v4 per run and quad)
//                            and, when asked for, the IndexedSlices sum of squares
//                              sumsq[dir] += sum_m norm_m^2 sum_k G[dst_m,k]^2 H[u,k]^2   (one atomic per warp)
// The reductions across split rows, across runs of one weight id and of the slice sums are fp32 atomics (the summation
// order is not deterministic).
#include <cuda_runtime.h>

#include "kernels.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void red4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void fma4(float4& a, float s, const float4& x) {
  a.x = fmaf(s, x.x, a.x);
  a.y = fmaf(s, x.y, a.y);
  a.z = fmaf(s, x.z, a.z);
  a.w = fmaf(s, x.w, a.w);
}
__device__ __forceinline__ void fma4v(float4& a, const float4& s, const float4& x) {
  a.x = fmaf(s.x, x.x, a.x);
  a.y = fmaf(s.y, x.y, a.y);
  a.z = fmaf(s.z, x.z, a.z);
  a.w = fmaf(s.w, x.w, a.w);
}
__device__ __forceinline__ float4 mul4(const float4& a, const float4& b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ const float* diag_row(const float* Df, const float* Db, int w, int half, int d) {
  return w >= half ? Db + (size_t)(w - half) * d : Df + (size_t)w * d;
}

constexpr int U_MSG = 4;  // messages whose gathered rows are in flight per lane

// A warp owns one destination-major work item and one column slab of NV*128 columns; a lane owns NV float4 quads.
// Items of rows without messages exist (beg == end): they still apply the epilogue to the self-loop term.  At NV = 4
// the U_MSG x NV gathered quads need more than the 128 registers two blocks per SM allow (one block keeps 64 KB of
// gathers in flight per SM).
template <int NV>
__global__ void __launch_bounds__(RGCN_THREADS, NV == 4 ? 1 : 2)
    k_diaggcn_fwd(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                  const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ H,
                  const float* __restrict__ Df, const float* __restrict__ Db, int d, int half,
                  const float* __restrict__ bias, const uint8_t* __restrict__ mask, float inv_keep, int relu,
                  const int32_t* __restrict__ split_nitems, float* __restrict__ scratch, int* __restrict__ counters,
                  float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, row = itv.z, split = itv.w;
  bool ok[NV];
  float4 acc[NV], xs[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = c0 + 4 * (lane + 32 * k) < d;
    acc[k] = xs[k] = zero4();
  }
  int cur = -1;
  auto apply = [&](int w) {
    const float* dr = diag_row(Df, Db, w, half, d) + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) fma4v(acc[k], ldg4(dr + 4 * (lane + 32 * k)), xs[k]);
  };

  for (int base = beg; base < end; base += 32) {
    const int n = min(32, end - base);
    int my_nbr = 0, my_rw = 0;
    float my_nm = 0.f;
    if (lane < n) {
      my_nbr = __ldg(nbr + base + lane);
      my_rw = __ldg(relw + base + lane);
      my_nm = __ldg(norm + base + lane);
    }
    for (int t = 0; t < n; t += U_MSG) {
      float4 x[U_MSG][NV];
      int rw[U_MSG];
      float nm[U_MSG];
#pragma unroll
      for (int u = 0; u < U_MSG; ++u) {
        const int tt = min(t + u, n - 1);  // tail: re-read the last row, skipped below
        const int src = __shfl_sync(FULL, my_nbr, tt);
        rw[u] = __shfl_sync(FULL, my_rw, tt);
        nm[u] = __shfl_sync(FULL, my_nm, tt);
        const float* xr = H + (size_t)src * d + c0;
#pragma unroll
        for (int k = 0; k < NV; ++k) x[u][k] = ok[k] ? ldg4(xr + 4 * (lane + 32 * k)) : zero4();
      }
#pragma unroll
      for (int u = 0; u < U_MSG; ++u) {
        if (t + u < n) {
          if (rw[u] != cur) {
            if (cur >= 0) apply(cur);
            cur = rw[u];
#pragma unroll
            for (int k = 0; k < NV; ++k) xs[k] = zero4();
          }
#pragma unroll
          for (int k = 0; k < NV; ++k) fma4(xs[k], nm[u], x[u][k]);
        }
      }
    }
  }
  if (cur >= 0) apply(cur);

  if (split >= 0) {
    float* sc = scratch + (size_t)split * d + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) red4(sc + 4 * (lane + 32 * k), acc[k]);
    __threadfence();
    __syncwarp();
    int last = 0;
    if (lane == 0) {
      const int old = atomicAdd(counters + (size_t)split * gridDim.y + blockIdx.y, 1);
      last = (old == __ldg(split_nitems + split) - 1);
    }
    if (!__shfl_sync(FULL, last, 0)) return;
    __threadfence();
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (ok[k]) acc[k] = ldcg4(sc + 4 * (lane + 32 * k));
  }
  float* po = out + (size_t)row * d + c0;
  const uint8_t* pm = mask ? mask + (size_t)row * d + c0 : nullptr;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!ok[k]) continue;
    const int lc = 4 * (lane + 32 * k);
    float4 sl = *reinterpret_cast<const float4*>(po + lc);
    if (pm) {
      const uchar4 mk = *reinterpret_cast<const uchar4*>(pm + lc);
      sl.x = mk.x ? sl.x * inv_keep : 0.f;
      sl.y = mk.y ? sl.y * inv_keep : 0.f;
      sl.z = mk.z ? sl.z * inv_keep : 0.f;
      sl.w = mk.w ? sl.w * inv_keep : 0.f;
    }
    const float4 b = ldg4(bias + c0 + lc);
    float4 r = make_float4(sl.x + acc[k].x + b.x, sl.y + acc[k].y + b.y, sl.z + acc[k].z + b.z,
                           sl.w + acc[k].w + b.w);
    if (relu) {
      r.x = fmaxf(r.x, 0.f);
      r.y = fmaxf(r.y, 0.f);
      r.z = fmaxf(r.z, 0.f);
      r.w = fmaxf(r.w, 0.f);
    }
    *reinterpret_cast<float4*>(po + lc) = r;
  }
}

// Source-major walk (rows = sources u, nbr = destinations, X = G).  dH must hold dS W_self^T (zeros for halo rows),
// dDf / dDb zeros, sumsq2 (if not null) the values to accumulate into.
template <int NV>
__global__ void __launch_bounds__(RGCN_THREADS, 1)
    k_diaggcn_bwd(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                  const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ G,
                  const float* __restrict__ H, const float* __restrict__ Df, const float* __restrict__ Db, int d,
                  int half, float* __restrict__ dH, float* __restrict__ dDf, float* __restrict__ dDb,
                  float* __restrict__ sumsq2) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, row = itv.z, split = itv.w;
  if (beg == end) return;
  const bool want_ss = sumsq2 != nullptr;
  bool ok[NV];
  float4 acc[NV], xs[NV], h[NV];
  const float* hr = H + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = c0 + 4 * (lane + 32 * k) < d;
    acc[k] = xs[k] = zero4();
    h[k] = ok[k] ? ldg4(hr + 4 * (lane + 32 * k)) : zero4();
  }
  float ssf = 0.f, ssb = 0.f;
  int cur = -1;
  auto flush = [&](int w) {
    const int dir = w >= half ? 1 : 0;
    const float* dr = diag_row(Df, Db, w, half, d) + c0;
    float* dd = (dir ? dDb + (size_t)(w - half) * d : dDf + (size_t)w * d) + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (ok[k]) {
        const int lc = 4 * (lane + 32 * k);
        fma4v(acc[k], ldg4(dr + lc), xs[k]);
        red4(dd + lc, mul4(h[k], xs[k]));
      }
    }
  };

  for (int base = beg; base < end; base += 32) {
    const int n = min(32, end - base);
    int my_nbr = 0, my_rw = 0;
    float my_nm = 0.f;
    if (lane < n) {
      my_nbr = __ldg(nbr + base + lane);
      my_rw = __ldg(relw + base + lane);
      my_nm = __ldg(norm + base + lane);
    }
    for (int t = 0; t < n; t += U_MSG) {
      float4 x[U_MSG][NV];
      int rw[U_MSG];
      float nm[U_MSG];
#pragma unroll
      for (int u = 0; u < U_MSG; ++u) {
        const int tt = min(t + u, n - 1);
        const int v = __shfl_sync(FULL, my_nbr, tt);
        rw[u] = __shfl_sync(FULL, my_rw, tt);
        nm[u] = __shfl_sync(FULL, my_nm, tt);
        const float* gr = G + (size_t)v * d + c0;
#pragma unroll
        for (int k = 0; k < NV; ++k) x[u][k] = ok[k] ? ldg4(gr + 4 * (lane + 32 * k)) : zero4();
      }
#pragma unroll
      for (int u = 0; u < U_MSG; ++u) {
        if (t + u < n) {
          if (rw[u] != cur) {
            if (cur >= 0) flush(cur);
            cur = rw[u];
#pragma unroll
            for (int k = 0; k < NV; ++k) xs[k] = zero4();
          }
#pragma unroll
          for (int k = 0; k < NV; ++k) fma4(xs[k], nm[u], x[u][k]);
          if (want_ss) {
            float p = 0.f;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
              const float4 q = mul4(x[u][k], h[k]);
              p = fmaf(q.x, q.x, fmaf(q.y, q.y, fmaf(q.z, q.z, fmaf(q.w, q.w, p))));
            }
            if (rw[u] >= half)
              ssb = fmaf(nm[u] * nm[u], p, ssb);
            else
              ssf = fmaf(nm[u] * nm[u], p, ssf);
          }
        }
      }
    }
  }
  flush(cur);

  float* pd = dH + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!ok[k]) continue;
    float* p = pd + 4 * (lane + 32 * k);
    if (split >= 0) {
      red4(p, acc[k]);
    } else {
      float4 o = *reinterpret_cast<float4*>(p);
      o.x += acc[k].x;
      o.y += acc[k].y;
      o.z += acc[k].z;
      o.w += acc[k].w;
      *reinterpret_cast<float4*>(p) = o;
    }
  }
  if (want_ss) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ssf += __shfl_xor_sync(FULL, ssf, o);
      ssb += __shfl_xor_sync(FULL, ssb, o);
    }
    if (lane == 0) {
      if (ssf != 0.f) atomicAdd(sumsq2, ssf);
      if (ssb != 0.f) atomicAdd(sumsq2 + 1, ssb);
    }
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

// quads per lane: min(ceil(d / 128), 4); wider rows are cut into column slabs of 512
int pick_nv(int d) {
  const int nv = (d + 127) / 128;
  return nv > 4 ? 4 : nv;
}

}  // namespace

int launch_diaggcn_fwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* H, const float* Df, const float* Db, int d, int n_relw, const float* bias,
                       const uint8_t* mask, float inv_keep, int relu, const int32_t* split_nitems, float* scratch,
                       int* counters, float* out, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int nv = pick_nv(d);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  const int half = n_relw / 2;
#define FWD(NV_)                                                                                                  \
  k_diaggcn_fwd<NV_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, H, Df, Db, d, half, bias, mask, \
                                                    inv_keep, relu, split_nitems, scratch, counters, out)
  switch (nv) {
    case 1: FWD(1); break;
    case 2: FWD(2); break;
    case 3: FWD(3); break;
    default: FWD(4); break;
  }
#undef FWD
  return check_launch("k_diaggcn_fwd");
}

int launch_diaggcn_bwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* G, const float* H, const float* Df, const float* Db, int d, int n_relw, float* dH,
                       float* dDf, float* dDb, float* sumsq2, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int nv = pick_nv(d);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  const int half = n_relw / 2;
#define BWD(NV_)                                                                                                  \
  k_diaggcn_bwd<NV_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, G, H, Df, Db, d, half, dH, dDf, \
                                                    dDb, sumsq2)
  switch (nv) {
    case 1: BWD(1); break;
    case 2: BWD(2); break;
    case 3: BWD(3); break;
    default: BWD(4); break;
  }
#undef BWD
  return check_launch("k_diaggcn_bwd");
}
