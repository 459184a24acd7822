// basis_diagcoef.cu -- walks of the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes) for
// sm_90a.  Reference: gcn_basis_times_diag.py with message_gcn.py:49-79.  One message s -> o of weight id w:
//   m = sum_b sig[w,b,:] (.) P_dir[s,b,:]        sig = sigmoid(C) as a [2R][B][d] table, P = H [V_f | V_b]
// The coefficient is a vector over the OUTPUT channels, applied after the basis transform, so the plain basis layer's
// "aggregate, then transform" regrouping does not hold: the walks gather the transformed rows P (B*d floats per
// message) instead of H rows.
//   forward   k_diagcoef_fwd  destination-major pull: out[o] += norm * m (out holds the masked self-loop term)
//   backward  k_diagcoef_dp   source-major: dP_dir[u,b,:] = sum_{m from u} norm sig[w,b,:] (.) G[dst]; a run of one
//                             (source, weight id) sums G once and applies sig once
//             k_diagcoef_dc   weight-id-major (rows = sources): dC[w,b,:] = sig'(C) (.) sum norm P_dir[src,b,:] (.) G[dst];
//                             the item's partial sum stays in registers and is flushed once per item
// The sums across split rows and across items of one weight id use fp32 vector reductions (not deterministic).
#include <cuda_runtime.h>

#include "kernels.cuh"

#define FULL 0xffffffffu

namespace {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
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

constexpr int U_MSG = 4;  // messages whose gathered rows are in flight per lane (backward source-major walk)

__global__ void k_diagcoef_sigmoid(const float* __restrict__ Cf, const float* __restrict__ Cb, int64_t n_half,
                                   float* __restrict__ sig) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < 2 * n_half;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float c = i < n_half ? __ldg(Cf + i) : __ldg(Cb + (i - n_half));
    sig[i] = 1.f / (1.f + expf(-c));
  }
}

// A warp owns one destination-major work item and one column slab of NV*128 columns; a lane owns NV float4 quads.
template <int NV>
__global__ void __launch_bounds__(RGCN_THREADS)
    k_diagcoef_fwd(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                   const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ P,
                   const float* __restrict__ sig, int B, int d, int half, float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, row = itv.z, split = itv.w;
  if (beg == end) return;
  const size_t dB = (size_t)d * B;
  bool ok[NV];
  float4 acc[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = c0 + 4 * (lane + 32 * k) < d;
    acc[k] = zero4();
  }
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
      const int v = __shfl_sync(FULL, my_v, t);
      const int rw = __shfl_sync(FULL, my_rw, t);
      const float nm = __shfl_sync(FULL, my_nm, t);
      const float* pr = P + (size_t)v * 2 * dB + (rw >= half ? dB : 0) + c0;
      const float* sr = sig + (size_t)rw * dB + c0;
      float4 m[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) m[k] = zero4();
#pragma unroll 2
      for (int b = 0; b < B; ++b) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          if (ok[k]) {
            const int lc = (int)((size_t)b * d) + 4 * (lane + 32 * k);
            fma4v(m[k], ldg4(sr + lc), ldg4(pr + lc));
          }
        }
      }
#pragma unroll
      for (int k = 0; k < NV; ++k) fma4(acc[k], nm, m[k]);
    }
  }
  float* po = out + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!ok[k]) continue;
    float* p = po + 4 * (lane + 32 * k);
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
}

// out = act(out + b)
__global__ void k_diagcoef_bias_act(float* __restrict__ out, const float* __restrict__ bias, int64_t n4, int d4,
                                    int relu) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 o = reinterpret_cast<float4*>(out)[i];
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + (int)(i % d4));
    o.x += b.x;
    o.y += b.y;
    o.z += b.z;
    o.w += b.w;
    if (relu) {
      o.x = fmaxf(o.x, 0.f);
      o.y = fmaxf(o.y, 0.f);
      o.z = fmaxf(o.z, 0.f);
      o.w = fmaxf(o.w, 0.f);
    }
    reinterpret_cast<float4*>(out)[i] = o;
  }
}

// db[c] += sum over rows of G[:, c]: a thread owns one column quad (grid.y = column blocks of 128 quads), a block a
// strided set of rows
__global__ void k_diagcoef_colsum(const float* __restrict__ G, int64_t V, int d4, float* __restrict__ db) {
  const int q = blockIdx.y * blockDim.x + threadIdx.x;
  if (q >= d4) return;
  float4 s = zero4();
  for (int64_t r = blockIdx.x; r < V; r += gridDim.x) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(G) + r * d4 + q);
    s.x += g.x;
    s.y += g.y;
    s.z += g.z;
    s.w += g.w;
  }
  red4(db + 4 * q, s);
}

// Source-major walk (rows = sources, nbr = destinations, X = G).  BC bases per pass over the item; each run of one
// weight id pre-sums xs = sum norm G[dst] and adds sig[w,b,:] (.) xs into the row's accumulators of its direction.
// Rows covered by one item write both directions (zeros where there is no message); split rows are pre-zeroed and
// reduced into.
template <int BC, int NV>
__global__ void __launch_bounds__(RGCN_THREADS, 1)
    k_diagcoef_dp(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                  const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ G,
                  const float* __restrict__ sig, int B, int d, int half, float* __restrict__ dP) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, row = itv.z, split = itv.w;
  const size_t dB = (size_t)d * B;

  for (int b0 = 0; b0 < B; b0 += BC) {
    float4 acc[BC][NV], xs[NV];
#pragma unroll
    for (int b = 0; b < BC; ++b)
#pragma unroll
      for (int k = 0; k < NV; ++k) acc[b][k] = zero4();
#pragma unroll
    for (int k = 0; k < NV; ++k) xs[k] = zero4();
    int cur = -1, curdir = -1, written = 0;

    auto write_out = [&](int dir) {
      float* ad = dP + (size_t)row * 2 * dB + (size_t)dir * dB;
#pragma unroll
      for (int b = 0; b < BC; ++b) {
        if (b0 + b < B) {
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            const int col = c0 + 4 * (lane + 32 * k);
            if (col < d) {
              float* p = ad + (size_t)(b0 + b) * d + col;
              if (split >= 0)
                red4(p, acc[b][k]);
              else
                *reinterpret_cast<float4*>(p) = acc[b][k];
            }
          }
        }
      }
      written |= (1 << dir);
    };
    auto flush = [&](int w) {
      const int dir = (w >= half) ? 1 : 0;
      if (dir != curdir) {
        if (curdir >= 0) write_out(curdir);
#pragma unroll
        for (int b = 0; b < BC; ++b)
#pragma unroll
          for (int k = 0; k < NV; ++k) acc[b][k] = zero4();
        curdir = dir;
      }
      const float* sr = sig + (size_t)w * dB + c0;
#pragma unroll
      for (int b = 0; b < BC; ++b) {
        if (b0 + b < B) {
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            const int lc = 4 * (lane + 32 * k);
            if (c0 + lc < d) fma4v(acc[b][k], ldg4(sr + (size_t)(b0 + b) * d + lc), xs[k]);
          }
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
          const float* xr = G + (size_t)v * d + c0;
#pragma unroll
          for (int k = 0; k < NV; ++k) {
            const int lc = 4 * (lane + 32 * k);
            x[u][k] = (c0 + lc < d) ? ldg4(xr + lc) : zero4();
          }
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
          }
        }
      }
    }
    if (cur >= 0) flush(cur);
    if (curdir >= 0) write_out(curdir);
    if (split < 0) {
      // directions that received no message: explicit zeros (dP is not pre-zeroed for these rows)
#pragma unroll
      for (int b = 0; b < BC; ++b)
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[b][k] = zero4();
      if (!(written & 1)) write_out(0);
      if (!(written & 2)) write_out(1);
    }
  }
}

// Weight-id-major walk over the source-row view (item.row = weight id w; r_row = source, r_nbr = destination):
// acc[b] = sum_m norm_m P_dir[src_m, b, :] (.) G[dst_m, :] over the item's messages, BC bases per pass, then ONE
// flush per item and pass: dC_dir[w mod R, b, :] += sig (1 - sig) (.) acc  (dCf / dCb zeroed by the caller).
template <int BC, int NV>
__global__ void __launch_bounds__(RGCN_THREADS, 1)
    k_diagcoef_dc(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ r_row,
                  const int32_t* __restrict__ r_nbr, const float* __restrict__ r_norm, const float* __restrict__ P,
                  const float* __restrict__ G, const float* __restrict__ sig, int B, int d, int half,
                  float* __restrict__ dCf, float* __restrict__ dCb) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, w = itv.z;
  if (beg == end) return;
  const size_t dB = (size_t)d * B;
  const int dir = w >= half ? 1 : 0;
  float* dC = (dir ? dCb : dCf) + (size_t)(w - dir * half) * dB + c0;
  const float* sr = sig + (size_t)w * dB + c0;

  for (int b0 = 0; b0 < B; b0 += BC) {
    float4 acc[BC][NV];
#pragma unroll
    for (int b = 0; b < BC; ++b)
#pragma unroll
      for (int k = 0; k < NV; ++k) acc[b][k] = zero4();
    for (int base = beg; base < end; base += 32) {
      const int n = min(32, end - base);
      int my_src = 0, my_dst = 0;
      float my_nm = 0.f;
      if (lane < n) {
        my_src = __ldg(r_row + base + lane);
        my_dst = __ldg(r_nbr + base + lane);
        my_nm = __ldg(r_norm + base + lane);
      }
      for (int t = 0; t < n; ++t) {
        const int src = __shfl_sync(FULL, my_src, t);
        const int dst = __shfl_sync(FULL, my_dst, t);
        const float nm = __shfl_sync(FULL, my_nm, t);
        const float* gr = G + (size_t)dst * d + c0;
        const float* pr = P + (size_t)src * 2 * dB + (size_t)dir * dB + c0;
        float4 g[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const int lc = 4 * (lane + 32 * k);
          g[k] = zero4();
          if (c0 + lc < d) fma4(g[k], nm, ldg4(gr + lc));
        }
#pragma unroll
        for (int b = 0; b < BC; ++b) {
          if (b0 + b < B) {
#pragma unroll
            for (int k = 0; k < NV; ++k) {
              const int lc = 4 * (lane + 32 * k);
              if (c0 + lc < d) fma4v(acc[b][k], g[k], ldg4(pr + (size_t)(b0 + b) * d + lc));
            }
          }
        }
      }
    }
#pragma unroll
    for (int b = 0; b < BC; ++b) {
      if (b0 + b < B) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const int lc = 4 * (lane + 32 * k);
          if (c0 + lc < d) {
            const size_t off = (size_t)(b0 + b) * d + lc;
            const float4 s = ldg4(sr + off);
            const float4 a = acc[b][k];
            red4(dC + off, make_float4(s.x * (1.f - s.x) * a.x, s.y * (1.f - s.y) * a.y, s.z * (1.f - s.z) * a.z,
                                       s.w * (1.f - s.w) * a.w));
          }
        }
      }
    }
  }
}

int grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = 132 * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int pick_nv(int d, int cap) {
  const int nv = (d + 127) / 128;
  return nv > cap ? cap : nv;
}

}  // namespace

int launch_diagcoef_sigmoid(const float* Cf, const float* Cb, int64_t n_half, float* sig, cudaStream_t st) {
  if (n_half == 0) return RGCN_OK;
  k_diagcoef_sigmoid<<<grid_for(2 * n_half, 256), 256, 0, st>>>(Cf, Cb, n_half, sig);
  return check_launch("k_diagcoef_sigmoid");
}

int launch_diagcoef_fwd(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                        const float* P, const float* sig, int B, int d, int n_relw, float* out, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int nv = pick_nv(d, 4);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  const int half = n_relw / 2;
#define FWD(NV_) \
  k_diagcoef_fwd<NV_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, P, sig, B, d, half, out)
  switch (nv) {
    case 1: FWD(1); break;
    case 2: FWD(2); break;
    case 3: FWD(3); break;
    default: FWD(4); break;
  }
#undef FWD
  return check_launch("k_diagcoef_fwd");
}

int launch_diagcoef_bias_act(float* out, const float* bias, int64_t rows, int d, int relu, cudaStream_t st) {
  const int64_t n4 = rows * d / 4;
  if (n4 == 0) return RGCN_OK;
  k_diagcoef_bias_act<<<grid_for(n4, 256), 256, 0, st>>>(out, bias, n4, d / 4, relu);
  return check_launch("k_diagcoef_bias_act");
}

int launch_diagcoef_colsum(const float* G, int64_t rows, int d, float* db, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(db, 0, (size_t)d * sizeof(float), st), "memset(db)");
  if (rc || rows == 0) return rc;
  const int d4 = d / 4;
  dim3 grid((unsigned)(rows < 1024 ? rows : 1024), (d4 + 127) / 128);
  k_diagcoef_colsum<<<grid, 128, 0, st>>>(G, rows, d4, db);
  return check_launch("k_diagcoef_colsum");
}

// bases per pass: all of them for B in {1, 2, 5}, else passes of 4; quads per lane at most 2 (column slabs of 256),
// which keeps the BC * NV accumulators and the rows in flight inside the register file
static int diagcoef_bc(int B) { return (B == 1 || B == 2 || B == 5) ? B : 4; }

template <int BC>
static int launch_dp_t(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* G, const float* sig, int B, int d, int half, float* dP, cudaStream_t st) {
  const int nv = pick_nv(d, 2);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  if (nv == 1)
    k_diagcoef_dp<BC, 1><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP);
  else
    k_diagcoef_dp<BC, 2><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP);
  return check_launch("k_diagcoef_dp");
}

int launch_diagcoef_dp(const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw, const float* norm,
                       const float* G, const float* sig, int B, int d, int n_relw, float* dP, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int half = n_relw / 2;
  switch (diagcoef_bc(B)) {
    case 1: return launch_dp_t<1>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP, st);
    case 2: return launch_dp_t<2>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP, st);
    case 5: return launch_dp_t<5>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP, st);
    default: return launch_dp_t<4>(items, n_items, nbr, relw, norm, G, sig, B, d, half, dP, st);
  }
}

template <int BC>
static int launch_dc_t(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                       const float* r_norm, const float* P, const float* G, const float* sig, int B, int d, int half,
                       float* dCf, float* dCb, cudaStream_t st) {
  const int nv = pick_nv(d, 2);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  if (nv == 1)
    k_diagcoef_dc<BC, 1><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half,
                                                         dCf, dCb);
  else
    k_diagcoef_dc<BC, 2><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half,
                                                         dCf, dCb);
  return check_launch("k_diagcoef_dc");
}

int launch_diagcoef_dc(const WorkItem* items, int n_items, const int32_t* r_row, const int32_t* r_nbr,
                       const float* r_norm, const float* P, const float* G, const float* sig, int B, int d, int n_relw,
                       float* dCf, float* dCb, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int half = n_relw / 2;
  switch (diagcoef_bc(B)) {
    case 1: return launch_dc_t<1>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half, dCf, dCb, st);
    case 2: return launch_dc_t<2>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half, dCf, dCb, st);
    case 5: return launch_dc_t<5>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half, dCf, dCb, st);
    default: return launch_dc_t<4>(items, n_items, r_row, r_nbr, r_norm, P, G, sig, B, d, half, dCf, dCb, st);
  }
}
