// compgcn.cu -- message walks of the CompGCN layer (Name=compgcn, Vashishth et al., ICLR 2020) for sm_90a.
// One message s -> o of weight id w (forward relation r: w = r, its inverse: w = R + r) carries
//   m = norm * phi(H[s], Z[w])        phi = h (.) z  (OP 0, mult)  or  h - z  (OP 1, sub);  Z : [2R][d]
// Both compositions are linear in h inside a run of one weight id:  sum n (h (.) z) = z (.) sum n h  and
// sum n (h - z) = sum n h - (sum n) z,  so a walk sums norm * H[src] (and norm) over the run and composes once.
//   forward   k_compgcn_fwd  destination-major pull.  Writes the GEMM operand Cat [V_dst, 3d] =
//                            [ A_f | A_b | phi(H[v], z_loop) ] / 3 with the dropout mask and 1/keep on the two message
//                            slabs.  by_dst is sorted by (dst, weight id), so a row's forward runs come before its
//                            backward runs: one accumulator, stored to the forward slab when the first backward run
//                            starts.  Items of split rows add their partial slabs with vector reductions into rows the
//                            caller zeroed; the first item of a row writes its loop slab.
//   backward  k_compgcn_bwd  ONE source-major walk over dCat = G W_cat^T.  Per (u, w) run it sums
//                            S = sum norm dCat_slab(w)[dst] (mask applied per message; 1/keep and 1/3 once per run), then
//                              mult: dH[u] += Z[w] (.) S,  dZ[w] += H[u] (.) S      sub: dH[u] += S,  dZ[w] -= S
//                            and the first item of every row u < V_dst adds the loop term of g_L = dCat[u, 2d:3d] / 3:
//                              mult: dH[u] += z_loop (.) g_L,  dz_loop += H[u] (.) g_L      sub: dH[u] += g_L,  dz_loop -= g_L
//                            Halo rows [V_dst, V_src) get message gradients only.
// The reductions across split rows, across runs of one weight id and into dz_loop are fp32 atomics (the summation
// order is not deterministic).
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
__device__ __forceinline__ float4 scale4(const float4& a, float s) {
  return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}
__device__ __forceinline__ float4 mul4(const float4& a, const float4& b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 neg4(const float4& a) { return make_float4(-a.x, -a.y, -a.z, -a.w); }
__device__ __forceinline__ void add4(float4& a, const float4& b) {
  a.x += b.x;
  a.y += b.y;
  a.z += b.z;
  a.w += b.w;
}
__device__ __forceinline__ float4 mask4(const float4& x, uchar4 m) {
  return make_float4(m.x ? x.x : 0.f, m.y ? x.y : 0.f, m.z ? x.z : 0.f, m.w ? x.w : 0.f);
}
// phi(h, z)
template <int OP>
__device__ __forceinline__ float4 compose4(const float4& h, const float4& z) {
  return OP == 0 ? mul4(h, z) : make_float4(h.x - z.x, h.y - z.y, h.z - z.z, h.w - z.w);
}
// the first work item of its row: items are in row order, so the item before it belongs to another row
__device__ __forceinline__ bool first_of_row(const WorkItem* items, int item, int row) {
  return item == 0 || __ldg(&items[item - 1].row) != row;
}

constexpr int U_MSG = 4;  // messages whose gathered rows are in flight per lane
constexpr float THIRD = 1.0f / 3.0f;

// A warp owns one destination-major work item and one column slab of NV*128 columns; a lane owns NV float4 quads.
// Items of rows without messages exist (beg == end): they write zero message slabs and the loop slab.
template <int NV, int OP>
__global__ void __launch_bounds__(RGCN_THREADS, NV == 4 ? 1 : 2)
    k_compgcn_fwd(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                  const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ H,
                  const float* __restrict__ Z, const float* __restrict__ zloop, int d, int half,
                  const uint8_t* __restrict__ mask, float inv_keep, float* __restrict__ Cat) {
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
  float* crow = Cat + (size_t)row * 3 * d + c0;
  float ns = 0.f;  // sum of norm over the run (sub)
  int cur = -1;
  auto compose_run = [&](int w) {
    const float* zr = Z + (size_t)w * d + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (!ok[k]) continue;
      const float4 z = ldg4(zr + 4 * (lane + 32 * k));
      if (OP == 0) {
        fma4v(acc[k], z, xs[k]);
      } else {
        add4(acc[k], xs[k]);
        fma4(acc[k], -ns, z);
      }
    }
  };
  // acc / 3 (masked, / keep) into message slab `dir`; split items skip slabs they have no runs for
  auto emit = [&](int dir, bool have) {
    if (split >= 0 && !have) return;
    const uint8_t* pm = mask ? mask + (size_t)row * 2 * d + (size_t)dir * d + c0 : nullptr;
    const float s = pm ? THIRD * inv_keep : THIRD;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (!ok[k]) continue;
      const int lc = 4 * (lane + 32 * k);
      float4 v = scale4(acc[k], s);
      if (pm) v = mask4(v, *reinterpret_cast<const uchar4*>(pm + lc));
      float* p = crow + (size_t)dir * d + lc;
      if (split >= 0)
        red4(p, v);
      else
        *reinterpret_cast<float4*>(p) = v;
    }
  };

  int dir = 0;
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
            if (cur >= 0) compose_run(cur);
            if (rw[u] >= half && dir == 0) {  // the first backward run: the forward slab is complete
              emit(0, cur >= 0);
#pragma unroll
              for (int k = 0; k < NV; ++k) acc[k] = zero4();
              dir = 1;
            }
            cur = rw[u];
            ns = 0.f;
#pragma unroll
            for (int k = 0; k < NV; ++k) xs[k] = zero4();
          }
          ns += nm[u];
#pragma unroll
          for (int k = 0; k < NV; ++k) fma4(xs[k], nm[u], x[u][k]);
        }
      }
    }
  }
  if (cur >= 0) compose_run(cur);
  if (dir == 0) {
    emit(0, cur >= 0);
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = zero4();
    emit(1, false);
  } else {
    emit(1, true);
  }

  if (!first_of_row(items, item, row)) return;
  const float* hr = H + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!ok[k]) continue;
    const int lc = 4 * (lane + 32 * k);
    *reinterpret_cast<float4*>(crow + 2 * (size_t)d + lc) =
        scale4(compose4<OP>(ldg4(hr + lc), ldg4(zloop + c0 + lc)), THIRD);
  }
}

// Source-major walk (rows = sources u, nbr = destinations, X = dCat).  dZ and dzloop hold zeros (or the values to
// accumulate into); the rows of dH that several items cover hold zeros.
template <int NV, int OP>
__global__ void __launch_bounds__(RGCN_THREADS, 1)
    k_compgcn_bwd(const WorkItem* __restrict__ items, int n_items, const int32_t* __restrict__ nbr,
                  const int32_t* __restrict__ relw, const float* __restrict__ norm, const float* __restrict__ dCat,
                  const float* __restrict__ H, const float* __restrict__ Z, const float* __restrict__ zloop, int d,
                  int half, int V_dst, const uint8_t* __restrict__ mask, float inv_keep, float* __restrict__ dH,
                  float* __restrict__ dZ, float* __restrict__ dzloop) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int item = blockIdx.x * RGCN_WARPS_PER_BLOCK + warp;
  if (item >= n_items) return;
  const int c0 = blockIdx.y * (NV * 128);
  const int4 itv = __ldg(reinterpret_cast<const int4*>(items) + item);
  const int beg = itv.x, end = itv.y, row = itv.z, split = itv.w;
  const size_t ldc = 3 * (size_t)d;
  const float s_msg = mask ? THIRD * inv_keep : THIRD;
  bool ok[NV];
  float4 acc[NV], xs[NV], h[NV];
  const float* hr = H + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    ok[k] = c0 + 4 * (lane + 32 * k) < d;
    acc[k] = xs[k] = zero4();
    h[k] = (OP == 0 && ok[k]) ? ldg4(hr + 4 * (lane + 32 * k)) : zero4();
  }
  int cur = -1;
  auto flush = [&](int w) {
    const float* zr = Z + (size_t)w * d + c0;
    float* dz = dZ + (size_t)w * d + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (!ok[k]) continue;
      const int lc = 4 * (lane + 32 * k);
      const float4 S = scale4(xs[k], s_msg);
      if (OP == 0) {
        fma4v(acc[k], ldg4(zr + lc), S);
        red4(dz + lc, mul4(h[k], S));
      } else {
        add4(acc[k], S);
        red4(dz + lc, neg4(S));
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
        const size_t off = (rw[u] >= half ? (size_t)d : 0) + c0;
        const float* gr = dCat + (size_t)v * ldc + off;
        const uint8_t* pm = mask ? mask + (size_t)v * 2 * d + off : nullptr;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const int lc = 4 * (lane + 32 * k);
          x[u][k] = ok[k] ? ldg4(gr + lc) : zero4();
          if (pm && ok[k]) x[u][k] = mask4(x[u][k], __ldg(reinterpret_cast<const uchar4*>(pm + lc)));
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

  if (row < V_dst && first_of_row(items, item, row)) {
    const float* gl = dCat + (size_t)row * ldc + 2 * (size_t)d + c0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (!ok[k]) continue;
      const int lc = 4 * (lane + 32 * k);
      const float4 g = scale4(ldg4(gl + lc), THIRD);
      if (OP == 0) {
        fma4v(acc[k], ldg4(zloop + c0 + lc), g);
        red4(dzloop + c0 + lc, mul4(h[k], g));
      } else {
        add4(acc[k], g);
        red4(dzloop + c0 + lc, neg4(g));
      }
    }
  }

  float* pd = dH + (size_t)row * d + c0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (!ok[k]) continue;
    float* p = pd + 4 * (lane + 32 * k);
    if (split >= 0)
      red4(p, acc[k]);
    else
      *reinterpret_cast<float4*>(p) = acc[k];
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

int launch_compgcn_fwd(int op, const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                       const float* norm, const float* H, const float* Z, const float* zloop, int d, int n_relw,
                       const uint8_t* mask, float inv_keep, float* Cat, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int nv = pick_nv(d);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  const int half = n_relw / 2;
#define FWD(NV_, OP_)                                                                                             \
  k_compgcn_fwd<NV_, OP_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, H, Z, zloop, d, half, mask, \
                                                         inv_keep, Cat)
#define FWD_NV(OP_)               \
  switch (nv) {                   \
    case 1: FWD(1, OP_); break;   \
    case 2: FWD(2, OP_); break;   \
    case 3: FWD(3, OP_); break;   \
    default: FWD(4, OP_); break;  \
  }
  if (op == 0) {
    FWD_NV(0)
  } else {
    FWD_NV(1)
  }
#undef FWD_NV
#undef FWD
  return check_launch("k_compgcn_fwd");
}

int launch_compgcn_bwd(int op, const WorkItem* items, int n_items, const int32_t* nbr, const int32_t* relw,
                       const float* norm, const float* dCat, const float* H, const float* Z, const float* zloop, int d,
                       int n_relw, int V_dst, const uint8_t* mask, float inv_keep, float* dH, float* dZ,
                       float* dzloop, cudaStream_t st) {
  if (n_items == 0) return RGCN_OK;
  const int nv = pick_nv(d);
  dim3 grid((n_items + RGCN_WARPS_PER_BLOCK - 1) / RGCN_WARPS_PER_BLOCK, (d + nv * 128 - 1) / (nv * 128));
  const int half = n_relw / 2;
#define BWD(NV_, OP_)                                                                                          \
  k_compgcn_bwd<NV_, OP_><<<grid, RGCN_THREADS, 0, st>>>(items, n_items, nbr, relw, norm, dCat, H, Z, zloop, d, \
                                                         half, V_dst, mask, inv_keep, dH, dZ, dzloop)
#define BWD_NV(OP_)               \
  switch (nv) {                   \
    case 1: BWD(1, OP_); break;   \
    case 2: BWD(2, OP_); break;   \
    case 3: BWD(3, OP_); break;   \
    default: BWD(4, OP_); break;  \
  }
  if (op == 0) {
    BWD_NV(0)
  } else {
    BWD_NV(1)
  }
#undef BWD_NV
#undef BWD
  return check_launch("k_compgcn_bwd");
}
