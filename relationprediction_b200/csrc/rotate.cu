// rotate.cu -- RotatE (Sun et al., ICLR 2019) triple scorer, loss, backward and all-entity ranking for sm_90a.
// Semantics in DESIGN.md section 1.  Entity rows are [re | im] (h = d / 2 columns each), the phases theta of relation r
// are the first h columns of its row, and with a = codes[s], c = codes[o]:
//   u_k = a_k e^{i theta_k} - c_k,   D = sum_{k<h} |u_k|,   E = gamma - D.
// The scorer and its backward have the ComplEx shape (a warp owns a triple, a lane the column pairs (k, k + h)).  The
// ranking cannot be a GEMM -- a modulus is not a product -- so k_rotate_rank is a tiled all-pairs distance kernel on
// the CUDA cores.
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

// loss_acc[0] += sum of per-triple cross-entropy terms, loss_acc[1] += sum of squares of the two entity rows
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_fwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, float gamma, float* __restrict__ energies,
                 float* __restrict__ loss_acc) {
  // per-warp sums, kept by lane 0 in shared memory: as registers live across the whole loop, ptxas spills them
  __shared__ double sh_l[8], sh_q[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const RotateRows<W> rows{gamma};
  if (lane == 0) sh_l[warp] = sh_q[warp] = 0.0;
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float e = 0.f, q = 0.f;
    rows.partial(codes, rel, d, s, r, o, lane, e, q);
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

__global__ void k_rotate_finalize(float* loss_acc, float inv_n, float inv_nd) {
  loss_acc[0] *= inv_n;
  loss_acc[1] *= inv_nd;
}

// With g = dL/dE, m = |u|, w = u / m (0 where m = 0), p = a e^{i theta} and dE = -dD:
//   dc = g w,   da = -g [w_re cos + w_im sin, -w_re sin + w_im cos],   dtheta = -g (w_im p_re - w_re p_im)
// plus c_reg x on the entity rows (the L2 term).  Columns h..d-1 of the relation row get nothing.
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_bwd(const float* __restrict__ codes, const float* __restrict__ rel, int d, const int32_t* __restrict__ X,
                 int64_t N, const float* __restrict__ Y, const float* __restrict__ energies, float g_loss_over_n,
                 float c_reg, const float* __restrict__ g_scale, const float* __restrict__ g_energy,
                 float* __restrict__ dcodes, float* __restrict__ drel, float* __restrict__ rel_slice_sumsq) {
  if (g_scale) {
    g_loss_over_n *= __ldg(g_scale + 0);
    c_reg *= __ldg(g_scale + 1);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  float slice_sq = 0.f;  // sum over this warp's triples of |gradient slice of the relation row|^2 (IndexedSlices norm)
  for (int64_t n = (int64_t)blockIdx.x * 8 + warp; n < N; n += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * n), r = __ldg(X + 3 * n + 1), o = __ldg(X + 3 * n + 2);
    float gx = g_energy ? __ldg(g_energy + n) : 0.f;
    if (Y) {
      const float e = __ldg(energies + n);
      gx += g_loss_over_n * (1.f / (1.f + expf(-e)) - __ldg(Y + n));
    }
    const float* e1 = codes + (size_t)s * d;
    const float* th = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    float* g1 = dcodes + (size_t)s * d;
    float* gr = drel + (size_t)r * d;
    float* g2 = dcodes + (size_t)o * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float ar[W], ai[W], t[W], cr[W], ci[W];
      Vec<W>::load(e1 + k, ar), Vec<W>::load(e1 + h + k, ai);
      Vec<W>::load(th + k, t);
      Vec<W>::load(e2 + k, cr), Vec<W>::load(e2 + h + k, ci);
      float dar[W], dai[W], dt[W], dcr[W], dci[W];
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float ur, ui, sn, cs;
        rotate_residual(ar[j], ai[j], t[j], cr[j], ci[j], ur, ui, sn, cs);
        const float m = rotate_modulus(ur, ui);
        const float gm = m > 0.f ? gx / m : 0.f;   // g / m: the subgradient 0 where u = 0
        const float wr = gm * ur, wi = gm * ui;     // g w
        const float pr = fmaf(ar[j], cs, -ai[j] * sn), pi = fmaf(ar[j], sn, ai[j] * cs);
        dcr[j] = fmaf(c_reg, cr[j], wr);
        dci[j] = fmaf(c_reg, ci[j], wi);
        dar[j] = fmaf(c_reg, ar[j], -fmaf(wr, cs, wi * sn));
        dai[j] = fmaf(c_reg, ai[j], -fmaf(wi, cs, -wr * sn));
        dt[j] = fmaf(wr, pi, -wi * pr);
        slice_sq += dt[j] * dt[j];
      }
      Vec<W>::red(g1 + k, dar), Vec<W>::red(g1 + h + k, dai);
      Vec<W>::red(gr + k, dt);
      Vec<W>::red(g2 + k, dcr), Vec<W>::red(g2 + h + k, dci);
    }
  }
  if (rel_slice_sumsq) {  // warp-uniform
    slice_sq = warp_sum(slice_sq);
    if (lane == 0 && slice_sq != 0.f) atomicAdd(rel_slice_sumsq, slice_sq);
  }
}

// ---- all-entity ranking by distance -------------------------------------------------------------------------------
// D = sum_k |q_k - v_k| in one fixed order: ascending k in chunks of RK_KC column pairs, each chunk summed from 0 by
// rotate_dist_step and its sum added to the total, every rounding pinned (no contraction choice is left to the
// compiler).  The gold's distance (k_rotate_rank_prepare) and every candidate's (k_rotate_rank) are formed this way on
// one thread each, so the gold ties with itself -- and duplicated rows tie -- bit for bit; zero-padded columns add +0.
// The chunked sum keeps the float32 error of D near 440 (d = 500) several times below that of one running sum, which
// decides how many near-ties float32 ranks differently from float64.
constexpr int RK_TILE = 128, RK_KC = 8, RK_LD = RK_TILE + 4;   // +4: spread the transposing writes over the banks
constexpr int RK_STAGE = 2 * RK_KC * RK_LD;                    // floats of one operand's chunk

__device__ __forceinline__ float rotate_dist_step(float qr, float qi, float vr, float vi, float acc) {
  return __fadd_rn(acc, rotate_modulus(__fsub_rn(qr, vr), __fsub_rn(qi, vi)));
}

// One warp per query t.  side 1 (objects corrupted): q = codes[s] e^{i theta}, gold o; side 0 (subjects corrupted):
// q = codes[o] e^{-i theta}, gold s -- |a e^{i theta} - c| = |a - c e^{-i theta}|.  Lane 0 then sums the gold's
// distance sequentially from the float32 q just stored, as k_rotate_rank will.
template <int W>
__global__ void __launch_bounds__(256)
    k_rotate_rank_prepare(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                          const int32_t* __restrict__ X, int64_t n, int side, float* __restrict__ Q,
                          float* __restrict__ gold_D, int32_t* __restrict__ gold_col) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = d >> 1;
  for (int64_t t = (int64_t)blockIdx.x * 8 + warp; t < n; t += (int64_t)gridDim.x * 8) {
    const int s = __ldg(X + 3 * t), r = __ldg(X + 3 * t + 1), o = __ldg(X + 3 * t + 2);
    const int kept = side == 0 ? o : s, gold = side == 0 ? s : o;
    const float* ek = codes + (size_t)kept * d;
    const float* th = rel + (size_t)r * d;
    float* q = Q + (size_t)t * d;
    for (int k = lane * W; k < h; k += 32 * W) {
      float kr[W], ki[W], tt[W], qr[W], qi[W];
      Vec<W>::load(ek + k, kr), Vec<W>::load(ek + h + k, ki);
      Vec<W>::load(th + k, tt);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float sn, cs;
        sincosf(tt[j], &sn, &cs);
        if (side == 0) sn = -sn;
        qr[j] = fmaf(kr[j], cs, -ki[j] * sn);
        qi[j] = fmaf(kr[j], sn, ki[j] * cs);
      }
      Vec<W>::store(q + k, qr), Vec<W>::store(q + h + k, qi);
    }
    __syncwarp();   // the warp's stores of q are visible to lane 0
    if (lane == 0) {
      const float* g = codes + (size_t)gold * d;
      float D = 0.f;
      for (int k0 = 0; k0 < h; k0 += RK_KC) {
        float part = 0.f;
        for (int k = k0; k < min(k0 + RK_KC, h); ++k)
          part = rotate_dist_step(q[k], q[h + k], __ldg(g + k), __ldg(g + h + k), part);
        D = __fadd_rn(D, part);
      }
      gold_D[t] = D;
      gold_col[t] = gold;
    }
    __syncwarp();
  }
}

// The tiled all-pairs distance kernel: a CTA owns 128 queries x 128 entities, 256 threads as a 16 x 16 grid, each
// thread an 8 x 8 register tile (rows ty*4 + 64 i + a, columns tx*4 + 64 j + b, i, j < 2, a, b < 4).  The k range goes
// in chunks of RK_KC column pairs; each chunk of both operands is staged k-major ([re 0..KC-1 | im 0..KC-1][row]) in
// shared memory by 4-byte cp.async, double-buffered, with zero fill past n / V / h.  The epilogue counts, per query
// row, the columns < V with D <= gold_D (or the gold itself), and among them the known ones; the 16 threads of a row
// sum by shuffles and add once per row and CTA.

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const unsigned saddr = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(saddr), "l"(src), "r"(valid ? 4 : 0) : "memory");
}

// chunk k0 of rows row0.. of a [rows, d] operand into stage (thread tid copies 8 of its 128 x 16 floats)
__device__ __forceinline__ void rk_load_chunk(float* stage, const float* __restrict__ A, int64_t rows, int64_t row0,
                                              int d, int h, int k0, int tid) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int e = tid + 256 * i, row = e >> 4, c = e & 15, kk = c & 7;
    const int64_t gr = row0 + row;
    const bool valid = gr < rows && k0 + kk < h;
    const float* src = valid ? A + (size_t)gr * d + (c < RK_KC ? 0 : h) + k0 + kk : A;
    cp_async4(stage + c * RK_LD + row, src, valid);
  }
}

__global__ void __launch_bounds__(256, 1)
    k_rotate_rank(const float* __restrict__ Q, const float* __restrict__ codes, int V, int d, int64_t n,
                  const float* __restrict__ gold_D, const int32_t* __restrict__ gold_col,
                  const uint32_t* __restrict__ known, int words, int32_t* __restrict__ raw_cnt,
                  int32_t* __restrict__ known_cnt) {
  __shared__ __align__(16) float sq[2][RK_STAGE];
  __shared__ __align__(16) float sv[2][RK_STAGE];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int h = d >> 1, chunks = (h + RK_KC - 1) / RK_KC;
  const int64_t col0 = (int64_t)blockIdx.x * RK_TILE;
  for (int64_t row0 = (int64_t)blockIdx.y * RK_TILE; row0 < n; row0 += (int64_t)gridDim.y * RK_TILE) {
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    rk_load_chunk(sq[0], Q, n, row0, d, h, 0, tid);
    rk_load_chunk(sv[0], codes, V, col0, d, h, 0, tid);
    asm volatile("cp.async.commit_group;" ::: "memory");
    for (int c = 0; c < chunks; ++c) {
      if (c + 1 < chunks) {
        rk_load_chunk(sq[(c + 1) & 1], Q, n, row0, d, h, (c + 1) * RK_KC, tid);
        rk_load_chunk(sv[(c + 1) & 1], codes, V, col0, d, h, (c + 1) * RK_KC, tid);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 1;" ::: "memory");
      __syncthreads();
      const float* a = sq[c & 1];
      const float* b = sv[c & 1];
      float part[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) part[i][j] = 0.f;
#pragma unroll 1
      for (int kk = 0; kk < RK_KC; ++kk) {
        float qr[8], qi[8], vr[8], vi[8];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float4 x = *reinterpret_cast<const float4*>(a + kk * RK_LD + ty * 4 + 64 * i);
          const float4 y = *reinterpret_cast<const float4*>(a + (RK_KC + kk) * RK_LD + ty * 4 + 64 * i);
          const float4 z = *reinterpret_cast<const float4*>(b + kk * RK_LD + tx * 4 + 64 * i);
          const float4 w = *reinterpret_cast<const float4*>(b + (RK_KC + kk) * RK_LD + tx * 4 + 64 * i);
          qr[4 * i] = x.x, qr[4 * i + 1] = x.y, qr[4 * i + 2] = x.z, qr[4 * i + 3] = x.w;
          qi[4 * i] = y.x, qi[4 * i + 1] = y.y, qi[4 * i + 2] = y.z, qi[4 * i + 3] = y.w;
          vr[4 * i] = z.x, vr[4 * i + 1] = z.y, vr[4 * i + 2] = z.z, vr[4 * i + 3] = z.w;
          vi[4 * i] = w.x, vi[4 * i + 1] = w.y, vi[4 * i + 2] = w.z, vi[4 * i + 3] = w.w;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) part[i][j] = rotate_dist_step(qr[i], qi[i], vr[j], vi[j], part[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = __fadd_rn(acc[i][j], part[i][j]);
      __syncthreads();   // the buffer just read is the one the next iteration refills
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
      int raw = 0, kn = 0;
      if (row < n) {
        const float g = __ldg(gold_D + row);
        const int gc = __ldg(gold_col + row);
#pragma unroll
        for (int jb = 0; jb < 2; ++jb) {
          const int64_t cb = col0 + tx * 4 + 64 * jb;   // 4 columns in one 32-bit word of the mask
          const uint32_t word = (known && cb < V) ? __ldg(known + (size_t)row * words + (cb >> 5)) : 0u;
#pragma unroll
          for (int b4 = 0; b4 < 4; ++b4) {
            const int64_t col = cb + b4;
            if (col < V && (acc[i][4 * jb + b4] <= g || col == gc)) {
              ++raw;
              kn += (int)((word >> (col & 31)) & 1u);
            }
          }
        }
      }
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) {
        raw += __shfl_xor_sync(FULL, raw, o);
        kn += __shfl_xor_sync(FULL, kn, o);
      }
      if (tx == 0 && row < n) {
        if (raw) atomicAdd(raw_cnt + row, raw);
        if (kn) atomicAdd(known_cnt + row, kn);
      }
    }
  }
}

int check_launch(const char* what) {
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), what);
}

int blocks_for_triples(int64_t N) { return (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, 132 * 8)); }

}  // namespace

int launch_rotate_forward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                          float gamma, float* energies, float* loss_out, cudaStream_t st) {
  int rc = rgcn_check_cuda(cudaMemsetAsync(loss_out, 0, 2 * sizeof(float), st), "memset(loss)");
  if (rc || N == 0) return rc;
  if (d % 8 == 0)
    k_rotate_fwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, gamma, energies, loss_out);
  else
    k_rotate_fwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, gamma, energies, loss_out);
  rc = check_launch("k_rotate_fwd");
  if (rc) return rc;
  k_rotate_finalize<<<1, 1, 0, st>>>(loss_out, 1.0f / (float)N, 1.0f / ((float)N * (float)d));
  return check_launch("k_rotate_finalize");
}

int launch_rotate_backward(const float* codes, const float* rel, int d, const int32_t* X, int64_t N, const float* Y,
                           const float* energies, float g_loss, float g_reg, const float* g_scale_dev,
                           const float* g_energy, float* dcodes, float* drel, float* rel_slice_sumsq, cudaStream_t st) {
  if (N == 0) return RGCN_OK;
  const float g_loss_over_n = g_loss / (float)N;
  const float c_reg = g_reg * 2.0f / ((float)N * (float)d);
  if (d % 8 == 0)
    k_rotate_bwd<4><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                           g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  else
    k_rotate_bwd<2><<<blocks_for_triples(N), 256, 0, st>>>(codes, rel, d, X, N, Y, energies, g_loss_over_n, c_reg,
                                                           g_scale_dev, g_energy, dcodes, drel, rel_slice_sumsq);
  return check_launch("k_rotate_bwd");
}

int launch_rotate_rank_prepare(const float* codes, const float* rel, int d, const int32_t* X, int64_t n, int side,
                               float* Q, float* gold_D, int32_t* gold_col, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  if (d % 8 == 0)
    k_rotate_rank_prepare<4><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_D, gold_col);
  else
    k_rotate_rank_prepare<2><<<blocks_for_triples(n), 256, 0, st>>>(codes, rel, d, X, n, side, Q, gold_D, gold_col);
  return check_launch("k_rotate_rank_prepare");
}

int launch_rotate_rank(const float* Q, const float* codes, int V, int d, int64_t n, const float* gold_D,
                       const int32_t* gold_col, const uint32_t* known, int32_t* raw_cnt, int32_t* known_cnt,
                       cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  const dim3 grid((V + RK_TILE - 1) / RK_TILE, (unsigned)std::min<int64_t>((n + RK_TILE - 1) / RK_TILE, 65535));
  k_rotate_rank<<<grid, 256, 0, st>>>(Q, codes, V, d, n, gold_D, gold_col, known, (V + 31) / 32, raw_cnt, known_cnt);
  return check_launch("k_rotate_rank");
}
