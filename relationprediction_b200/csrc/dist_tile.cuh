// dist_tile.cuh -- the tiled all-pairs distance kernel of the distance decoders (rotate.cu, transe.cu), sm_90a.
//
// Every query row q of Q [n, d] against every candidate row v of a table [V, d]: D = sum over the column pairs
// (k, h + k), h = d / 2, of the decoder's per-pair term, in one fixed order: ascending k in chunks of RK_KC pairs, each
// chunk summed from 0 by Step::step and its sum added to the total, every rounding pinned (no contraction choice is
// left to the compiler).  A decoder's prepare kernel sums its gold's distance this way on one thread, so the gold ties
// with itself -- and duplicated rows tie -- bit for bit; zero-padded columns add +0.  The chunked sum keeps the float32
// error of D near 440 (d = 500) several times below that of one running sum, which decides how many near-ties float32
// ranks differently from float64.
//
// A CTA owns 128 queries x 128 candidates, 256 threads as a 16 x 16 grid, each thread an 8 x 8 register tile (rows
// ty*4 + 64 i + a, columns tx*4 + 64 j + b, i, j < 2, a, b < 4).  The k range goes in chunks of RK_KC column pairs;
// each chunk of both operands is staged k-major ([re 0..KC-1 | im 0..KC-1][row]) in shared memory by 4-byte cp.async,
// double-buffered, with zero fill past n / V / h.  The epilogue (Epi) gets the finished register tile:
//   DistRankEpi: per query row, the columns < V with D <= gold_D (or the gold itself), and among them the known ones;
//                the 16 threads of a row sum by shuffles and add once per row and CTA.
//   DistTopKEpi: per query row, the tile's best k eligible columns by D ascending, the smaller column first on ties.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int RK_TILE = 128, RK_KC = 8, RK_LD = RK_TILE + 4;   // +4: spread the transposing writes over the banks
constexpr int RK_STAGE = 2 * RK_KC * RK_LD;                    // floats of one operand's chunk

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

// Rank epilogue: raw_cnt / known_cnt (zeroed by the caller) += the counts of D_v <= gold_D[row] (the gold column
// gold_col[row] always counts) and of those whose bit is set in `known` [n, words] (or nullptr)
struct DistRankEpi {
  const float* gold_D;
  const int32_t* gold_col;
  const uint32_t* known;
  int words;
  int32_t* raw_cnt;
  int32_t* known_cnt;

  __device__ __forceinline__ void operator()(const float (&acc)[8][8], int64_t row0, int64_t col0, int tx, int ty,
                                             int V, int64_t n) const {
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
        raw += __shfl_xor_sync(0xffffffffu, raw, o);
        kn += __shfl_xor_sync(0xffffffffu, kn, o);
      }
      if (tx == 0 && row < n) {
        if (raw) atomicAdd(raw_cnt + row, raw);
        if (kn) atomicAdd(known_cnt + row, kn);
      }
    }
  }
};

// Top-k epilogue: for every query row the tile's best k eligible columns -- D ascending, the smaller column first on
// ties; columns >= V and columns whose bit is set in `excl` [n, words] (or nullptr) are not eligible -- in order at
// cand[(row * gridDim.x + blockIdx.x) * k + p] as (bits of -D, column), the tail padded (bits of -inf, 0xffffffff):
// the candidate format of the scoring GEMM's top-k epilogue, so launch_topk_merge (energy descending, smaller id first)
// merges them unchanged.  k <= RK_TILE.  k rounds per row: every thread takes its best column not yet placed (strict
// < in column order), the 16 threads of the row keep the best by shuffles on (D, column), and the owner marks it.
struct DistTopKEpi {
  const uint32_t* excl;
  int words;
  int k;
  uint2* cand;

  __device__ __forceinline__ void operator()(const float (&acc)[8][8], int64_t row0, int64_t col0, int tx, int ty,
                                             int V, int64_t n) const {
    constexpr int NONE = 0x7fffffff;
    const uint2 none = make_uint2(__float_as_uint(-INFINITY), 0xffffffffu);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t row = row0 + ty * 4 + 64 * (i >> 2) + (i & 3);
      uint32_t left = 0u;   // bit j: column tx*4 + 64 (j >> 2) + (j & 3) is eligible and not yet placed
      if (row < n) {
#pragma unroll
        for (int jb = 0; jb < 2; ++jb) {
          const int64_t cb = col0 + tx * 4 + 64 * jb;
          const uint32_t word = (excl && cb < V) ? __ldg(excl + (size_t)row * words + (cb >> 5)) : 0u;
#pragma unroll
          for (int b4 = 0; b4 < 4; ++b4) {
            const int64_t col = cb + b4;
            if (col < V && !((word >> (col & 31)) & 1u)) left |= 1u << (4 * jb + b4);
          }
        }
      }
      int p = 0;
      for (; p < k; ++p) {
        float bd = INFINITY;
        int bj = -1;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (((left >> j) & 1u) && (bj < 0 || acc[i][j] < bd)) {
            bd = acc[i][j];
            bj = j;
          }
        const int mine = bj < 0 ? NONE : (int)col0 + tx * 4 + 64 * (bj >> 2) + (bj & 3);
        int bc = mine;
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
          const float od = __shfl_xor_sync(0xffffffffu, bd, o);
          const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
          if (oc != NONE && (bc == NONE || od < bd || (od == bd && oc < bc))) {
            bd = od;
            bc = oc;
          }
        }
        if (bj >= 0 && bc == mine) left &= ~(1u << bj);
        if (!__any_sync(0xffffffffu, bc != NONE)) break;   // both rows of the warp ran dry
        if (tx == 0 && row < n)
          cand[((size_t)row * gridDim.x + blockIdx.x) * k + p] =
              bc == NONE ? none : make_uint2(__float_as_uint(-bd), (uint32_t)bc);
      }
      if (tx == 0 && row < n)
        for (; p < k; ++p) cand[((size_t)row * gridDim.x + blockIdx.x) * k + p] = none;
    }
  }
};

// Step: the decoder's per-pair term, Step::step(qr, qi, vr, vi, part) = part + term(q_k, q_{h+k}, v_k, v_{h+k}).
// Epi is built in the kernel from its fields, which are passed as separate kernel parameters (EpiArgs): NVVM keeps a
// struct parameter as one aggregate and schedules its loads differently.
template <class Step, class Epi, class... EpiArgs>
__global__ void __launch_bounds__(256, 1)
    k_dist_tile(const float* __restrict__ Q, const float* __restrict__ codes, int V, int d, int64_t n,
                EpiArgs... epi_args) {
  const Epi epi{epi_args...};
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
          for (int j = 0; j < 8; ++j) part[i][j] = Step::step(qr[i], qi[i], vr[j], vi[j], part[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = __fadd_rn(acc[i][j], part[i][j]);
      __syncthreads();   // the buffer just read is the one the next iteration refills
    }
    epi(acc, row0, col0, tx, ty, V, n);
  }
}

// grid of k_dist_tile for n queries against V candidates
inline dim3 dist_tile_grid(int V, int64_t n) {
  const int64_t rows = (n + RK_TILE - 1) / RK_TILE;
  return dim3((V + RK_TILE - 1) / RK_TILE, (unsigned)(rows < 65535 ? rows : 65535));
}

}  // namespace
