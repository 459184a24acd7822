// topk.cu -- merge step of the fused top-k prediction (distmult_topk / rgcn_complex_topk, and the ensemble's
// rgcn_ensemble_topk / rgcn_ensemble_relation_topk), sm_90a.
//
// The scoring GEMM's top-k epilogue (k_gemm_tf32x3<4>) leaves, for every query row, ceil(V / 128) lists of k
// (energy, entity) candidates, one per 128-entity tile.  Every entity appears in at most one list, so a row's best
// k overall are among its candidates; this kernel picks them in order.
//
// Order: energy descending, smaller entity id first on ties.  It is kept as one 64-bit key per candidate:
// high word = the energy's bits mapped to an unsigned order (-0 counts as +0), low word = ~id; key 0 = no candidate.
// One block per row: every thread keeps the best key of its share of the candidates; each round the block maximum
// is the next answer, and only the thread that owned it rescans its share for its best key below that one.
//
// k_ensemble_topk_merge is the same design for the ensemble's candidates (k_gemm_ensemble<EnsTopKEpi>: (double u, id),
// u ascending, one list per 64-column tile), which do not fit 64 bits: its key is the pair (~bits(u), ~id), compared
// high word first.  u >= 0, so its bits order as the doubles do and ~bits(u) is never 0: (0, 0) = no candidate.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace {

constexpr int MERGE_THREADS = 128;

__device__ __forceinline__ uint64_t cand_key(uint2 c) {
  if (c.y == 0xffffffffu) return 0ull;
  uint32_t u = c.x == 0x80000000u ? 0u : c.x;                 // -0 == +0
  u ^= (u & 0x80000000u) ? 0xffffffffu : 0x80000000u;         // order-preserving map of the float bits
  return ((uint64_t)u << 32) | (uint64_t)(~c.y);
}

__device__ __forceinline__ float key_energy(uint64_t key) {
  const uint32_t u = (uint32_t)(key >> 32);
  return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}

// best key of this thread's candidates (i = tid, tid + T, ...) strictly below `below`
__device__ __forceinline__ uint64_t best_below(const uint2* __restrict__ c, int per_row, uint64_t below) {
  uint64_t b = 0ull;
  for (int i = threadIdx.x; i < per_row; i += MERGE_THREADS) {
    const uint64_t key = cand_key(__ldg(c + i));
    if (key < below && key > b) b = key;
  }
  return b;
}

__global__ void __launch_bounds__(MERGE_THREADS)
    k_topk_merge(const uint2* __restrict__ cand, int64_t n, int per_row, int k, int32_t* __restrict__ ids,
                 float* __restrict__ energies) {
  __shared__ uint64_t sh_warp[MERGE_THREADS / 32];
  __shared__ uint64_t sh_best;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t row = blockIdx.x; row < n; row += gridDim.x) {
    const uint2* c = cand + (size_t)row * per_row;
    int32_t* orow_id = ids + (size_t)row * k;
    float* orow_e = energies + (size_t)row * k;
    uint64_t mine = best_below(c, per_row, ~0ull);
    int p = 0;
    for (; p < k; ++p) {
      uint64_t b = mine;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const uint64_t x = __shfl_xor_sync(0xffffffffu, b, o);
        b = x > b ? x : b;
      }
      if (lane == 0) sh_warp[warp] = b;
      __syncthreads();
      if (threadIdx.x == 0) {
        uint64_t m = sh_warp[0];
        for (int w = 1; w < MERGE_THREADS / 32; ++w) m = sh_warp[w] > m ? sh_warp[w] : m;
        sh_best = m;
        if (m) {
          orow_id[p] = (int32_t)~(uint32_t)m;
          orow_e[p] = key_energy(m);
        }
      }
      __syncthreads();
      const uint64_t best = sh_best;
      if (!best) break;                                        // every eligible entity of the row is placed
      if (mine == best) mine = best_below(c, per_row, best);
      __syncthreads();                                         // sh_warp / sh_best are rewritten next round
    }
    for (int q = p + (int)threadIdx.x; q < k; q += MERGE_THREADS) {
      orow_id[q] = -1;
      orow_e[q] = -INFINITY;
    }
    __syncthreads();
  }
}

// ---- the ensemble's (u, id) candidates
struct UKey {
  uint64_t hi, lo;
};
__device__ __forceinline__ bool ukey_gt(UKey a, UKey b) { return a.hi > b.hi || (a.hi == b.hi && a.lo > b.lo); }
__device__ __forceinline__ bool ukey_none(UKey a) { return a.hi == 0ull && a.lo == 0ull; }
__device__ __forceinline__ UKey ens_key(const EnsCand* c) {
  const int32_t id = __ldg(&c->id);
  if (id < 0) return UKey{0ull, 0ull};
  return UKey{~(uint64_t)__double_as_longlong(__ldg(&c->u)), (uint64_t)(~(uint32_t)id)};
}
// best key of this thread's candidates strictly below `below`
__device__ __forceinline__ UKey ens_best_below(const EnsCand* __restrict__ c, int per_row, UKey below) {
  UKey b{0ull, 0ull};
  for (int i = threadIdx.x; i < per_row; i += MERGE_THREADS) {
    const UKey key = ens_key(c + i);
    if (ukey_gt(below, key) && ukey_gt(key, b)) b = key;
  }
  return b;
}

__global__ void __launch_bounds__(MERGE_THREADS)
    k_ensemble_topk_merge(const EnsCand* __restrict__ cand, int64_t n, int per_row, int k, int32_t* __restrict__ ids,
                          double* __restrict__ u, double* __restrict__ scores) {
  __shared__ UKey sh_warp[MERGE_THREADS / 32];
  __shared__ UKey sh_best;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t row = blockIdx.x; row < n; row += gridDim.x) {
    const EnsCand* c = cand + (size_t)row * per_row;
    int32_t* orow_id = ids + (size_t)row * k;
    double* orow_u = u + (size_t)row * k;
    double* orow_s = scores + (size_t)row * k;
    UKey mine = ens_best_below(c, per_row, UKey{~0ull, ~0ull});
    int p = 0;
    for (; p < k; ++p) {
      UKey b = mine;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const UKey x{__shfl_xor_sync(0xffffffffu, b.hi, o), __shfl_xor_sync(0xffffffffu, b.lo, o)};
        b = ukey_gt(x, b) ? x : b;
      }
      if (lane == 0) sh_warp[warp] = b;
      __syncthreads();
      if (threadIdx.x == 0) {
        UKey m = sh_warp[0];
        for (int w = 1; w < MERGE_THREADS / 32; ++w) m = ukey_gt(sh_warp[w], m) ? sh_warp[w] : m;
        sh_best = m;
        if (!ukey_none(m)) {
          const double mu = __longlong_as_double((long long)~m.hi);
          orow_id[p] = (int32_t)~(uint32_t)m.lo;
          orow_u[p] = mu;
          orow_s[p] = 1.0 - mu;
        }
      }
      __syncthreads();
      const UKey best = sh_best;
      if (ukey_none(best)) break;                              // every eligible candidate of the row is placed
      if (mine.hi == best.hi && mine.lo == best.lo) mine = ens_best_below(c, per_row, best);
      __syncthreads();                                         // sh_warp / sh_best are rewritten next round
    }
    for (int q = p + (int)threadIdx.x; q < k; q += MERGE_THREADS) {
      orow_id[q] = -1;
      orow_u[q] = INFINITY;
      orow_s[q] = 0.0;
    }
    __syncthreads();
  }
}

}  // namespace

int launch_topk_merge(const uint2* cand, int64_t n, int per_row, int k, int32_t* ids, float* energies,
                      cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  const int64_t blocks = n < 132 * 16 ? n : 132 * 16;
  k_topk_merge<<<(unsigned)blocks, MERGE_THREADS, 0, st>>>(cand, n, per_row, k, ids, energies);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_topk_merge");
}

int launch_ensemble_topk_merge(const EnsCand* cand, int64_t n, int per_row, int k, int32_t* ids, double* u,
                               double* scores, cudaStream_t st) {
  if (n == 0) return RGCN_OK;
  const int64_t blocks = n < 132 * 16 ? n : 132 * 16;
  k_ensemble_topk_merge<<<(unsigned)blocks, MERGE_THREADS, 0, st>>>(cand, n, per_row, k, ids, u, scores);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_ensemble_topk_merge");
}
