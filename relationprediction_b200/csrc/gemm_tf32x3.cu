// gemm_tf32x3.cu -- fp32-accurate dense GEMM on the Hopper tensor cores (wgmma), sm_90a.
//
//   C[M,N] (+)= A[M,K] * B^T      A row-major (K contiguous), B given K-major as Bt[N,K]
//
// Used for the self-loop terms of the R-GCN layer (H @ W_self, dS @ W_self^T; reference:
// gcn_basis.py:70-71 / gcn_basis_concat.py:65-66 `tf.matmul`).  The 1e-4 parity bar rules out a
// single TF32 pass (10-bit mantissa), so every fp32 operand is split a = a_hi + a_lo with both parts exact
// TF32 values (the streamed operand by truncation in the producers, the small pre-split operand with
// cvt.rna.tf32.f32) and three MMAs are issued per K-step:  a_hi*b_hi + a_hi*b_lo + a_lo*b_hi
// (the a_lo*b_lo term is below fp32 rounding).
//
// Three kernels (k_gemm_tf32x3<EPI>, k_gemm_tn_tf32x3, k_gemm_ensemble<EPI>): 384 threads = three warpgroups,
// 1 CTA/SM, 128-row tiles, 32-wide K blocks.
//   warpgroup 0     producer: global fp32 -> registers -> (hi, lo) -> st.shared in the K-major SWIZZLE_128B layout
//                   that wgmma reads (TF32 wgmma takes K-major operands only, so the TN kernel transposes here);
//                   cp.async of the pre-split Bt_hi / Bt_lo tiles (NT kernel; the ensemble kernel gets both
//                   operands pre-split and only copies); fence.proxy.async + mbarrier arrive.
//   warpgroups 1-2  consumers: rows 0-63 / 64-127 of the tile.  Per K block 4 K-steps x 3 wgmma.m64nNk8.tf32
//                   into two register accumulators (hi*hi; the two cross terms), then the stage is released
//                   (consume_tile, the one K loop of all three kernels).  The epilogue works straight from the
//                   accumulator registers.
//   NT: 128x128 tiles, 3-stage smem ring (64 KB per stage: A_hi, A_lo, B_hi, B_lo); TN: 2 such stages plus a ring of
//   raw fp32 blocks that its producer fills with cp.async and transposes from (see k_gemm_tn_tf32x3); ensemble:
//   128x64 tiles, 4 stages of 48 KB (see k_gemm_ensemble).
// The NT and ensemble kernels are persistent (min(tiles, SMs) CTAs walk the tiles; the producer runs on into the next
// tile while the consumers finish the last one); the TN kernel keeps one tile (x split-K) per CTA.
//
// The epilogues of the NT kernel are functors (StoreEpi, BiasActEpi, RankEpi, HighwayEpi, VarEpi, TopKEpi, BceEpi): a
// struct with the epilogue's data and one operator()(tile, big, small) over the accumulator fragment.  Epilogue<EPI>
// maps the integer of k_gemm_tf32x3<EPI> to its functor (EPI_STORE = 0 .. EPI_BIAS_ACT = 6).  A new epilogue is one such struct, one
// Epilogue<n> line and one launcher that ends in launch_persistent.  The two-member kernel k_gemm_ensemble<EPI> takes its
// functor (EnsRankEpi, EnsTopKEpi) directly, over both members' accumulators.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>

#include "kernels.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 32;  // BK floats = 128 bytes = one swizzle row
constexpr int STAGES = 3;
// One stage of a shared-memory ring of NST stages: the hi and lo planes of 128 A rows, then those of TBN B rows
template <int NST, int TBN>
struct StageShape {
  static constexpr int STAGE_COUNT = NST;
  static constexpr int A_PLANE = BM * BK * 4;              // bytes of A_hi (= A_lo)
  static constexpr int B_PLANE = TBN * BK * 4;             // bytes of B_hi (= B_lo)
  static constexpr int BYTES = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int FRAG = TBN / 2;                     // accumulator registers per thread and array
};
using NtStage = StageShape<STAGES, BN>;
constexpr int TILE_BYTES = NtStage::A_PLANE;   // 16 KB (A_hi, A_lo, B_hi, B_lo each)
constexpr int STAGE_BYTES = NtStage::BYTES;    // 64 KB
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;  // + alignment slack
constexpr int N_PRODUCERS = 128;            // one producer warpgroup
constexpr int N_CONSUMERS = 256;            // two consumer warpgroups, 64 tile rows each
constexpr int N_THREADS = N_PRODUCERS + N_CONSUMERS;
constexpr int N_FRAG = BN / 2;              // accumulator registers per thread: 64 x BN floats over 128 threads
static_assert(BM == BN, "the producers use one row schedule for both operands");

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor of wgmma (cute::GMMA::GmmaDescriptor layout):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B) | [62,64) layout type = 1 (SWIZZLE_128B)
// A K-step of 8 tf32 (32 bytes) inside the 128-byte swizzle row advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// d[64 rows of this warpgroup x 128] (+)= A(desc) * B(desc)^T, TF32 inputs, fp32 accumulators
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
      "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
// the same for a 64-column tile: d[64 rows of this warpgroup x 64]
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
// keeps the compiler from touching the accumulators while wgmma owns them
template <int NF>
__device__ __forceinline__ void fence_acc(float (&d)[NF]) {
#pragma unroll
  for (int i = 0; i < NF; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Producer-side split by TRUNCATION: hi = a with the 13 low mantissa bits cleared, lo = (a - hi) (exact in fp32) with
// its low bits cleared.  Three integer/FP instructions per element instead of two cvt.rna.tf32 each; both parts are
// exact TF32 values; the split error is |a - hi - lo| < 2^-20 |a| (round-to-nearest: 2^-22), still two orders below
// the 1e-4 bar of the layer and inside the 1e-5 bar of tests/test_gpu_gemm.py.  The small K-major operand is split
// with round-to-nearest (once): a = hi + lo with hi = RN_tf32(a) and lo = RN_tf32(a - hi).
__device__ __forceinline__ void split_tf32_trunc(float a, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(a) & 0xffffe000u);
  lo = __uint_as_float(__float_as_uint(a - hi) & 0xffffe000u);
}
__device__ __forceinline__ void split_tf32(float a, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(a));
  hi = __uint_as_float(h);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(a - hi));
  lo = __uint_as_float(l);
}

__device__ __forceinline__ uint32_t swz(int r, int c) {  // byte offset of 16 B chunk c of tile row r
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
}

template <int NST = STAGES>
__device__ __forceinline__ void init_barriers(uint64_t* full_bar, uint64_t* empty_bar) {
  for (int s = 0; s < NST; ++s) {
    mbar_init(&full_bar[s], N_PRODUCERS);
    mbar_init(&empty_bar[s], N_CONSUMERS);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// The K loop of one tile for one consumer warpgroup: k-blocks g0 .. g0 + num_kb - 1 of the CTA's stage sequence.
// The hi*hi products and the cross terms go to separate accumulators (the tensor core adds into its accumulator
// with truncation; same-magnitude additions per accumulator keep the result at SGEMM-level accuracy) and are summed
// in fp32 in the epilogue.  S: the StageShape of the kernel's ring.  Every output element of every kernel sees its
// K steps in this order, which is what makes the ensemble kernel reproduce the single-model ranks at w = 0 and 1.
template <class S>
__device__ __forceinline__ void consume_tile(uint32_t smem_base, uint64_t* full_bar, uint64_t* empty_bar, int g0,
                                             int num_kb, uint32_t a_rows, float (&big)[S::FRAG],
                                             float (&small)[S::FRAG]) {
  for (int kb = 0; kb < num_kb; ++kb) {
    const int g = g0 + kb;
    const int s = g % S::STAGE_COUNT;
    mbar_wait(&full_bar[s], (uint32_t)(g / S::STAGE_COUNT) & 1u);
    const uint32_t a_hi = smem_base + s * S::BYTES + a_rows, a_lo = a_hi + S::A_PLANE;
    const uint32_t b_hi = smem_base + s * S::BYTES + 2 * S::A_PLANE, b_lo = b_hi + S::B_PLANE;
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int kk = 0; kk < BK / 8; ++kk) {
      const uint64_t dah = make_desc(a_hi + kk * 32), dal = make_desc(a_lo + kk * 32);
      const uint64_t dbh = make_desc(b_hi + kk * 32), dbl = make_desc(b_lo + kk * 32);
      const uint32_t acc = (kb == 0 && kk == 0) ? 0u : 1u;  // first touch overwrites
      wgmma_tf32(small, dal, dbh, acc);
      wgmma_tf32(small, dah, dbl, 1u);
      wgmma_tf32(big, dah, dbh, acc);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    fence_acc(big);
    fence_acc(small);
    mbar_arrive(&empty_bar[s]);  // this thread's MMAs have read the stage
  }
}

// ------------------------------------------------------------------------------------------------
// The accumulator fragment of wgmma m64nN, as every epilogue sees it: register 4j + 2h + e of a consumer thread holds
// row 16 * (warp % 4) + lane / 4 + 8 h and column 8 j + 2 (lane % 4) + e of the warpgroup's 64 x N block.  TileCtx
// gives the thread's place in the output: its rows are r0 and r0 + 8, its columns c0 + 8 j + e.
// ------------------------------------------------------------------------------------------------
struct TileCtx {
  int tile;        // index in the kernel's tile order (N tiles fastest)
  int m0, n0;      // first row and column of the tile
  int r0, c0;      // this thread's row (h = 0) and its first column
  int M, N;
  int lane, warp;  // warp: 0..7 over the two consumer warpgroups
};

// Element walk of row r0 + 8 h over a fragment of NF registers: fn(reg, i, col, word) for the thread's i-th column
// (i = 2 j + e, columns increasing with i) held in register reg; col_bit(word, col) is bit `col` of row r0 + 8 h of
// the bitmap `bits` ([M, words], one 32-bit word loaded per 32 columns; 0 when bits is null).  Rows >= M and columns
// >= N are visited too (with word 0): the caller decides what they mean.  The callers take the bit where they use it:
// handing it over as a value costs the top-k epilogue 250 instructions per tile.
__device__ __forceinline__ uint32_t col_bit(uint32_t word, int col) { return (word >> (col & 31)) & 1u; }
template <int NF, class Fn>
__device__ __forceinline__ void for_each_col(const TileCtx& t, int h, const uint32_t* bits, int words, Fn fn) {
  const int row = t.r0 + 8 * h;
#pragma unroll
  for (int cb = 0; cb < NF / 16; ++cb) {
    const int chunk = t.n0 + 32 * cb;
    const uint32_t w =
        (bits && row < t.M && chunk < t.N) ? __ldg(bits + (size_t)row * words + (chunk >> 5)) : 0u;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = 4 * cb + jj, col = t.c0 + 8 * j + e;
        fn(4 * j + 2 * h + e, 2 * j + e, col, w);
      }
    }
  }
}
// Pair walk of row r0 + 8 h for the float2 epilogues: fn(reg, col) for every pair of columns (col, col + 1) < N held
// in registers (reg, reg + 1); col is even.  N % 2 == 0, so both columns of a pair exist or neither does.
template <class Fn>
__device__ __forceinline__ void for_each_pair(const TileCtx& t, int h, Fn fn) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = t.c0 + 8 * j;
    if (col < t.N) fn(4 * j + 2 * h, col);
  }
}
// The rank counts of one row: the four lanes of a quad hold the row's columns; their counts are summed by two
// shuffles and added to the row's totals (integer atomics: the totals do not depend on the order of the tiles).
__device__ __forceinline__ void rank_counts_flush(int raw, int kn, int row, int M, int32_t* raw_cnt,
                                                  int32_t* known_cnt, int lane) {
  raw += __shfl_xor_sync(0xffffffffu, raw, 1);
  raw += __shfl_xor_sync(0xffffffffu, raw, 2);
  kn += __shfl_xor_sync(0xffffffffu, kn, 1);
  kn += __shfl_xor_sync(0xffffffffu, kn, 2);
  if ((lane & 3) == 0 && row < M) {
    if (raw) atomicAdd(raw_cnt + row, raw);
    if (kn) atomicAdd(known_cnt + row, kn);
  }
}
// part[tile * 8 + warp] = the sum of x over the warp, by a shuffle tree in a fixed order: a sum reduced from the
// parts is bitwise repeatable
__device__ __forceinline__ void warp_part_store(float x, float* part, const TileCtx& t) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if (t.lane == 0) part[(size_t)t.tile * 8 + t.warp] = x;
}
__device__ __forceinline__ float sigmoid_ref(float x) { return 1.0f / (1.0f + expf(-x)); }

// EPI = 0: STORE epilogue: C[M, N] = or += the tile.
struct StoreEpi {
  float* C;                    // [M, ldc]
  int64_t ldc;
  int accumulate;              // C += instead of C =

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      if (row >= t.M) continue;
      float* crow = C + (size_t)row * ldc;
      for_each_pair(t, h, [&](int r, int col) {
        float2 o = make_float2(big[r] + small[r], big[r + 1] + small[r + 1]);
        if (accumulate) {
          const float2 old = *reinterpret_cast<const float2*>(crow + col);
          o.x += old.x;
          o.y += old.y;
        }
        *reinterpret_cast<float2*>(crow + col) = o;
      });
    }
  }
};

// EPI = 6: BIAS + ACTIVATION epilogue (the CompGCN layer, compgcn.cu): C[M, N] = act(tile + bias[col]), act = ReLU
// when `relu` is set, the identity otherwise.
struct BiasActEpi {
  float* C;                    // [M, ldc]
  int64_t ldc;
  const float* bias;           // [N]
  int relu;

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      if (row >= t.M) continue;
      float* crow = C + (size_t)row * ldc;
      for_each_pair(t, h, [&](int r, int col) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
        float2 o = make_float2(big[r] + small[r] + bb.x, big[r + 1] + small[r + 1] + bb.y);
        if (relu) {
          o.x = fmaxf(o.x, 0.f);
          o.y = fmaxf(o.y, 0.f);
        }
        *reinterpret_cast<float2*>(crow + col) = o;
      });
    }
  }
};

// EPI = 1: RANKING epilogue (all-entity scoring of the DistMult decoder, decoders/bilinear_diag.py:51-61, fused with
// the rank counts of common/evaluation.py:148-159): the C tile is never written.  Row m of A is a query (e1*r or r*e2),
// row n of Bt an entity code; each energy goes through the reference's float32 sigmoid and is compared with the gold
// entity's score; entities scoring >= gold add to the raw rank, and those among them whose bit is set in `known`
// to the filtered correction.
struct RankEpi {
  const float* gold_sig;       // [M] sigmoid(energy of the gold entity)
  const int32_t* gold_col;     // [M] gold entity id (always counted: score >= itself)
  const uint32_t* known;       // [M, words] bit v = entity v is a known true answer (or nullptr)
  int words;                   // ceil(N / 32)
  int32_t* raw_cnt;            // [M] += #{v : score_v >= gold}
  int32_t* known_cnt;          // [M] += #{known v : score_v >= gold}

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      int raw = 0, kn = 0;
      if (row < t.M) {
        const float gold_s = __ldg(gold_sig + row);
        const int gold_c = __ldg(gold_col + row);
        for_each_col<N_FRAG>(t, h, known, words, [&](int r, int, int col, uint32_t word) {
          // the gold entity always scores >= itself
          if (col < t.N && (sigmoid_ref(big[r] + small[r]) >= gold_s || col == gold_c)) {
            ++raw;
            kn += (int)col_bit(word, col);
          }
        });
      }
      rank_counts_flush(raw, kn, row, t.M, raw_cnt, known_cnt, t.lane);
    }
  }
};

// EPI = 2: HIGHWAY epilogue (the gate of extras/highway_layer.py:19-38): A = c2 [M, K = N] is the layer input, Bt the
// gate weight W^T, and each accumulator pair becomes  z = acc + bias[col],  g = sigmoid(z),
// out = c2 + g (c1 - c2)  (= g c1 + (1 - g) c2), written to `out` together with g (kept for the backward pass).  z
// itself is never stored.  c1, c2, out and gate share the leading dimension ld.
struct HighwayEpi {
  const float* bias;           // [N]
  const float* c1;             // [M, ld] the wrapped layer's output
  const float* c2;             // [M, ld] the layer input (the GEMM's A)
  float* out;                  // [M, ld]
  float* gate;                 // [M, ld] g
  int64_t ld;

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      if (row >= t.M) continue;
      const float* c2row = c2 + (size_t)row * ld;
      const float* c1row = c1 + (size_t)row * ld;
      float* orow = out + (size_t)row * ld;
      float* grow = gate + (size_t)row * ld;
      asm volatile("" : "+l"(c2row), "+l"(c1row));   // no hoisting of the 16 pairs' loads ahead of use (spills)
      for_each_pair(t, h, [&](int r, int col) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
        const float2 x1 = __ldg(reinterpret_cast<const float2*>(c1row + col));
        const float2 x2 = __ldg(reinterpret_cast<const float2*>(c2row + col));
        const float g0 = sigmoid_ref(big[r] + small[r] + bb.x);
        const float g1 = sigmoid_ref(big[r + 1] + small[r + 1] + bb.y);
        *reinterpret_cast<float2*>(orow + col) = make_float2(x2.x + g0 * (x1.x - x2.x), x2.y + g1 * (x1.y - x2.y));
        *reinterpret_cast<float2*>(grow + col) = make_float2(g0, g1);
      });
    }
  }
};

// EPI = 3: VARIATIONAL epilogue (extras/variational_encoding.py:14-31): A = H [M, K], Bt the pre-split W_int^T whose
// rows interleave the columns of W_mu and W_sigma (row 2j = W_mu[:, j], row 2j + 1 = W_sigma[:, j]), so each
// accumulator pair (col, col + 1) = (2j, 2j + 1) is the (mu, log sigma) of element (row, j):
//   mu = acc + b_mu[j],  l = acc' + b_sigma[j],  P[row, 2j .. 2j+1] = (mu, l)  (kept for the backward pass),
//   z[row, j] = mu + exp(l) eps[row, j],
// and every consumer warp writes kl_part[tile * 8 + warp] = sum of (1 + 2 l - mu^2 - exp(2 l)) over its elements,
// summed in a fixed order (per thread, then a shuffle tree), so the KL reduced from the parts is bitwise repeatable.
struct VarEpi {
  const float* b_mu;           // [w]
  const float* b_sigma;        // [w]
  const float* eps;            // [M, w]
  float* P;                    // [M, ldp] (mu, log sigma) interleaved, N = 2 w columns
  int64_t ldp;
  float* z;                    // [M, w]
  float* kl_part;              // [tiles * 8]
  int w;

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
    float kl = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      if (row >= t.M) continue;
      float* prow = P + (size_t)row * ldp;
      const float* erow = eps + (size_t)row * w;
      float* zrow = z + (size_t)row * w;
      asm volatile("" : "+l"(erow), "+l"(zrow));   // no hoisting of the 16 pairs' loads ahead of use (spills)
      for_each_pair(t, h, [&](int r, int col) {   // the pair is (mu, log sigma) of element col / 2
        const int e = col >> 1;
        const float mu = big[r] + small[r] + __ldg(b_mu + e);
        const float ls = big[r + 1] + small[r + 1] + __ldg(b_sigma + e);
        *reinterpret_cast<float2*>(prow + col) = make_float2(mu, ls);
        zrow[e] = mu + expf(ls) * __ldg(erow + e);
        kl += 1.f + 2.f * ls - mu * mu - expf(2.f * ls);
      });
    }
    warp_part_store(kl, kl_part, t);
  }
};

// EPI = 4: TOP-K epilogue (filtered top-k prediction over all entities, decoders/bilinear_diag.py:51-61 and
// complex.py:77-106 without the [M, N] score matrix): row m of A is a query, row n of Bt an entity code.  For each
// row the tile's best k eligible (energy, column) pairs -- energy descending, smaller column first on ties; columns
// >= N and columns whose bit is set in `excl` are not eligible -- are written in that order to
// cand[(row * tn + tile column) * k + p]; the tail past the eligible columns is (-inf, -1).  k <= BN.
struct TopKEpi {
  const uint32_t* excl;        // [M, words] bit v = entity v never appears in row m (or nullptr)
  int words;                   // ceil(N / 32)
  int k;                       // candidates per row and tile, 1 <= k <= BN
  int tn;                      // N tiles
  uint2* cand;                 // [M, tn, k] (energy bits, column)

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
    // The quad of lanes lane & ~3 holds rows r0 and r0 + 8 of the tile: 32 columns each per lane, value i
    // (= 2 j + e) at column c0 + 8 j + e, so a lane's columns increase with i.  k rounds per row: every lane
    // takes its best value not yet taken (strict > in i order: the smaller column wins a tie), the quad keeps
    // the best of the four by two shuffles on (energy, column), and the lane that owned it marks it taken.
    const int r0 = t.r0, c0 = t.c0, M = t.M;
    float v[2][32];
    uint32_t left[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      left[h] = 0u;
      for_each_col<N_FRAG>(t, h, excl, words, [&](int r, int i, int col, uint32_t word) {
        v[h][i] = big[r] + small[r];
        if (r0 + 8 * h < M && col < t.N && !col_bit(word, col)) left[h] |= 1u << i;
      });
    }
    // candidate p of row r0 + 8 h (formed at the store: a live pointer pair would spill)
    auto slot = [&](int h, int p) { return cand + ((size_t)(r0 + 8 * h) * tn + (size_t)(t.n0 / BN)) * k + p; };
    const bool writer = (t.lane & 3) == 0;
    const uint2 none = make_uint2(__float_as_uint(-INFINITY), 0xffffffffu);
    int p = 0;
    for (; p < k; ++p) {
      float be[2];
      int bc[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int bi = -1;
        be[h] = -INFINITY;
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (((left[h] >> i) & 1u) && (bi < 0 || v[h][i] > be[h])) {
            be[h] = v[h][i];
            bi = i;
          }
        const int mine = bi < 0 ? 0x7fffffff : c0 + 8 * (bi >> 1) + (bi & 1);
        bc[h] = mine;
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float oe = __shfl_xor_sync(0xffffffffu, be[h], o);
          const int oc = __shfl_xor_sync(0xffffffffu, bc[h], o);
          if (oc != 0x7fffffff && (bc[h] == 0x7fffffff || oe > be[h] || (oe == be[h] && oc < bc[h]))) {
            be[h] = oe;
            bc[h] = oc;
          }
        }
        if (bi >= 0 && bc[h] == mine) left[h] &= ~(1u << bi);
      }
      if (!__any_sync(0xffffffffu, bc[0] != 0x7fffffff || bc[1] != 0x7fffffff)) break;   // the warp's rows ran dry
      if (writer) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (r0 + 8 * h < M)
            *slot(h, p) = bc[h] == 0x7fffffff ? none : make_uint2(__float_as_uint(be[h]), (uint32_t)bc[h]);
      }
    }
    if (writer) {
      for (; p < k; ++p) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (r0 + 8 * h < M) *slot(h, p) = none;
      }
    }
  }
};

// EPI = 5: 1-N BCE epilogue (1-N training of DistMult / ComplEx): row m of A is a query, row n of Bt an entity code,
// z the energy.  With y' = pos if bit n of labels row m is set, else neg (the smoothed targets),
//   loss term  max(z, 0) - z y' + log1p(exp(-|z|)),   g = (sigmoid(z) - y') * scale * g_scale[0]
// and g is written TRANSPOSED, Gt[n * ldgt + m] (a warp's store covers 4 columns x 8 consecutive rows: whole 32 B
// sectors when ldgt % 8 == 0, as the caller pads it), so that the backward GEMMs read Gt with the contraction index
// contiguous.  Columns >= N and rows >= M are never written.  Every consumer warp writes loss_part[tile * 8 + warp] =
// the sum of its loss terms (per thread in a fixed order, then a shuffle tree), so the loss reduced from the parts is
// bitwise repeatable.
struct BceEpi {
  const uint32_t* labels;      // [M, words] bit n = entity n completes query m in the training split
  int words;                   // ceil(N / 32)
  float pos, neg;              // y' of a set and of a clear bit
  float scale;                 // 1 / (n V) of the whole query set
  const float* g_scale;        // [1] upstream gradient of the loss (device) or nullptr (1)
  float* Gt;                   // [N, ldgt] or nullptr: loss only
  int64_t ldgt;
  float* loss_part;            // [tiles * 8]

  __device__ __forceinline__ void operator()(const TileCtx& t, const float (&big)[N_FRAG],
                                             const float (&small)[N_FRAG]) const {
    const float gs = scale * (g_scale ? __ldg(g_scale) : 1.f);
    float ls = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      if (row >= t.M) continue;
      for_each_col<N_FRAG>(t, h, labels, words, [&](int r, int, int col, uint32_t word) {
        if (col < t.N) {
          const float z = big[r] + small[r];
          const float y = col_bit(word, col) ? pos : neg;
          ls += fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
          if (Gt) Gt[(size_t)col * ldgt + row] = (1.0f / (1.0f + expf(-z)) - y) * gs;
        }
      });
    }
    warp_part_store(ls, loss_part, t);
  }
};

// k_gemm_tf32x3<EPI> runs the epilogue Epilogue<EPI>::type.  There is no primary definition: an integer without a
// line here does not compile.
enum : int { EPI_STORE = 0, EPI_RANK = 1, EPI_HIGHWAY = 2, EPI_VAR = 3, EPI_TOPK = 4, EPI_BCE = 5, EPI_BIAS_ACT = 6 };
template <int EPI>
struct Epilogue;
template <> struct Epilogue<EPI_STORE> { using type = StoreEpi; };
template <> struct Epilogue<EPI_BIAS_ACT> { using type = BiasActEpi; };
template <> struct Epilogue<EPI_RANK> { using type = RankEpi; };
template <> struct Epilogue<EPI_HIGHWAY> { using type = HighwayEpi; };
template <> struct Epilogue<EPI_VAR> { using type = VarEpi; };
template <> struct Epilogue<EPI_TOPK> { using type = TopKEpi; };
template <> struct Epilogue<EPI_BCE> { using type = BceEpi; };

// PERSISTENT: a CTA walks the tiles blockIdx.x, blockIdx.x + gridDim.x, ... (N tiles fastest, see below); the
// shared-memory stages and their barrier phases run on across tile boundaries, so the producer fills the pipeline of
// tile t+1 (global-load latency included) while the consumers run the epilogue of tile t.
template <int EPI>
__global__ void __launch_bounds__(N_THREADS, 1)
    k_gemm_tf32x3(const float* __restrict__ A, int64_t lda, const float* __restrict__ Bhi,
                  const float* __restrict__ Blo, int64_t ldb, int M, int N, int K, int n_tiles,
                  const typename Epilogue<EPI>::type epi) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B: 1024 B aligned
  const int tid = threadIdx.x, lane = tid & 31;
  // Tile order, N tiles fastest: the CTAs that share an A tile (all N tiles of one M tile) run at the same time,
  // so the big operand is read from HBM once and from L2 afterwards; the small K-major operand (<= a few MB of
  // hi/lo planes) lives in L2 throughout.
  const int tn = (N + BN - 1) / BN;
  const int num_kb = (K + BK - 1) / BK;
  const int n_mine = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // tiles of this CTA (>= 1)
  const int total_g = n_mine * num_kb;                                                   // its k-blocks, all tiles

  if (tid == 0) init_barriers(full_bar, empty_bar);
  __syncthreads();

  if (tid < N_PRODUCERS) {
    // ================= producer warpgroup =================
    // Software-pipelined over the CTA's whole k-block sequence g = 0 .. total_g-1 (tile g / num_kb, block g % num_kb):
    // while block g is converted and stored, the global loads of A(g+1), A(g+2) are already in flight in registers
    // and the async copies of B(g+1) in the next smem stage -- also when g+1 belongs to the NEXT tile.
    const int c = tid & 7;        // 16 B chunk within the 128 B K-row
    const int rbase = tid >> 3;   // 0..15; this thread handles tile rows rbase + 16 i
    const uint32_t soff = swz(rbase, c);  // swizzled offset of (row rbase, chunk c); row rbase + 16 i is 2048 i further
    constexpr int NR = BM / 16;

    // ---- B request stream (async copies, one block ahead)
    int b_kb = 0, b_tile = (int)blockIdx.x, b_stage = 0;
    size_t b_off = 0;
    uint32_t b_ok = 0;            // bit i: tile row rbase + 16 i exists
    auto b_set_tile = [&]() {
      const int r0 = (b_tile % tn) * BN + rbase;
      b_ok = 0;
#pragma unroll
      for (int i = 0; i < NR; ++i) b_ok |= (r0 + 16 * i < N ? 1u : 0u) << i;
      b_off = (b_ok & 1u) ? (size_t)r0 * ldb + c * 4 : 0;
    };
    b_set_tile();
    auto issue_b = [&]() {        // requests the stream's current block, then advances it
      const uint32_t b_hi = smem_base + b_stage * STAGE_BYTES + 2 * TILE_BYTES + soff, b_lo = b_hi + TILE_BYTES;
      const bool col_ok = b_kb * BK + c * 4 < K;  // K % 4 == 0: a 16 B chunk is entirely valid or entirely padding
      const size_t kof = b_off + (size_t)b_kb * BK;
#pragma unroll
      for (int i = 0; i < NR; ++i) {
        const bool ok = col_ok && ((b_ok >> i) & 1u);
        const size_t o = kof + (size_t)(16 * i) * ldb;
        cp_async16(b_hi + 2048 * i, ok ? Bhi + o : Bhi, ok ? 16u : 0u);
        cp_async16(b_lo + 2048 * i, ok ? Blo + o : Blo, ok ? 16u : 0u);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      b_stage = b_stage + 1 == STAGES ? 0 : b_stage + 1;
      if (++b_kb == num_kb) {
        b_kb = 0;
        b_tile += (int)gridDim.x;
        b_set_tile();
      }
    };
    // ---- A request stream (register prefetch, PF blocks ahead)
    int a_kb = 0, a_tile = (int)blockIdx.x;
    size_t a_off = 0;
    uint32_t a_ok = 0;
    auto a_set_tile = [&]() {
      const int r0 = (a_tile / tn) * BM + rbase;
      a_ok = 0;
#pragma unroll
      for (int i = 0; i < NR; ++i) a_ok |= (r0 + 16 * i < M ? 1u : 0u) << i;
      a_off = (a_ok & 1u) ? (size_t)r0 * lda + c * 4 : 0;
    };
    a_set_tile();
    auto load_a = [&](float4 (&v)[NR]) {   // requests the stream's current block, then advances it
      const bool col_ok = a_kb * BK + c * 4 < K;
      const float* p = A + a_off + (size_t)a_kb * BK;
#pragma unroll
      for (int i = 0; i < NR; ++i)
        v[i] = (col_ok && ((a_ok >> i) & 1u)) ? __ldg(reinterpret_cast<const float4*>(p + (size_t)(16 * i) * lda))
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
      if (++a_kb == num_kb) {
        a_kb = 0;
        a_tile += (int)gridDim.x;
        a_set_tile();
      }
    };
    // PF k-blocks of A are in flight in registers (and of B as asynchronous copies) while block g is converted and
    // stored.  The asynchronous copies of B stay ONE block ahead: they need the shared-memory stage of block g + 1,
    // and asking for the stage of g + 2 would make the producer wait for the MMAs of block g - 1 before storing
    // block g.  The A rows only need registers, so they run two blocks ahead.
    constexpr int PF = 2;                    // register prefetch distance of A in k-blocks (PF + 1 buffers)
    float4 vbuf[PF + 1][NR];
    mbar_wait(&empty_bar[0], 1u);            // first use of a stage: the "previous phase" is complete
    issue_b();
    for (int p = 0; p < PF; ++p)
      if (p < total_g) load_a(vbuf[p]);
    int s = 0;                               // stage of block g
    uint32_t ph_next = 0;                    // phase bit of block g + 1's stage use
    for (int g0 = 0; g0 < total_g; g0 += PF + 1) {
#pragma unroll
      for (int u = 0; u <= PF; ++u) {
        const int g = g0 + u;
        if (g >= total_g) break;
        const bool more = g + 1 < total_g;
        const int s1 = s + 1 == STAGES ? 0 : s + 1;
        if (s1 == 0) ph_next ^= 1u;          // block g + 1 starts a new round of the stage ring
        if (more) {
          mbar_wait(&empty_bar[s1], ph_next ^ 1u);
          issue_b();
        }
        if (g + PF < total_g) load_a(vbuf[(u + PF) % (PF + 1)]);
        const uint32_t a_hi = smem_base + s * STAGE_BYTES + soff, a_lo = a_hi + TILE_BYTES;
#pragma unroll
        for (int i = 0; i < NR; ++i) {
          float4 hi, lo;
          split_tf32_trunc(vbuf[u][i].x, hi.x, lo.x);
          split_tf32_trunc(vbuf[u][i].y, hi.y, lo.y);
          split_tf32_trunc(vbuf[u][i].z, hi.z, lo.z);
          split_tf32_trunc(vbuf[u][i].w, hi.w, lo.w);
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a_hi + 2048 * i), "f"(hi.x), "f"(hi.y),
                       "f"(hi.z), "f"(hi.w)
                       : "memory");
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a_lo + 2048 * i), "f"(lo.x), "f"(lo.y),
                       "f"(lo.z), "f"(lo.w)
                       : "memory");
        }
        if (more)
          asm volatile("cp.async.wait_group 1;" ::: "memory");  // B(g) has landed, B(g+1) may still fly
        else
          asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> tensor core
        mbar_arrive(&full_bar[s]);
        s = s1;
      }
    }
  } else {
    // ================= consumer warpgroups =================
    const int ctid = tid - N_PRODUCERS;
    const int wg = ctid >> 7, warp = ctid >> 5;
    const uint32_t a_rows = (uint32_t)(wg * 64 * 128);   // the warpgroup's 64 A rows of 128 B
    float big[N_FRAG], small[N_FRAG];
    for (int ti = 0; ti < n_mine; ++ti) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int m0 = (tile / tn) * BM, n0 = (tile % tn) * BN;
      consume_tile<NtStage>(smem_base, full_bar, empty_bar, ti * num_kb, num_kb, a_rows, big, small);
      const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = n0 + 2 * (lane & 3);
      const TileCtx t{tile, m0, n0, r0, c0, M, N, lane, warp};
      epi(t, big, small);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// C[M,N] += A^T B with A [K,M] and B [K,N] row-major: the V-long reductions of the backward pass
// (dW_self = H^T dS, basis dV = Agg^T G).  Both operands are MN-major in memory (the contraction index is the
// slow one); TF32 wgmma reads K-major shared memory only, so the producer transposes while it splits.
//
// Producer, two passes per k-block:
//   copy       cp.async.cg of the raw fp32 [32 k x 128] slabs of A and B into a ring of TN_RAW staging blocks,
//              TN_RAW - 1 k-blocks ahead of the conversion.  The loads in flight live in shared memory, not in
//              registers.  A warp fetches one 512 B k-row per instruction.  Chunk q (16 B) of k-row k is stored at
//              chunk q ^ ((k / 4) % 8) of its row, so that the conversion reads without bank conflicts.
//   transpose  a thread reads 4 k-rows x 4 consecutive M (N) values (4 ld.shared.v4), transposes the 4 x 4 in
//              registers, splits, and writes 4 + 4 st.shared.v4: the (hi, lo) chunks of 4 K-major rows in the
//              SWIZZLE_128B layout.  The 8 lanes of a quarter-warp take the 8 k-groups of one 4-row group, so both
//              their reads (staging chunks h ^ g) and their writes (swizzled chunks g ^ (r % 8)) cover all 32 banks.
// Two MMA stages (128 KB) and three staging blocks (96 KB) fill the 227 KB of shared memory of a block.
//
// Split-K: CTA b computes tile b % tiles over k-block range b / tiles (see launch_gemm_tn_tf32x3 for the split
// count); partial tiles are added into C with red.global.add.v2.  The CTAs of one k range are consecutive in the
// grid and run at the same time, so each row of A and B comes from HBM once and is re-read from L2.
//
// Accuracy: the tensor core adds into its accumulator with truncation, so the error of one accumulation chain grows
// with its length (K = 50 000, M = N = 512, normal inputs: 7e-6 relative for 92 k-blocks per chain, 1.6e-5 for
// 196; K = 5 M with 17 splits: 5.8e-4).  A CTA therefore adds its partial tile into C (round-to-nearest) every
// TN_FLUSH_KB k-blocks and restarts the accumulators, which bounds the chain whatever the split length: 3e-6 at
// K = 50 000 and at K = 5 M.  On an H100 SXM the flushes cost about 1 ms of 29 at K = 5 M, M = N = 512.
// ------------------------------------------------------------------------------------------------
constexpr int TN_FLUSH_KB = 32;                         // k-blocks per accumulation chain
constexpr int TN_STAGES = 2;                            // MMA stages (A_hi, A_lo, B_hi, B_lo)
using TnStage = StageShape<TN_STAGES, BN>;
constexpr int TN_RAW = 3;                               // fp32 staging blocks
constexpr int RAW_TILE_BYTES = BK * BM * 4;             // 16 KB: 32 k-rows x 128 values of one operand
constexpr int RAW_BYTES = 2 * RAW_TILE_BYTES;           // A and B
constexpr int TN_SMEM_BYTES = TN_STAGES * STAGE_BYTES + TN_RAW * RAW_BYTES + 1024;
static_assert(TN_SMEM_BYTES <= 227 * 1024, "TN kernel exceeds the shared memory of a block");
static_assert(N_PRODUCERS == 128 && BK == 32 && BM == 128, "the TN producer's lane mapping assumes these");

__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, float x, float y, float z, float w) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}

__global__ void __launch_bounds__(N_THREADS, 1)
    k_gemm_tn_tf32x3(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb,
                     float* __restrict__ C, int64_t ldc, int M, int N, int K, int kb_per_split) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[TN_STAGES], empty_bar[TN_STAGES];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tm = (M + BM - 1) / BM, tiles = tm * ((N + BN - 1) / BN);
  const int tile = (int)blockIdx.x % tiles, split = (int)blockIdx.x / tiles;
  const int m0 = (tile % tm) * BM, n0 = (tile / tm) * BN;
  const int kb_begin = split * kb_per_split;
  const int num_kb = min(kb_per_split, (K + BK - 1) / BK - kb_begin);   // >= 1: the launch makes no empty split

  if (tid == 0) init_barriers<TN_STAGES>(full_bar, empty_bar);
  __syncthreads();

  if (tid < N_PRODUCERS) {
    const uint32_t raw_base = smem_base + TN_STAGES * STAGE_BYTES;
    // copy pass: this thread fetches chunk `lane` of k-rows warp + 4 i (i < 8) of both operands
    const bool a_ok = m0 + 4 * lane < M, b_ok = n0 + 4 * lane < N;   // M, N % 4 == 0: a chunk is all in or all out
    const float* pa = A + (a_ok ? m0 + 4 * lane : 0);
    const float* pb = B + (b_ok ? n0 + 4 * lane : 0);
    auto issue = [&](int kbi) {
      const uint32_t dst = raw_base + (kbi % TN_RAW) * RAW_BYTES;
      const int k0 = (kb_begin + kbi) * BK + warp;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bool kok = k0 + 4 * i < K;
        const size_t row = kok ? (size_t)(k0 + 4 * i) : 0;
        const uint32_t off = (uint32_t)((warp + 4 * i) * 512 + ((lane ^ i) << 4));   // (k / 4) % 8 == i
        cp_async16(dst + off, pa + row * lda, kok && a_ok ? 16u : 0u);
        cp_async16(dst + RAW_TILE_BYTES + off, pb + row * ldb, kok && b_ok ? 16u : 0u);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    };
    // transpose pass: this thread converts k-group g (k-rows 4g .. 4g+3) of the 4-row groups h and h + 16
    const int g = lane & 7;
    auto convert = [&](uint32_t raw, uint32_t hi_plane) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int h = (lane >> 3) + 4 * warp + 16 * u;
        float4 v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = ld_shared_v4(raw + (4 * g + j) * 512 + ((h ^ g) << 4));
        const float x[4][4] = {{v[0].x, v[1].x, v[2].x, v[3].x}, {v[0].y, v[1].y, v[2].y, v[3].y},
                               {v[0].z, v[1].z, v[2].z, v[3].z}, {v[0].w, v[1].w, v[2].w, v[3].w}};
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // K-major tile row 4 h + i, chunk g: k = 4g .. 4g+3
          float hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) split_tf32_trunc(x[i][j], hi[j], lo[j]);
          const uint32_t a = hi_plane + swz(4 * h + i, g);
          st_shared_v4(a, hi[0], hi[1], hi[2], hi[3]);
          st_shared_v4(a + TILE_BYTES, lo[0], lo[1], lo[2], lo[3]);
        }
      }
    };
    issue(0);
    if (num_kb > 1)
      issue(1);
    else
      asm volatile("cp.async.commit_group;" ::: "memory");   // one group per k-block, empty ones included
    for (int kb = 0; kb < num_kb; ++kb) {
      asm volatile("cp.async.wait_group 1;" ::: "memory");     // this thread's copies of block kb have landed
      // everyone's copies of block kb are visible, and nobody reads block kb - 1's staging block any more
      asm volatile("bar.sync 1, %0;" ::"n"(N_PRODUCERS) : "memory");
      if (kb + 2 < num_kb)
        issue(kb + 2);
      else
        asm volatile("cp.async.commit_group;" ::: "memory");
      const int s = kb % TN_STAGES;
      mbar_wait(&empty_bar[s], ((uint32_t)(kb / TN_STAGES) & 1u) ^ 1u);
      const uint32_t raw = raw_base + (kb % TN_RAW) * RAW_BYTES, stage = smem_base + s * STAGE_BYTES;
      convert(raw, stage);                                          // A -> A_hi, A_lo
      convert(raw + RAW_TILE_BYTES, stage + 2 * TILE_BYTES);        // B -> B_hi, B_lo
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> tensor core
      mbar_arrive(&full_bar[s]);
    }
  } else {
    // consumers: the same K loop as the NT kernel, in chunks of at most TN_FLUSH_KB k-blocks; after each chunk the
    // partial tile is added into C and the accumulators start again from zero
    const int ctid = tid - N_PRODUCERS;
    const int wg = ctid >> 7;
    const int r0 = m0 + wg * 64 + ((ctid >> 5) & 3) * 16 + (lane >> 2);
    const int c0 = n0 + 2 * (lane & 3);
    float* const cbase = C + (size_t)r0 * ldc + c0;
    float big[N_FRAG], small[N_FRAG];
    for (int kc = 0; kc < num_kb; kc += TN_FLUSH_KB) {
      consume_tile<TnStage>(smem_base, full_bar, empty_bar, kc, min(TN_FLUSH_KB, num_kb - kc),
                            (uint32_t)(wg * 64 * 128), big, small);
      float* cp = cbase;
      asm volatile("" : "+l"(cp));   // keeps the 32 addresses below from being hoisted out of the loop (spills)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (r0 + 8 * h >= M) continue;
        float* crow = cp + (size_t)(8 * h) * ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (c0 + 8 * j < N)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(crow + 8 * j),
                         "f"(big[4 * j + 2 * h] + small[4 * j + 2 * h]),
                         "f"(big[4 * j + 2 * h + 1] + small[4 * j + 2 * h + 1])
                         : "memory");
        }
      }
    }
  }
}

// Bt_hi/Bt_lo[n][k] from B: transposed = 0: B is [N,K] row-major already (K-major);
//                                  transposed = 1: B is [K,N] row-major -> transpose while splitting
__global__ void k_split_b(const float* __restrict__ B, int64_t ldb, int N, int K, int transposed,
                          float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t total = (int64_t)N * K;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / K), k = (int)(i % K);
    const float v = transposed ? __ldg(B + (size_t)k * ldb + n) : __ldg(B + (size_t)n * ldb + k);
    float h, l;
    split_tf32(v, h, l);
    hi[i] = h;
    lo[i] = l;
  }
}

// The pre-split of the interleaved variational weight W_int [K = d, 2w] (column 2j = W_mu[:, j], column 2j + 1 =
// W_sigma[:, j]; W_mu, W_sigma [d, w] row-major), made from the two tables directly (no interleaved copy):
//   transposed = 1:  Bt = W_int^T [N = 2w, K = d]     (forward, P = H W_int)
//   transposed = 0:  Bt = W_int   [N = d, K = 2w]     (backward, dH = dP W_int^T)
__global__ void k_split_b_interleave(const float* __restrict__ Wmu, const float* __restrict__ Wsig, int d, int w,
                                     int transposed, float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t total = (int64_t)2 * d * w;
  const int K = transposed ? d : 2 * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / K), k = (int)(i % K);
    const int row = transposed ? k : n, c = transposed ? n : k;   // W_int[row, c]
    const float v = __ldg(((c & 1) ? Wsig : Wmu) + (size_t)row * w + (c >> 1));
    float h, l;
    split_tf32(v, h, l);
    hi[i] = h;
    lo[i] = l;
  }
}

// ------------------------------------------------------------------------------------------------
// ENSEMBLE SCORING (R-GCN+: the weighted sum of two models' scores, tools/ensemble.py `weighted_sum`): every tile
// runs the K blocks of member A (Q_A [M, K_A] against codes_A [N, K_A]) and then those of member B into separate
// accumulators, and the epilogue k_gemm_ensemble<EPI> was instantiated with combines them.  [M, N] is never written.
//   EnsRankEpi: each member's float32 sigmoid score as RankEpi forms it, combined in float64,
//     c = w s_A + (1 - w) s_B   (separately rounded multiplies and add: the reference tool's Python arithmetic),
//     and c >= G counted into raw_cnt / known_cnt by RankEpi's rules, G = w g_A + (1 - w) g_B.
//   EnsTopKEpi: each row's best k of the tile by u = w sigma(-E_A) + (1 - w) sigma(-E_B) ascending (see there).
// The candidates (N columns) are entity codes or, for relation queries (h, ?, t), the first R relation rows.
//
// Tile 128 x 64 (wgmma.m64n64k8): two members x (hi*hi, cross terms) x 64 x 64 / 128 threads = 128 accumulator
// registers per consumer thread, the count of the 128 x 128 single-model kernel.  Both operands come pre-split
// (the codes by round-to-nearest as for k_gemm_tf32x3, the query rows by the same truncation its producer applies),
// so the producer only issues asynchronous copies, EN_LOOKAHEAD blocks ahead.  A stage is Q hi/lo (2 x 16 KB) and
// code hi/lo (2 x 8 KB); four stages fit.  Each output element sees the K steps of its member in the order of the
// single-model kernel, so w = 1 (w = 0) reproduces member A's (B's) fused ranks and energies.
// ------------------------------------------------------------------------------------------------
constexpr int EN_BN = 64;
constexpr int EN_STAGES = 4;
constexpr int EN_LOOKAHEAD = 2;                                    // blocks in flight ahead of the one published
using EnsStage = StageShape<EN_STAGES, EN_BN>;
constexpr int EN_Q_BYTES = EnsStage::A_PLANE;                      // 16 KB (Q_hi, Q_lo)
constexpr int EN_C_BYTES = EnsStage::B_PLANE;                      // 8 KB (code_hi, code_lo)
constexpr int EN_STAGE_BYTES = EnsStage::BYTES;                    // 48 KB
constexpr int EN_SMEM_BYTES = EN_STAGES * EN_STAGE_BYTES + 1024;
constexpr int EN_FRAG = EnsStage::FRAG;                            // accumulator registers per thread and array
static_assert(EN_SMEM_BYTES <= 227 * 1024, "ensemble kernel exceeds the shared memory of a block");
static_assert(EN_LOOKAHEAD < EN_STAGES, "the lookahead needs a free stage");

struct EnsMember {
  const float* q_hi;           // [M, K] query rows, split by truncation
  const float* q_lo;
  const float* c_hi;           // [N, K] candidate codes, split by round-to-nearest
  const float* c_lo;
  const float* gold_sig;       // [M] sigmoid(energy of the gold candidate) (rank; nullptr for top-k)
  int K;                       // K % 4 == 0; the leading dimension of all four planes
};
// What every ensemble epilogue starts with: the operands the producer copies and the weights.
struct EnsPair {
  EnsMember a, b;
  double w, omw;               // weight of A and 1 - w (formed once on the host, in double)
};
// The accumulators of one tile: member A's and member B's (hi*hi, cross terms)
using EnsAcc = float[EN_FRAG];

struct EnsRankEpi : EnsPair {
  const int32_t* gold_col;     // [M]
  const uint32_t* known;       // [M, words] or nullptr
  int words;
  int32_t* raw_cnt;            // [M] += #{v : c_v >= G}
  int32_t* known_cnt;          // [M] += #{known v : c_v >= G}

  __device__ __forceinline__ void operator()(const TileCtx& t, const EnsAcc& big_a, const EnsAcc& small_a,
                                             const EnsAcc& big_b, const EnsAcc& small_b) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      int raw = 0, kn = 0;
      if (row < t.M) {
        const double G = __dadd_rn(__dmul_rn(w, (double)__ldg(a.gold_sig + row)),
                                   __dmul_rn(omw, (double)__ldg(b.gold_sig + row)));
        const int gold_c = __ldg(gold_col + row);
        for_each_col<EN_FRAG>(t, h, known, words, [&](int r, int, int col, uint32_t word) {
          const float sa = sigmoid_ref(big_a[r] + small_a[r]);
          const float sb = sigmoid_ref(big_b[r] + small_b[r]);
          const double cv = __dadd_rn(__dmul_rn(w, (double)sa), __dmul_rn(omw, (double)sb));
          if (col < t.N && (cv >= G || col == gold_c)) {   // the gold entity always counts
            ++raw;
            kn += (int)col_bit(word, col);
          }
        });
      }
      rank_counts_flush(raw, kn, row, t.M, raw_cnt, known_cnt, t.lane);
    }
  }
};

// exp(-x) for x >= 0 in double: x = n ln2 + r (Cody-Waite, |r| <= ln2 / 2), exp(-r) by its degree-12 Taylor
// polynomial (within 5e-16 relative of exp over [0, 800]), 2^-n applied as two exact power-of-two factors so that
// results down to the smallest subnormal come out; x > 800 gives 0.  Written out rather than the library's exp(),
// whose range handling keeps more registers live than the top-k epilogue has beside its accumulators.
__device__ __forceinline__ double exp_neg_d(double x) {
  if (!(x <= 800.0)) return 0.0;
  const double n = rint(x * 1.4426950408889634);
  double r = fma(-n, 6.93147180369123816490e-01, x);
  r = fma(-n, 1.90821492927058770002e-10, r);
  const double s = -r;
  double p = 2.08767569878680989792e-09;                     // 1 / 12!
  p = fma(p, s, 2.50521083854417187751e-08);                 // 1 / 11!
  p = fma(p, s, 2.75573192239858906526e-07);
  p = fma(p, s, 2.75573192239858906526e-06);
  p = fma(p, s, 2.48015873015873015873e-05);
  p = fma(p, s, 1.98412698412698412698e-04);
  p = fma(p, s, 1.38888888888888888889e-03);
  p = fma(p, s, 8.33333333333333333333e-03);
  p = fma(p, s, 4.16666666666666666667e-02);
  p = fma(p, s, 1.66666666666666666667e-01);
  p = fma(p, s, 0.5);
  p = fma(p, s, 1.0);
  p = fma(p, s, 1.0);
  const int ni = (int)n, n1 = ni >> 1, n2 = ni - n1;           // 0 <= n1, n2 <= 578
  return (p * __hiloint2double((1023 - n1) << 20, 0)) * __hiloint2double((1023 - n2) << 20, 0);
}
// sigma(-E) = 1 / (1 + exp(E)) in double from a float32 energy, through t = exp(-|E|) in [0, 1] so that the one
// reciprocal is of 1 + t in [1, 2]: sigma(-E) = 1 / (1 + t) for E <= 0 and t / (1 + t) for E > 0.  For E > 0 it does
// not saturate until t underflows (E > 745); for E < 0 it rounds to exactly 1 once exp(E) < 2^-53 (E < about -37).
// The reciprocal is MUFU's approximation refined by two Newton steps (within an ulp): the IEEE division would call its
// slow path, and a call spills the epilogue.
__device__ __forceinline__ double sigmoid_neg_d(float e) {
  const double t = exp_neg_d(fabs((double)e));
  const double d = 1.0 + t;
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  r = fma(r, fma(-d, r, 1.0), r);
  r = fma(r, fma(-d, r, 1.0), r);
  return e > 0.f ? t * r : r;
}

// TOP-K epilogue of the ensemble: for each row the tile's best min(k, 64) eligible (u, column) pairs, u ascending and
// the smaller column first on ties, where
//   u = w sigma(-E_A) + (1 - w) sigma(-E_B)   (double; separately rounded products and sum)
// is 1 - c in exact arithmetic, so ascending u is descending combined score without the saturation of the float32
// sigmoid.  Columns >= N and columns whose bit is set in `excl` are not eligible.  The pairs go in that order to
// cand[(row * tn + tile column) * kt + p]; the tail past the eligible columns is (+inf, -1).
// The energies of both tile rows are formed first (32 floats per member and lane: the accumulators die there), then
// one row at a time: every lane forms the u of its 16 eligible columns of the row (value i = 2 j + e at column
// c0 + 8 j + e, so a lane's columns increase with i) into its own slots of a 32 KB shared-memory scratch after the
// stage ring, and keeps the best of them in registers.  Each round the quad of lanes lane & ~3 (the row's 64 columns)
// keeps the best of its four by two shuffles on (u, column), and only the lane that owned it rescans its slots, as
// the merge kernel does.  166 registers, no spills.
constexpr int EN_TOPK_NV = EN_FRAG / 2;                                   // columns per lane and row
constexpr int EN_TOPK_SCRATCH = N_CONSUMERS * EN_TOPK_NV * 8;             // 32 KB
static_assert(EN_SMEM_BYTES + EN_TOPK_SCRATCH <= 227 * 1024, "ensemble top-k scratch exceeds the shared memory");

struct EnsTopKEpi : EnsPair {
  const uint32_t* excl;        // [M, words] bit v = candidate v never appears in row m (or nullptr)
  int words;                   // ceil(N / 32)
  int kt;                      // candidates per row and tile, min(k, EN_BN)
  int tn;                      // N tiles
  EnsCand* cand;               // [M, tn, kt]

  __device__ __forceinline__ void operator()(const TileCtx& t, const EnsAcc& big_a, const EnsAcc& small_a,
                                             const EnsAcc& big_b, const EnsAcc& small_b) const {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw), aligned = (raw + 1023u) & ~1023u;
    // this lane's slot i is ubuf[i * N_CONSUMERS]: a warp's accesses are consecutive doubles
    double* ubuf = reinterpret_cast<double*>(smem_raw + (aligned - raw) + EN_STAGES * EN_STAGE_BYTES) +
                   (t.warp * 32 + t.lane);
    const bool writer = (t.lane & 3) == 0;
    const EnsCand none{INFINITY, -1, 0};
    float ea[2][EN_TOPK_NV], eb[2][EN_TOPK_NV];   // the members' energies
    uint32_t eligible[2];                          // bit i: column i of row r0 + 8 h may be returned
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      eligible[h] = 0u;
      for_each_col<EN_FRAG>(t, h, excl, words, [&](int r, int i, int col, uint32_t word) {
        ea[h][i] = big_a[r] + small_a[r];
        eb[h][i] = big_b[r] + small_b[r];
        if (t.r0 + 8 * h < t.M && col < t.N && !col_bit(word, col)) eligible[h] |= 1u << i;
      });
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = t.r0 + 8 * h;
      const bool row_ok = row < t.M;
      uint32_t left = eligible[h];
#pragma unroll
      for (int i = 0; i < EN_TOPK_NV; ++i)   // u of the eligible columns only
        if ((left >> i) & 1u)
          ubuf[i * N_CONSUMERS] = __dadd_rn(__dmul_rn(w, sigmoid_neg_d(ea[h][i])),
                                            __dmul_rn(omw, sigmoid_neg_d(eb[h][i])));
      int bi;
      double bu;
      auto rescan = [&]() {   // the lane's best (u, i) among its slots still left
        bi = -1;
        bu = INFINITY;
#pragma unroll
        for (int i = 0; i < EN_TOPK_NV; ++i)
          if ((left >> i) & 1u) {
            const double x = ubuf[i * N_CONSUMERS];
            if (bi < 0 || x < bu) {
              bu = x;
              bi = i;
            }
          }
      };
      rescan();
      // candidate p of this row (formed at the store: a live pointer would cost a register pair)
      auto slot = [&](int p) { return cand + ((size_t)row * tn + (size_t)(t.n0 / EN_BN)) * kt + p; };
      int p = 0;
      for (; p < kt; ++p) {
        const int mine = bi < 0 ? 0x7fffffff : t.c0 + 8 * (bi >> 1) + (bi & 1);
        double qu = bu;
        int qc = mine;
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const double ou = __shfl_xor_sync(0xffffffffu, qu, o);
          const int oc = __shfl_xor_sync(0xffffffffu, qc, o);
          if (oc != 0x7fffffff && (qc == 0x7fffffff || ou < qu || (ou == qu && oc < qc))) {
            qu = ou;
            qc = oc;
          }
        }
        if (!__any_sync(0xffffffffu, qc != 0x7fffffff)) break;   // the warp's rows ran dry
        if (bi >= 0 && qc == mine) {
          left &= ~(1u << bi);
          rescan();
        }
        if (writer && row_ok) *slot(p) = qc == 0x7fffffff ? none : EnsCand{qu, qc, 0};
      }
      if (writer && row_ok)
        for (; p < kt; ++p) *slot(p) = none;
    }
  }
};

// Persistent like k_gemm_tf32x3 (N tiles fastest); a tile is num_kb_a + num_kb_b consecutive k-blocks of the CTA's
// stage sequence.  EPI: EnsRankEpi or EnsTopKEpi.
template <class EPI>
__global__ void __launch_bounds__(N_THREADS, 1)
    k_gemm_ensemble(int M, int N, int n_tiles, const EPI re) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[EN_STAGES], empty_bar[EN_STAGES];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, lane = tid & 31;
  const int tn = (N + EN_BN - 1) / EN_BN;
  const int nkb_a = (re.a.K + BK - 1) / BK, nkb_b = (re.b.K + BK - 1) / BK, nkb = nkb_a + nkb_b;
  const int n_mine = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int total_g = n_mine * nkb;

  if (tid == 0) init_barriers<EN_STAGES>(full_bar, empty_bar);
  __syncthreads();

  if (tid < N_PRODUCERS) {
    // ================= producer warpgroup: asynchronous copies only =================
    const int c = tid & 7;                     // 16 B chunk within the 128 B K-row
    const int rbase = tid >> 3;                // tile rows rbase + 16 i
    const uint32_t soff = swz(rbase, c);
    int i_tile = (int)blockIdx.x, i_kb = 0, stage = 0;
    auto issue = [&]() {                       // copies the next block of the sequence into `stage`
      const bool mb = i_kb >= nkb_a;
      const float* qh = mb ? re.b.q_hi : re.a.q_hi;
      const float* ql = mb ? re.b.q_lo : re.a.q_lo;
      const float* ch = mb ? re.b.c_hi : re.a.c_hi;
      const float* cl = mb ? re.b.c_lo : re.a.c_lo;
      const int K = mb ? re.b.K : re.a.K;
      const int k = (mb ? i_kb - nkb_a : i_kb) * BK + c * 4;
      const bool col_ok = k < K;               // K % 4 == 0: a 16 B chunk is entirely valid or entirely padding
      const int m0 = (i_tile / tn) * BM, n0 = (i_tile % tn) * EN_BN;
      const uint32_t st = smem_base + stage * EN_STAGE_BYTES + soff;
#pragma unroll
      for (int i = 0; i < BM / 16; ++i) {
        const int row = m0 + rbase + 16 * i;
        const bool ok = col_ok && row < M;
        const size_t o = ok ? (size_t)row * K + k : 0;
        cp_async16(st + 2048 * i, qh + o, ok ? 16u : 0u);
        cp_async16(st + EN_Q_BYTES + 2048 * i, ql + o, ok ? 16u : 0u);
      }
#pragma unroll
      for (int i = 0; i < EN_BN / 16; ++i) {
        const int row = n0 + rbase + 16 * i;
        const bool ok = col_ok && row < N;
        const size_t o = ok ? (size_t)row * K + k : 0;
        cp_async16(st + 2 * EN_Q_BYTES + 2048 * i, ch + o, ok ? 16u : 0u);
        cp_async16(st + 2 * EN_Q_BYTES + EN_C_BYTES + 2048 * i, cl + o, ok ? 16u : 0u);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      stage = stage + 1 == EN_STAGES ? 0 : stage + 1;
      if (++i_kb == nkb) {
        i_kb = 0;
        i_tile += (int)gridDim.x;
      }
    };
    // block g goes to stage g % EN_STAGES in use round g / EN_STAGES; the copies of blocks g + 1 .. g + EN_LOOKAHEAD
    // are in flight while block g is published.  One commit group per block (empty past the end) keeps the count.
    for (int g = 0; g < EN_LOOKAHEAD; ++g) {
      if (g < total_g) {
        mbar_wait(&empty_bar[g % EN_STAGES], ((uint32_t)(g / EN_STAGES) & 1u) ^ 1u);
        issue();
      } else {
        asm volatile("cp.async.commit_group;" ::: "memory");
      }
    }
    for (int g = 0; g < total_g; ++g) {
      const int gn = g + EN_LOOKAHEAD;
      if (gn < total_g) {
        mbar_wait(&empty_bar[gn % EN_STAGES], ((uint32_t)(gn / EN_STAGES) & 1u) ^ 1u);
        issue();
      } else {
        asm volatile("cp.async.commit_group;" ::: "memory");
      }
      asm volatile("cp.async.wait_group %0;" ::"n"(EN_LOOKAHEAD) : "memory");   // block g has landed
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");             // generic-proxy writes -> tensor core
      mbar_arrive(&full_bar[g % EN_STAGES]);
    }
  } else {
    // ================= consumer warpgroups =================
    const int ctid = tid - N_PRODUCERS;
    const int wg = ctid >> 7, warp = ctid >> 5;
    const uint32_t a_rows = (uint32_t)(wg * 64 * 128);
    float big_a[EN_FRAG], small_a[EN_FRAG], big_b[EN_FRAG], small_b[EN_FRAG];
    for (int ti = 0; ti < n_mine; ++ti) {
      const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
      const int m0 = (tile / tn) * BM, n0 = (tile % tn) * EN_BN;
      consume_tile<EnsStage>(smem_base, full_bar, empty_bar, ti * nkb, nkb_a, a_rows, big_a, small_a);
      consume_tile<EnsStage>(smem_base, full_bar, empty_bar, ti * nkb + nkb_a, nkb_b, a_rows, big_b, small_b);
      const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = n0 + 2 * (lane & 3);
      const TileCtx t{tile, m0, n0, r0, c0, M, N, lane, warp};
      re(t, big_a, small_a, big_b, small_b);
    }
  }
}

// In-place truncation split of [count] floats (count % 4 == 0, 16 B aligned): a -> hi (kept in a) and lo, the split
// the k_gemm_tf32x3 producer applies to its streamed operand
__global__ void k_split_trunc(float* __restrict__ a, float* __restrict__ lo, int64_t count4) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(a)[i], h, l;
    split_tf32_trunc(v.x, h.x, l.x);
    split_tf32_trunc(v.y, h.y, l.y);
    split_tf32_trunc(v.z, h.z, l.z);
    split_tf32_trunc(v.w, h.w, l.w);
    reinterpret_cast<float4*>(a)[i] = h;
    reinterpret_cast<float4*>(lo)[i] = l;
  }
}

}  // namespace

// SM count of the current device
static int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// Tiles of an [M, N] output in 128 x bn tiles: the one count the launchers, the kernels' part arrays
// (gemm_onen_loss_parts, gemm_variational_kl_parts) and the kernels' tile walk agree on
static int64_t tiles_of(int64_t M, int64_t N, int bn) { return ((M + BM - 1) / BM) * ((N + bn - 1) / bn); }

// The one launch path of the persistent kernels: the dynamic shared memory size is raised once per kernel, `tiles`
// is checked against `tile_limit` (what the kernel's index arithmetic holds in an int), and min(tiles, SMs) CTAs walk
// the tiles, at most one per SM.  `what` names the launcher in the error text, `label` the kernel.
template <auto Kernel, class... Args>
static int launch_persistent(const char* what, const char* label, int smem, int64_t tiles, int64_t tile_limit,
                             cudaStream_t st, Args... args) {
  static bool attr_set = false;   // one per kernel: Kernel is a template argument
  if (!attr_set) {
    int rc = rgcn_check_cuda(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem),
                             (std::string("cudaFuncSetAttribute(") + label + " smem)").c_str());
    if (rc) return rc;
    attr_set = true;
  }
  if (tiles > tile_limit) {
    rgcn_set_error(std::string(what) + ": too many tiles");
    return RGCN_ERR_INVALID;
  }
  const unsigned grid = (unsigned)std::min<int64_t>(tiles, sm_count());
  Kernel<<<grid, N_THREADS, smem, st>>>(args...);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), label);
}
constexpr int64_t TILE_LIMIT = 0x7fffffffLL;         // the tile index is an int
constexpr int64_t PART_TILE_LIMIT = TILE_LIMIT / 8;  // ... and so is part[tile * 8 + warp]'s count (VarEpi, BceEpi)

// The NT kernel with the epilogue `epi` of EPI over an [M, N] output
template <int EPI>
static int launch_nt(const char* what, const char* label, int64_t tile_limit, cudaStream_t st, const float* A,
                     int64_t lda, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M, int N, int K,
                     const typename Epilogue<EPI>::type& epi) {
  const int64_t tiles = tiles_of(M, N, BN);
  return launch_persistent<k_gemm_tf32x3<EPI>>(what, label, SMEM_BYTES, tiles, tile_limit, st, A, lda, Bt_hi, Bt_lo,
                                               ldb, M, N, K, (int)tiles, epi);
}

// grid of the element-wise split kernels (256 threads, grid-stride)
static int split_blocks(int64_t items) { return (int)std::min<int64_t>((items + 255) / 256, 132 * 8); }

int launch_gemm_split_b(const float* B, int64_t ldb, int N, int K, int transposed, float* hi, float* lo,
                        cudaStream_t st) {
  const int64_t total = (int64_t)N * K;
  if (total == 0) return RGCN_OK;
  k_split_b<<<split_blocks(total), 256, 0, st>>>(B, ldb, N, K, transposed, hi, lo);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_split_b");
}

int launch_gemm_tf32x3(const float* A, int64_t lda, const float* Bt_hi, const float* Bt_lo, int64_t ldb,
                       float* C, int64_t ldc, int M, int N, int K, int accumulate, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (K % 4 != 0 || N % 4 != 0 || lda % 4 != 0 || ldb % 4 != 0 || ldc % 4 != 0) {
    rgcn_set_error("gemm_tf32x3: K, N and leading dimensions must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  if (K == 0) {   // empty contraction: C = 0 (or unchanged); the kernel would publish accumulators no MMA ever wrote
    if (accumulate) return RGCN_OK;
    return rgcn_check_cuda(cudaMemset2DAsync(C, ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, st), "memset(C)");
  }
  return launch_nt<EPI_STORE>("gemm_tf32x3", "k_gemm_tf32x3", TILE_LIMIT, st, A, lda, Bt_hi, Bt_lo, ldb, M, N, K,
                              StoreEpi{C, ldc, accumulate});
}

// GEMM with the bias + activation epilogue (EPI = 6): C[M, N] = act(A[M, K] B + bias), B pre-split as Bt [N, K].
int launch_gemm_bias_act_tf32x3(const float* A, int64_t lda, const float* Bt_hi, const float* Bt_lo, int64_t ldb,
                                const float* bias, int relu, float* C, int64_t ldc, int M, int N, int K,
                                cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (K <= 0 || K % 4 != 0 || N % 4 != 0 || lda % 4 != 0 || ldb % 4 != 0 || ldc % 4 != 0) {
    rgcn_set_error("gemm_bias_act_tf32x3: K > 0; K, N and leading dimensions must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_BIAS_ACT>("gemm_bias_act_tf32x3", "k_gemm_tf32x3<bias_act>", TILE_LIMIT, st, A, lda, Bt_hi,
                                 Bt_lo, ldb, M, N, K, BiasActEpi{C, ldc, bias, relu});
}

// Scoring GEMM with the ranking epilogue: queries Q [M,K] against the pre-split entity codes Bt [N,K]; the counts
// accumulate (+=) into raw_cnt / known_cnt (zeroed by the caller).
int launch_gemm_rank_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const float* gold_sig, const int32_t* gold_col, const uint32_t* known,
                            int words, int32_t* raw_cnt, int32_t* known_cnt, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (K <= 0 || K % 4 != 0 || ldq % 4 != 0 || ldb % 4 != 0) {
    rgcn_set_error("gemm_rank_tf32x3: K > 0; K and leading dimensions must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_RANK>("gemm_rank_tf32x3", "k_gemm_tf32x3<rank>", TILE_LIMIT, st, Q, ldq, Bt_hi, Bt_lo, ldb, M,
                             N, K, RankEpi{gold_sig, gold_col, known, words, raw_cnt, known_cnt});
}

// Scoring GEMM with the top-k epilogue (EPI = 4): queries Q [M,K] against the pre-split entity codes Bt [N,K]; each
// row's best k eligible (energy, column) pairs of every N tile go to cand [M, ceil(N / BN), k].
int launch_gemm_topk_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const uint32_t* excl, int words, int k, uint2* cand, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (K <= 0 || K % 4 != 0 || ldq % 4 != 0 || ldb % 4 != 0 || k < 1 || k > BN) {
    rgcn_set_error("gemm_topk_tf32x3: K > 0; K and leading dimensions must be multiples of 4; 1 <= k <= 128");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_TOPK>("gemm_topk_tf32x3", "k_gemm_tf32x3<topk>", TILE_LIMIT, st, Q, ldq, Bt_hi, Bt_lo, ldb, M,
                             N, K, TopKEpi{excl, words, k, (N + BN - 1) / BN, cand});
}

int64_t gemm_onen_loss_parts(int64_t M, int N) { return tiles_of(M, N, BN) * 8; }

// 1-N scoring GEMM with the BCE epilogue (EPI = 5): queries Q [M,K] against the pre-split entity codes Bt [N,K];
// gemm_onen_loss_parts(M, N) loss parts, and Gt [N, ldgt] (transposed gradients of the energies) unless Gt is null.
int launch_gemm_onen_tf32x3(const float* Q, int64_t ldq, const float* Bt_hi, const float* Bt_lo, int64_t ldb, int M,
                            int N, int K, const uint32_t* labels, float pos, float neg, float scale,
                            const float* g_scale, float* Gt, int64_t ldgt, float* loss_part, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (K <= 0 || K % 4 != 0 || ldq % 4 != 0 || ldb % 4 != 0) {
    rgcn_set_error("gemm_onen_tf32x3: K > 0; K and leading dimensions must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_BCE>("gemm_onen_tf32x3", "k_gemm_tf32x3<onen>", PART_TILE_LIMIT, st, Q, ldq, Bt_hi, Bt_lo, ldb,
                            M, N, K, BceEpi{labels, (N + 31) / 32, pos, neg, scale, g_scale, Gt, ldgt, loss_part});
}

int launch_split_trunc(float* a, float* lo, int64_t count, cudaStream_t st) {
  if (count == 0) return RGCN_OK;
  const int64_t count4 = count / 4;
  k_split_trunc<<<split_blocks(count4), 256, 0, st>>>(a, lo, count4);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_split_trunc");
}

// Two-member ranking GEMM (see k_gemm_ensemble); the counts accumulate (+=) into raw_cnt / known_cnt.
int launch_gemm_ensemble_rank_tf32x3(const float* qa_hi, const float* qa_lo, const float* ca_hi, const float* ca_lo,
                                     const float* gold_sig_a, int Ka, const float* qb_hi, const float* qb_lo,
                                     const float* cb_hi, const float* cb_lo, const float* gold_sig_b, int Kb, int M,
                                     int N, double w, double omw, const int32_t* gold_col, const uint32_t* known,
                                     int words, int32_t* raw_cnt, int32_t* known_cnt, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (Ka <= 0 || Ka % 4 != 0 || Kb <= 0 || Kb % 4 != 0) {
    rgcn_set_error("gemm_ensemble_rank_tf32x3: K > 0 and K % 4 == 0 for both members");
    return RGCN_ERR_INVALID;
  }
  const int64_t tiles = tiles_of(M, N, EN_BN);
  EnsRankEpi re;
  static_cast<EnsPair&>(re) = {{qa_hi, qa_lo, ca_hi, ca_lo, gold_sig_a, Ka}, {qb_hi, qb_lo, cb_hi, cb_lo, gold_sig_b, Kb},
                               w, omw};
  re.gold_col = gold_col;
  re.known = known;
  re.words = words;
  re.raw_cnt = raw_cnt;
  re.known_cnt = known_cnt;
  return launch_persistent<k_gemm_ensemble<EnsRankEpi>>("gemm_ensemble_rank_tf32x3", "k_gemm_ensemble<rank>",
                                                        EN_SMEM_BYTES, tiles, TILE_LIMIT, st, M, N, (int)tiles, re);
}

// Two-member top-k GEMM (see EnsTopKEpi): each row's best min(k, 64) eligible (u, column) pairs of every 64-column
// tile go to cand [M, ceil(N / 64), min(k, 64)].
int launch_gemm_ensemble_topk_tf32x3(const float* qa_hi, const float* qa_lo, const float* ca_hi, const float* ca_lo,
                                     int Ka, const float* qb_hi, const float* qb_lo, const float* cb_hi,
                                     const float* cb_lo, int Kb, int M, int N, double w, double omw,
                                     const uint32_t* excl, int words, int k, EnsCand* cand, cudaStream_t st) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (Ka <= 0 || Ka % 4 != 0 || Kb <= 0 || Kb % 4 != 0 || k < 1 || k > 128) {
    rgcn_set_error("gemm_ensemble_topk_tf32x3: K > 0 and K % 4 == 0 for both members; 1 <= k <= 128");
    return RGCN_ERR_INVALID;
  }
  const int64_t tiles = tiles_of(M, N, EN_BN);
  EnsTopKEpi te;
  static_cast<EnsPair&>(te) = {{qa_hi, qa_lo, ca_hi, ca_lo, nullptr, Ka}, {qb_hi, qb_lo, cb_hi, cb_lo, nullptr, Kb},
                               w, omw};
  te.excl = excl;
  te.words = words;
  te.kt = ensemble_topk_per_tile(k);
  te.tn = (N + EN_BN - 1) / EN_BN;
  te.cand = cand;
  return launch_persistent<k_gemm_ensemble<EnsTopKEpi>>("gemm_ensemble_topk_tf32x3", "k_gemm_ensemble<topk>",
                                                        EN_SMEM_BYTES + EN_TOPK_SCRATCH, tiles, TILE_LIMIT, st, M, N, (int)tiles, te);
}

// Highway gate GEMM with the blend epilogue (EPI = 2): z = c2 @ W + bias with W pre-split as Bt = W^T [d, d];
// out = c2 + sigmoid(z) (c1 - c2), gate = sigmoid(z).  All matrices [M, d] row-major, contiguous.
int launch_gemm_highway_tf32x3(const float* c2, const float* Bt_hi, const float* Bt_lo, const float* bias,
                               const float* c1, float* out, float* gate, int M, int d, cudaStream_t st) {
  if (M == 0) return RGCN_OK;
  if (d <= 0 || d % 4 != 0) {
    rgcn_set_error("gemm_highway_tf32x3: d > 0, d % 4 == 0");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_HIGHWAY>("gemm_highway_tf32x3", "k_gemm_tf32x3<highway>", TILE_LIMIT, st, c2, d, Bt_hi, Bt_lo,
                                d, M, d, d, HighwayEpi{bias, c1, c2, out, gate, d});
}

int launch_gemm_split_b_interleave(const float* Wmu, const float* Wsig, int d, int w, int transposed, float* hi,
                                   float* lo, cudaStream_t st) {
  const int64_t total = (int64_t)2 * d * w;
  if (total == 0) return RGCN_OK;
  k_split_b_interleave<<<split_blocks(total), 256, 0, st>>>(Wmu, Wsig, d, w, transposed, hi, lo);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_split_b_interleave");
}

int64_t gemm_variational_kl_parts(int64_t M, int w) { return tiles_of(M, 2 * (int64_t)w, BN) * 8; }

// Variational head GEMM (EPI = 3): P = H W_int + [b_mu, b_sigma] interleaved, z = mu + exp(l) eps, one KL part per
// consumer warp and tile (gemm_variational_kl_parts of them).  H [M, d], P [M, 2w], eps / z [M, w], contiguous.
int launch_gemm_variational_tf32x3(const float* H, const float* Bt_hi, const float* Bt_lo, const float* b_mu,
                                   const float* b_sigma, const float* eps, float* P, float* z, float* kl_part, int M,
                                   int d, int w, cudaStream_t st) {
  if (M == 0) return RGCN_OK;
  if (d <= 0 || d % 4 != 0 || w <= 0 || w % 2 != 0) {
    rgcn_set_error("gemm_variational_tf32x3: d > 0, d % 4 == 0, w > 0, w % 2 == 0");
    return RGCN_ERR_INVALID;
  }
  return launch_nt<EPI_VAR>("gemm_variational_tf32x3", "k_gemm_tf32x3<variational>", PART_TILE_LIMIT, st, H, d, Bt_hi,
                            Bt_lo, d, M, 2 * w, d, VarEpi{b_mu, b_sigma, eps, P, 2 * w, z, kl_part, w});
}

// C[M,N] (+)= A^T B, A [K,M] row-major, B [K,N] row-major (see k_gemm_tn_tf32x3)
int launch_gemm_tn_tf32x3(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc,
                          int M, int N, int K, int accumulate, cudaStream_t st, int max_splits) {
  if (M == 0 || N == 0) return RGCN_OK;
  if (M % 4 != 0 || N % 4 != 0 || lda % 4 != 0 || ldb % 4 != 0 || ldc % 4 != 0) {
    rgcn_set_error("gemm_tn_tf32x3: M, N and leading dimensions must be multiples of 4");
    return RGCN_ERR_INVALID;
  }
  if (!accumulate) {
    int rc = rgcn_check_cuda(cudaMemset2DAsync(C, ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, st),
                             "memset(C)");
    if (rc) return rc;
  }
  if (K == 0) return RGCN_OK;
  static bool attr_set = false;
  if (!attr_set) {
    int rc = rgcn_check_cuda(cudaFuncSetAttribute(k_gemm_tn_tf32x3, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  TN_SMEM_BYTES),
                             "cudaFuncSetAttribute(gemm tn smem)");
    if (rc) return rc;
    attr_set = true;
  }
  // Split count: one CTA per SM, so the CTAs run in waves of `sms`; a split of kb_per_split k-blocks costs its
  // k-blocks plus about TN_KB_FIXED k-blocks of pipeline fill and epilogue.  Take the split count with the least
  // waves x (kb_per_split + TN_KB_FIXED), the smallest one on ties.  When the tiles fit the SMs this is one wave of
  // floor(sms / tiles) splits for long K (M = N = 512, K = 5 M on 132 SMs: 8 splits, 128 CTAs); with more tiles
  // than one wave holds, more (shorter) splits fill the last wave.
  constexpr int64_t TN_KB_FIXED = 4;
  const int64_t tiles = tiles_of(M, N, BN);
  const int64_t kb_total = (K + BK - 1) / BK, sms = sm_count();
  int64_t splits = 1, kb_per_split = kb_total, best = -1;
  for (int64_t s = 1; s <= kb_total && (s == 1 || s * tiles <= 8 * sms) && (max_splits <= 0 || s <= max_splits); ++s) {
    const int64_t kps = (kb_total + s - 1) / s, s_eff = (kb_total + kps - 1) / kps;   // no empty split
    const int64_t cost = (s_eff * tiles + sms - 1) / sms * (kps + TN_KB_FIXED);
    if (best < 0 || cost < best) {
      best = cost;
      splits = s_eff;
      kb_per_split = kps;
    }
  }
  if (tiles * splits > 0x7fffffffLL) {
    rgcn_set_error("gemm_tn_tf32x3: too many tiles");
    return RGCN_ERR_INVALID;
  }
  k_gemm_tn_tf32x3<<<(unsigned)(tiles * splits), N_THREADS, TN_SMEM_BYTES, st>>>(A, lda, B, ldb, C, ldc, M, N, K,
                                                                                 (int)kb_per_split);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "k_gemm_tn_tf32x3");
}
