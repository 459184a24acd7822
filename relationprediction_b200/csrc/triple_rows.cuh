// triple_rows.cuh -- the row arithmetic of the DistMult, ComplEx, RotatE, TransE, QuatE and HolE triple scorers: one
// warp owns one triple (s, r, o) and each lane forms its share of the energy and of the squared norms of the gathered
// rows.  Shared by the NegativeSampling scorers (distmult.cu / complex.cu / rotate.cu / transe.cu / quate.cu / hole.cu)
// and the
// self-adversarial scorer (self_adversarial.cu), so both objectives score a triple with the same float operations in
// the same order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// W consecutive floats (W = 4: 16-byte aligned, W = 2: 8-byte aligned)
template <int W>
struct Vec;
template <>
struct Vec<4> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[4]) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  }
  __device__ __forceinline__ static void store(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
  __device__ __forceinline__ static void red(float* p, const float (&v)[4]) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]),
                 "f"(v[3])
                 : "memory");
  }
};
template <>
struct Vec<2> {
  __device__ __forceinline__ static void load(const float* p, float (&v)[2]) {
    const float2 t = __ldg(reinterpret_cast<const float2*>(p));
    v[0] = t.x, v[1] = t.y;
  }
  __device__ __forceinline__ static void store(float* p, const float (&v)[2]) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  }
  __device__ __forceinline__ static void red(float* p, const float (&v)[2]) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
  }
};

// DistMult (bilinear_diag.py:14-24): e = sum_k e1 r e2, rows read as float4 (d % 4 == 0)
struct DistMultRows {
  // this lane's share of the energy (e) and of the squared norms of the three rows (q), both starting from 0
  __device__ __forceinline__ static void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                                                 int s, int r, int o, int lane, float& e, float& q) {
    const float4* e1 = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* e2 = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    const int d4 = d >> 2;
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(e1 + i), b = __ldg(rr + i), c = __ldg(e2 + i);
      e = fmaf(a.x * b.x, c.x, e);
      e = fmaf(a.y * b.y, c.y, e);
      e = fmaf(a.z * b.z, c.z, e);
      e = fmaf(a.w * b.w, c.w, e);
      q += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
      q += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
      q += c.x * c.x + c.y * c.y + c.z * c.z + c.w * c.w;
    }
  }
};

// ComplEx (complex.py:38-41): a lane owns the column pairs (k, k + h) of all three rows, h = d / 2; W = 4 when
// d % 8 == 0, else 2 (the imaginary half is then only 8-byte aligned)
template <int W>
struct ComplexRows {
  __device__ __forceinline__ static void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                                                 int s, int r, int o, int lane, float& e, float& q) {
    const float* e1 = codes + (size_t)s * d;
    const float* rr = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    const int h = d >> 1;
    for (int k = lane * W; k < h; k += 32 * W) {
      float ar[W], ai[W], br[W], bi[W], cr[W], ci[W];
      Vec<W>::load(e1 + k, ar), Vec<W>::load(e1 + h + k, ai);
      Vec<W>::load(rr + k, br), Vec<W>::load(rr + h + k, bi);
      Vec<W>::load(e2 + k, cr), Vec<W>::load(e2 + h + k, ci);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        // e1r*rr*e2r + e1i*rr*e2i + e1r*ri*e2i - e1i*ri*e2r
        e = fmaf(br[j], fmaf(ar[j], cr[j], ai[j] * ci[j]), e);
        e = fmaf(bi[j], fmaf(ar[j], ci[j], -ai[j] * cr[j]), e);
        q += ar[j] * ar[j] + ai[j] * ai[j];
        q += br[j] * br[j] + bi[j] * bi[j];
        q += cr[j] * cr[j] + ci[j] * ci[j];
      }
    }
  }
};

// |u| for RotatE: the hardware square root (sqrt.approx.ftz.f32, one MUFU instruction).  The IEEE sqrtf calls a
// slow-path subroutine, and the registers live across that call go to local memory.
__device__ __forceinline__ float rotate_modulus(float ur, float ui) {
  float m;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(m) : "f"(__fmaf_rn(ur, ur, __fmul_rn(ui, ui))));
  return m;
}

// RotatE: u = a e^{i theta} - c for one column pair (a = ar + i ai, c = cr + i ci), with (sn, cs) = sincos(theta) --
// full range reduction: phases are unbounded.  The scorer, its backward and the self-adversarial scorer all form u
// here, so the backward differentiates exactly the forward's residual.
__device__ __forceinline__ void rotate_residual(float ar, float ai, float th, float cr, float ci, float& ur, float& ui,
                                                float& sn, float& cs) {
  sincosf(th, &sn, &cs);
  ur = fmaf(ar, cs, fmaf(-ai, sn, -cr));
  ui = fmaf(ar, sn, fmaf(ai, cs, -ci));
}

// RotatE (DESIGN.md section 1): energy gamma - sum_k |a_k e^{i theta_k} - c_k| with entity rows [re | im] (h = d / 2
// columns each) and the phases theta in the first h columns of the relation row; the other h are never read.  A lane
// owns the column pairs (k, k + h) as ComplexRows<W> does; lane 0's share carries gamma.  q gets the squared norms of
// the two entity rows only: phases are not regularised.
template <int W>
struct RotateRows {
  float gamma;

  __device__ __forceinline__ void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d, int s,
                                          int r, int o, int lane, float& e, float& q) const {
    const float* e1 = codes + (size_t)s * d;
    const float* th = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    const int h = d >> 1;
    if (lane == 0) e += gamma;
    for (int k = lane * W; k < h; k += 32 * W) {
      float ar[W], ai[W], t[W], cr[W], ci[W];
      Vec<W>::load(e1 + k, ar), Vec<W>::load(e1 + h + k, ai);
      Vec<W>::load(th + k, t);
      Vec<W>::load(e2 + k, cr), Vec<W>::load(e2 + h + k, ci);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        float ur, ui, sn, cs;
        rotate_residual(ar[j], ai[j], t[j], cr[j], ci[j], ur, ui, sn, cs);
        e -= rotate_modulus(ur, ui);
        q += ar[j] * ar[j] + ai[j] * ai[j];
        q += cr[j] * cr[j] + ci[j] * ci[j];
      }
    }
  }
};

// TransE: u_k = (h_k + r_k) - t_k with both roundings pinned, so that the ranker's query row q = h + r (rounded once)
// gives the same per-column term.  The scorer, its backward and the self-adversarial scorer all form u here.
__device__ __forceinline__ float transe_residual(float h, float r, float t) { return __fsub_rn(__fadd_rn(h, r), t); }

// TransE (DESIGN.md section 1): energy gamma - sum_k |h_k + r_k - t_k| over all d columns of plain real rows.  A lane
// owns W consecutive columns (W = 4: d % 4 == 0 is required); lane 0's share carries gamma.  q gets the squared norms
// of all three rows: a translation is regularised like a DistMult relation.
template <int W>
struct TransERows {
  float gamma;

  __device__ __forceinline__ void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d, int s,
                                          int r, int o, int lane, float& e, float& q) const {
    const float* e1 = codes + (size_t)s * d;
    const float* rr = rel + (size_t)r * d;
    const float* e2 = codes + (size_t)o * d;
    if (lane == 0) e += gamma;
    for (int k = lane * W; k < d; k += 32 * W) {
      float a[W], b[W], c[W];
      Vec<W>::load(e1 + k, a), Vec<W>::load(rr + k, b), Vec<W>::load(e2 + k, c);
#pragma unroll
      for (int j = 0; j < W; ++j) {
        e -= fabsf(transe_residual(a[j], b[j], c[j]));
        q += a[j] * a[j] + b[j] * b[j] + c[j] * c[j];
      }
    }
  }
};

// QuatE (DESIGN.md section 1): quaternion k of a row is the aligned float4 at column 4k, (x, y, z, w) = a + b i + c j +
// d k.  Every QuatE kernel -- scorer, backward, self-adversarial scorer, query rows, query backward -- forms the
// Hamilton product and the normalised relation quaternion with these helpers, so they all use the same float
// operations.
constexpr float QUATE_EPS = 1e-12f;

__device__ __forceinline__ float4 quat_conj(float4 q) { return make_float4(q.x, -q.y, -q.z, -q.w); }

__device__ __forceinline__ float quat_dot(float4 p, float4 q, float acc) {
  return fmaf(p.w, q.w, fmaf(p.z, q.z, fmaf(p.y, q.y, fmaf(p.x, q.x, acc))));
}

// the Hamilton product p q
__device__ __forceinline__ float4 quat_mul(float4 p, float4 q) {
  return make_float4(fmaf(p.x, q.x, -fmaf(p.y, q.y, fmaf(p.z, q.z, p.w * q.w))),
                     fmaf(p.x, q.y, fmaf(p.y, q.x, fmaf(p.z, q.w, -(p.w * q.z)))),
                     fmaf(p.x, q.z, fmaf(-p.y, q.w, fmaf(p.z, q.x, p.w * q.y))),
                     fmaf(p.x, q.w, fmaf(p.y, q.z, fmaf(-p.z, q.y, p.w * q.x))));
}

// r / max(|r|, eps) with |r| in m.  IEEE-rounded square root and division: a quaternion whose norm is a power of two
// normalises exactly.
__device__ __forceinline__ float4 quat_normalize(float4 r, float& m) {
  m = __fsqrt_rn(quat_dot(r, r, 0.f));
  const float s = fmaxf(m, QUATE_EPS);
  return make_float4(__fdiv_rn(r.x, s), __fdiv_rn(r.y, s), __fdiv_rn(r.z, s), __fdiv_rn(r.w, s));
}

// the gradient g with respect to rh = quat_normalize(r, m), taken back to r: (g - rh <rh, g>) / m when m > eps, else
// g / eps (the clamped norm is then a constant), so a zero quaternion never gives a NaN
__device__ __forceinline__ float4 quat_normalize_bwd(float4 rh, float m, float4 g) {
  if (!(m > QUATE_EPS)) return make_float4(g.x / QUATE_EPS, g.y / QUATE_EPS, g.z / QUATE_EPS, g.w / QUATE_EPS);
  const float c = quat_dot(rh, g, 0.f);
  return make_float4(fmaf(-rh.x, c, g.x) / m, fmaf(-rh.y, c, g.y) / m, fmaf(-rh.z, c, g.z) / m,
                     fmaf(-rh.w, c, g.w) / m);
}

// QuatE: e = sum_k <h_k (x) rh_k, t_k> with rh_k the normalised relation quaternion; a lane owns whole quaternions (one
// float4 per row, d % 4 == 0).  q gets the squared norms of the three raw rows, DistMult's L2 term.
struct QuatERows {
  __device__ __forceinline__ static void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                                                 int s, int r, int o, int lane, float& e, float& q) {
    const float4* e1 = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* e2 = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    const int d4 = d >> 2;
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(e1 + i), b = __ldg(rr + i), c = __ldg(e2 + i);
      float m;
      e = quat_dot(quat_mul(a, quat_normalize(b, m)), c, e);
      q += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
      q += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
      q += c.x * c.x + c.y * c.y + c.z * c.z + c.w * c.w;
    }
  }
};

// HolE (DESIGN.md section 1) on rows already in the real Fourier basis x~ = x U.  Float4 i of a row holds columns
// 4i..4i+3.  For i > 0 those are two frequencies, (re, im) pairs.  Float4 0 (lane 0's first) holds DC and Nyquist, two
// real columns, then frequency 1.  With the weights w0 = sqrt(d) (DC, Nyquist) and w1 = sqrt(d / 2) (every pair):
//   E = sum over the columns of  w * Re(conj(h r) t),  DC and Nyquist taken as real numbers.
// Every HolE kernel -- scorer, backward, self-adversarial scorer, query rows, query backward -- forms its products with
// these helpers, so they all use the same float operations.
__device__ __forceinline__ void hole_weights(int d, float& w0, float& w1) {
  w0 = __fsqrt_rn((float)d);
  w1 = __fsqrt_rn(0.5f * (float)d);
}

// w (a b) for float4 i of two rows; first = (i == 0): x and y are then the real DC and Nyquist columns
__device__ __forceinline__ float4 hole_mul(float4 a, float4 b, bool first, float w0, float w1) {
  const float x = first ? w0 * (a.x * b.x) : w1 * fmaf(a.x, b.x, -(a.y * b.y));
  const float y = first ? w0 * (a.y * b.y) : w1 * fmaf(a.x, b.y, a.y * b.x);
  return make_float4(x, y, w1 * fmaf(a.z, b.z, -(a.w * b.w)), w1 * fmaf(a.z, b.w, a.w * b.z));
}

// w conj(a) b for float4 i of two rows (DC and Nyquist are real: conj leaves them alone)
__device__ __forceinline__ float4 hole_cmul(float4 a, float4 b, bool first, float w0, float w1) {
  const float x = first ? w0 * (a.x * b.x) : w1 * fmaf(a.x, b.x, a.y * b.y);
  const float y = first ? w0 * (a.y * b.y) : w1 * fmaf(a.x, b.y, -(a.y * b.x));
  return make_float4(x, y, w1 * fmaf(a.z, b.z, a.w * b.w), w1 * fmaf(a.z, b.w, -(a.w * b.z)));
}

__device__ __forceinline__ float hole_dot(float4 p, float4 q, float acc) {
  return fmaf(p.w, q.w, fmaf(p.z, q.z, fmaf(p.y, q.y, fmaf(p.x, q.x, acc))));
}

// HolE: e = <w (h r), t> over the transformed rows; a lane owns whole float4s (d % 4 == 0).  q gets the squared norms of
// the three rows: U is orthogonal, so that is DistMult's L2 term of the raw rows.
struct HolERows {
  __device__ __forceinline__ static void partial(const float* __restrict__ codes, const float* __restrict__ rel, int d,
                                                 int s, int r, int o, int lane, float& e, float& q) {
    const float4* e1 = reinterpret_cast<const float4*>(codes + (size_t)s * d);
    const float4* rr = reinterpret_cast<const float4*>(rel + (size_t)r * d);
    const float4* e2 = reinterpret_cast<const float4*>(codes + (size_t)o * d);
    const int d4 = d >> 2;
    float w0, w1;
    hole_weights(d, w0, w1);
    for (int i = lane; i < d4; i += 32) {
      const float4 a = __ldg(e1 + i), b = __ldg(rr + i), c = __ldg(e2 + i);
      e = hole_dot(hole_mul(a, b, i == 0, w0, w1), c, e);
      q += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
      q += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
      q += c.x * c.x + c.y * c.y + c.z * c.z + c.w * c.w;
    }
  }
};
