// hnsw_codes.cuh — the compact uint8 copy of an index's f32 vectors and the exact bounds on the search kernel's distance
// (L2, Cosine and IP) that let the search reject a neighbour without fetching its f32 row.
//
// Layout: one code row per vector, code_row_bytes(ld) = 16 + round_up(ld, 16) bytes, so that a row is one
// cp.async.bulk (16-byte aligned, a multiple of 16 bytes long):
//   float lo, scale, err, X      the row header; X is X2 on an L2 index and Xn on a Cosine or IP index
//   uint8 c[ld]                  one code per element of the f32 row, padding elements included; zero padded
// Element j dequantises to  x~_j = fmaf((float)c_j, scale, lo)  (code_value), and in exact arithmetic to
// x^_j = lo + scale c_j.  err >= ||x - x~||_2 and err >= ||x - x^||_2 over all ld elements, computed in f64 and rounded
// up.  L2: X2 <= ||x^||^2, computed in f64 and rounded down.  Cosine and IP: Xn >= ||x||_2, computed in f64 and rounded
// up, so that ||x|| lies in [Xn (1 - 2^-22), Xn].  A row holding NaN or +-inf (or whose range or X2 overflows f32) gets
// err = +inf and is never pruned; so does a Cosine or IP row with Xn outside [CODE_XN_MIN, CODE_XN_MAX] (a zero row
// among them).
#pragma once
#include <math.h>

#include "common.cuh"

namespace cozo {

constexpr uint32_t CODE_HDR = 16;
// Only rows of at least this many elements get codes.  Pruning trades a second, dependent fetch per hop for fewer
// bytes: at D = 768 (3 KB rows) a step is 1.5x faster, at D = 128 (512 B rows, latency-bound) it was 13 % slower
// (one H100, bench.py config 2 and --dim 128); dims in between are not measured.  Overridable so that the CPU emulator
// of the library can run the pruned search at small dimensions.
#ifndef CODES_MIN_LD
#define CODES_MIN_LD 512u
#endif

__host__ __device__ inline uint32_t code_row_bytes(uint32_t ld) { return CODE_HDR + (ld + 15) / 16 * 16; }

__host__ __device__ inline float code_value(uint32_t c, float lo, float scale) { return fmaf((float)c, scale, lo); }

__host__ __device__ inline bool code_finite(float v) { return fabsf(v) <= 3.40282347e38f; }

// The range of Xn inside which a Cosine or IP row can be pruned (code_dot_prunes): below it the kernel's f32 sum of
// squares could lose more than REL to underflow, above it the f32 dot product with a query of norm <= CODE_XN_MAX could
// overflow (both norms <= 2^63 keep every partial sum below 2^127).
constexpr double CODE_XN_MIN = 0x1p-40, CODE_XN_MAX = 0x1p63;

// Affine per-row quantisation of x[0..ld) into `out` (code_row_bytes(ld) bytes), with the header word 3 of `metric`.
__host__ __device__ inline void quantize_row(const float* x, uint32_t ld, uint8_t* out, int metric = COZO_GPU_L2) {
  bool finite = true;
  float lo = x[0], hi = x[0];
  for (uint32_t j = 0; j < ld; ++j) {
    const float v = x[j];
    finite = finite && code_finite(v);
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  float scale = finite ? (hi - lo) / 255.f : 0.f;
  if (!code_finite(scale)) finite = false;
  if (!finite) lo = scale = 0.f;
  uint8_t* c = out + CODE_HDR;
  double ss = 0.0, x2 = 0.0, n2 = 0.0;
  for (uint32_t j = 0; j < ld; ++j) {
    uint32_t cj = 0;
    if (scale > 0.f) {
      const float t = rintf((x[j] - lo) / scale);
      cj = t > 0.f ? (t < 255.f ? (uint32_t)t : 255u) : 0u;
    }
    c[j] = (uint8_t)cj;
    // |x - x^| <= |x - x~| + |x~ - x^|, and x~ - x^ is the rounding of one fmaf: at most half an ulp of x~, which is
    // <= 2^-24 |x~| + 2^-150; none when c = 0 (x~ = x^ = lo)
    const float xt = code_value(cj, lo, scale);
    const double e = fabs((double)x[j] - (double)xt) + (cj ? fabs((double)xt) * 0x1p-24 + 0x1p-150 : 0.0);
    ss += e * e;
    const double xe = fma((double)scale, (double)cj, (double)lo);
    x2 += xe * xe;
    n2 += (double)x[j] * (double)x[j];  // exact products
  }
  for (uint32_t j = ld; j < code_row_bytes(ld) - CODE_HDR; ++j) c[j] = 0;
  // ss and x2 are sums of non-negative terms and carry at most (2 ld + 6) f64 roundings, far below the 2^-30 the
  // factors add
  float err = INFINITY, X2 = 0.f;
  if (finite) {
    const double e = sqrt(ss * (1.0 + 0x1p-30)) * (1.0 + 0x1p-30);
    err = (float)e;
    if ((double)err < e) err = nextafterf(err, INFINITY);
    const double xl = x2 * (1.0 - 0x1p-30);
    X2 = (float)xl;
    if ((double)X2 > xl) X2 = nextafterf(X2, 0.f);
    if (!code_finite(X2)) {
      err = INFINITY;
      X2 = 0.f;
    }
    if (metric != COZO_GPU_L2) {  // X2 is replaced by Xn
      const double xn = sqrt(n2 * (1.0 + 0x1p-30)) * (1.0 + 0x1p-30);
      X2 = (float)xn;
      if ((double)X2 < xn) X2 = nextafterf(X2, INFINITY);
      if (!((double)X2 >= CODE_XN_MIN && (double)X2 <= CODE_XN_MAX)) {
        err = INFINITY;
        X2 = 0.f;
      }
    }
  }
  float* hdr = reinterpret_cast<float*>(out);
  hdr[0] = lo;
  hdr[1] = scale;
  hdr[2] = err;
  hdr[3] = X2;
}

// Lower bound on the search kernel's f32 L2 distance d(q, x), from dt = the kernel's f32 distance to the
// dequantised row x~ and the row's err.
//   Exact arithmetic: ||q - x|| >= ||q - x~|| - err (triangle inequality), so D >= max(0, sqrt(D~) - err)^2.
//   Rounding: d and dt are f32 sums of non-negative terms (ld/32 fmaf per lane, a 5-level shuffle tree, the rounded
//   difference counted twice), so each is within a factor (1 +- (ld/32 + 7) 2^-24) of its exact value D or D~, at
//   most 2^-17 relative for ld <= 2048.  REL = 2^-14 covers both sides with room to spare; the absolute 1e-36
//   covers subnormal underflow (< 2^-140 over the whole sum).  The f64 steps below round at 2^-53.
// A distance that is NaN or overflowed gives no bound (0).  Prune only when the bound is >= the beam's worst.
constexpr double CODE_REL = 0x1p-14;
__host__ __device__ inline double code_lower_bound(float dt, float err) {
  if (!(dt <= 3.40282347e38f)) return 0.0;
  const double s = sqrt((double)dt * (1.0 - CODE_REL)) - (double)err;
  if (!(s > 0.0)) return 0.0;
  return s * s * (1.0 - CODE_REL) - 1e-36;
}

// The same test without a square root per row: code_lower_bound(dt, err) >= worst  <=>  s >= W with
// W = sqrt((worst + 1e-36) / (1 - REL))  <=>  dt (1 - REL) >= (err + W)^2, all in exact arithmetic.  W depends only on the
// beam's worst distance, so the search computes it once per value of worst (code_prune_radius) and tests each row with
// code_prunes.  Rounding: the f64 steps here round at 2^-53, far inside the 2^-14 - 2^-17 margin that REL leaves over the
// f32 error of d and dt, so pruning still implies d >= worst.  A NaN or overflowed dt, err = +inf, or a NaN or +inf
// worst never prunes.
__host__ __device__ inline double code_prune_radius(float worst) { return sqrt(((double)worst + 1e-36) / (1.0 - CODE_REL)); }
__host__ __device__ inline bool code_prunes(float dt, float err, double W) {
  const double r = (double)err + W;
  return dt <= 3.40282347e38f && (double)dt * (1.0 - CODE_REL) >= r * r;
}

// ---- the integer form of the bound: what the search runs ------------------------------------------------------------
// The query is held in fixed point, q^_j = s_q a_j with integers |a_j| <= A = code_query_amax(ld), so that the exact
// integer S = sum_j a_j c_j fits in an int32 over the whole row (|S| <= A 255 ld < 2^31, and so does every partial sum).
// s_q is a power of two, the least one with max_j |q_j| <= A s_q, so q_j - s_q a_j is exact in f64.
// With e_q >= ||q - q^|| (per query) and err >= ||x - x^|| (per row), the triangle inequality twice gives
//   ||q - x|| >= ||q^ - x^|| - e_q - err,    ||q^ - x^||^2 = D^ = Q2 + ||x^||^2 - 2 s_q (lo sum_j a_j + scale S)
// with Q2 = s_q^2 sum_j a_j^2 (exact in f64).  The search evaluates D^ in f64 with the row's X2 <= ||x^||^2 in place of
// ||x^||^2 (only lowering it) and subtracts 2^-45 (Q2 + X2 + 2 s_q (|lo sum a| + |scale S|)), which covers the f64
// roundings of the expansion (under 2^-50 of that sum).  The result D^_lo <= D^ prunes iff D^_lo >= (err + e_q + W)^2
// with W = code_prune_radius(worst): then sqrt(D) >= W, and the REL argument of code_prunes gives d >= worst.  The f64
// roundings of err + e_q + W and of its square are relative to err, e_q and W, and the 2^-30 on err and e_q and the
// REL on W cover them.  Nothing prunes when D^_lo, err or e_q is NaN or +inf; a query holding NaN or +-inf has e_q = +inf.
// Tightness: X2 is rounded to f32, so on rows whose offset dwarfs their spread (|lo| >> scale) D^_lo falls short of D^
// by up to 2^-24 ||x^||^2 and those rows prune less often; the bound stays valid.
struct CodeQuery {
  double q2;     // ||q^||^2 = s_q^2 sum a_j^2
  double sq2;    // 2 s_q
  int32_t suma;  // sum a_j
  double eq;     // >= ||q - q^||; +inf: nothing is pruned
};

__host__ __device__ inline int32_t code_query_amax(uint32_t ld) {
  const uint32_t a = 2147483647u / (255u * (ld ? ld : 1u));
  return (int32_t)(a < 32767u ? a : 32767u);
}

// s_q for a query whose largest |q_j| is m (finite): the least power of two with m <= A s_q (1 if m = 0)
__host__ __device__ inline double code_query_scale(float m, int32_t A) {
  if (!(m > 0.f)) return 1.0;
  int e;
  frexp((double)m / (double)A, &e);  // m / A < 2^e, up to the rounding of the division, which the clamp below absorbs
  return ldexp(1.0, e);
}

// a_j for q_j (any value: the clamp keeps |a_j| <= A; a NaN maps to 0 and is caught by e_q)
__host__ __device__ inline int32_t code_query_level(float q, double sq, int32_t A) {
  const double t = rint((double)q / sq);
  if (t >= (double)A) return A;
  if (t <= -(double)A) return -A;
  return t == t ? (int32_t)t : 0;
}

// the square of q_j - s_q a_j (exact before squaring: both are multiples of min(ulp(q_j), s_q), within 2^25 of it)
__host__ __device__ inline double code_query_resid2(float q, double sq, int32_t a) {
  const double r = (double)q - sq * (double)a;
  return r * r;
}

// the per-query constants from sum a, sum a^2 (exact), sum of code_query_resid2 (ss) and whether every q_j is finite
__host__ __device__ inline CodeQuery code_query_finish(double sq, int32_t suma, double suma2, double ss, bool finite) {
  CodeQuery c;
  c.q2 = sq * sq * suma2;
  c.sq2 = 2.0 * sq;
  c.suma = suma;
  // ss carries at most (2 ld) f64 roundings, far below the 2^-30 the two factors add
  c.eq = finite ? sqrt(ss * (1.0 + 0x1p-30)) * (1.0 + 0x1p-30) : INFINITY;
  if (!(c.eq <= 1.7976931348623157e308)) c.eq = INFINITY;
  return c;
}

// The reference form of the preparation (the search does the same per lane and sums across the warp): a[0..ld) and the
// constants for the query q[0..ld).
__host__ __device__ inline CodeQuery code_query_prepare(const float* q, uint32_t ld, int32_t* a) {
  float m = 0.f;
  bool finite = true;
  for (uint32_t j = 0; j < ld; ++j) {
    finite = finite && code_finite(q[j]);
    m = fmaxf(m, fabsf(q[j]));
  }
  const int32_t A = code_query_amax(ld);
  const double sq = code_query_scale(finite ? m : 0.f, A);
  int32_t suma = 0;
  double suma2 = 0.0, ss = 0.0;
  for (uint32_t j = 0; j < ld; ++j) {
    a[j] = code_query_level(q[j], sq, A);
    suma += a[j];
    suma2 += (double)a[j] * (double)a[j];
    ss += code_query_resid2(q[j], sq, a[j]);
  }
  return code_query_finish(sq, suma, suma2, ss, finite);
}

// The radius the integer test compares with: e_q + W, once per value of the beam's worst distance.
__host__ __device__ inline double code_int_radius(const CodeQuery& cq, float worst) { return cq.eq + code_prune_radius(worst); }

// Whether the row with header hdr = {lo, scale, err, X2} and S = sum a_j c_j can be dropped; WE = code_int_radius.
__host__ __device__ inline bool code_int_prunes(const CodeQuery& cq, int32_t S, const float* hdr, double WE) {
  const double x = (double)hdr[0] * (double)cq.suma, y = (double)hdr[1] * (double)S, X2 = (double)hdr[3];
  const double dlo = (cq.q2 + X2) - cq.sq2 * (x + y) - 0x1p-45 * (cq.q2 + X2 + cq.sq2 * (fabs(x) + fabs(y)));
  const double r = (double)hdr[2] + WE;
  return dlo <= 1.7976931348623157e308 && dlo >= r * r;
}

// ---- the bound for Cosine and IP: an upper bound on the kernel's f32 dot product ---------------------------------------
// What the kernel computes (finish<METRIC>, hnsw_device.cuh): a = the f32 dot product q.x (lane-strided fmaf chains over
// all ld elements, then the shuffle tree), b = the f32 sum of x_j^2 in the same order, qnorm = load_query's f32 sum of
// q_j^2, and then  IP: d = (float)(1 - (double)a),  Cosine: d = (float)(1 - (double)a / sqrt((double)qnorm (double)b)).
// Both are non-increasing in a.  The test proves d >= worst from an upper bound U >= a:
//   Exact arithmetic: q.x = q^.x^ + (q - q^).x + q^.(x - x^), with q^.x^ = s_q (lo sum_j a_j + scale S) (CodeQuery) exact,
//   |(q - q^).x| <= e_q ||x|| <= e_q Xn  and  |q^.(x - x^)| <= ||q^|| err,  ||q^|| = sqrt(Q2) (Q2 exact in f64).
//   Rounding of a: a sum of ld/32 + 5 roundings per term, so |a - q.x| <= (ld/32 + 7) 2^-24 sum_j |q_j x_j| <=
//   REL ||q|| ||x|| <= REL (||q^|| + e_q) Xn for ld <= 2048 (the L2 argument), plus 1e-36 for subnormal underflow.  The
//   norms are at most CODE_XN_MAX = 2^63 (the row's by quantize_row, the query's by code_dot_query), so no partial sum
//   overflows.  So
//     U = s_q (lo sum a + scale S) + Xn (e_q + REL (||q^|| + e_q)) + ||q^|| err + 1e-36 >= a.
//   The f64 evaluation of U takes under 16 roundings, each at most 2^-53 of M = |lo s_q sum a| + |s_q scale S| +
//   Xn (e_q + ...) + ||q^|| err + 1e-36; adding 2^-45 M covers them.
// IP: a <= U <= T = 1 - worst exactly  =>  1 - (double)a >= worst (rounding is monotone and worst is a float)  =>
//   d >= worst.  T is taken as the f64 1 - worst lowered by 2^-50 of itself (the subtraction rounds at 2^-53).
// Cosine: with the kernel's qnorm known, s = sqrt(qnorm b) rounds once (qnorm b is exact in f64), and so does a / s.
//   b is within REL of ||x||^2 (a sum of non-negative terms; Xn >= CODE_XN_MIN keeps underflow below 2^-61 of it), and
//   ||x|| is in [Xn (1 - 2^-22), Xn], so  sqrt(qnorm) Xn (1 - 2^-13) <= s (1 -+ 2^-53) <= sqrt(qnorm) Xn (1 + 2^-13)
//   with room to spare.  If U >= 0: a / s <= U / s_min, and the rounded quotient is at most (1 + 2^-53) of that, so
//   U <= T sqrt(qnorm) Xn (1 - 2^-13) suffices.  If U < 0: a / s <= U / s_max and the rounded quotient is at most
//   (1 - 2^-53) of that, so U <= T sqrt(qnorm) Xn (1 + 2^-13) suffices.  Then (double)a / s <= T, and as for IP
//   d >= worst.  The f64 steps from worst to T sqrt(qnorm) Xn (1 -+ 2^-13) round 6 times, far inside the margin that
//   2^-13 leaves over REL + 2^-22.
//   |a / s| lies in [2^-275, 2^277] unless a = 0, so the quotient neither underflows nor overflows.
// Nothing prunes when: err = +inf (non-finite rows, rows outside the Xn range, zero rows), e_q = +inf (non-finite
// queries), the query's norm bound exceeds CODE_XN_MAX, Cosine with qnorm = 0 (or NaN), worst NaN or +-inf, or U NaN.
// Tightness: the Cauchy-Schwarz term ||q^|| err is larger than the L2 bound's error term on most data.
constexpr double CODE_COS_LO = 1.0 - 0x1p-13, CODE_COS_HI = 1.0 + 0x1p-13;

struct CodeDotQuery {
  double sq;   // s_q
  double ssa;  // s_q sum a_j (exact: s_q is a power of two)
  double qn;   // ||q^|| = sqrt(Q2)
  double k1;  // e_q + REL (||q^|| + e_q): the factor of Xn in U
  double rq;  // IP: 1; Cosine: sqrt(qnorm); NaN: nothing is pruned for this query
};

// the per-query constants of code_dot_prunes, from the fixed-point query and the kernel's f32 qnorm
template <int METRIC>
__host__ __device__ inline CodeDotQuery code_dot_query(const CodeQuery& cq, float qnorm) {
  CodeDotQuery d;
  d.sq = 0.5 * cq.sq2;
  d.ssa = d.sq * (double)cq.suma;
  d.qn = sqrt(cq.q2);
  d.k1 = cq.eq + CODE_REL * (d.qn + cq.eq);
  const bool ok = d.qn + cq.eq <= CODE_XN_MAX && (METRIC == COZO_GPU_IP || qnorm > 0.f);
  d.rq = !ok ? (double)NAN : METRIC == COZO_GPU_IP ? 1.0 : sqrt((double)qnorm);
  return d;
}

// what U is compared with, once per value of the beam's worst distance: T = 1 - worst (lowered), times rq
__host__ __device__ inline double code_dot_radius(const CodeDotQuery& cd, float worst) {
  if (!code_finite(worst)) return NAN;
  const double t = 1.0 - (double)worst;
  return (t - fabs(t) * 0x1p-50) * cd.rq;
}

// Whether the row with header hdr = {lo, scale, err, Xn} and S = sum a_j c_j can be dropped; R = code_dot_radius.
template <int METRIC>
__host__ __device__ inline bool code_dot_prunes(const CodeDotQuery& cd, int32_t S, const float* hdr, double R) {
  const double x = (double)hdr[0] * cd.ssa, y = cd.sq * ((double)hdr[1] * (double)S), xn = (double)hdr[3];
  const double e = xn * cd.k1 + cd.qn * (double)hdr[2] + 1e-36;
  const double u = (x + y) + e + 0x1p-45 * (fabs(x) + fabs(y) + e);
  if (METRIC == COZO_GPU_IP) return u <= R;
  return u <= R * xn * (u >= 0.0 ? CODE_COS_LO : CODE_COS_HI);
}

// Fills the code rows of vectors ids[i] (ids == nullptr: first + i) for i < count.  One thread per row: this runs
// once per write of the vectors, not per search.
static __global__ void quantize_rows_kernel(const float* vec, uint32_t ld, uint8_t* codes, const uint32_t* ids,
                                            uint32_t first, uint32_t count, int metric) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const size_t r = ids ? ids[i] : first + i;
  quantize_row(vec + r * ld, ld, codes + r * code_row_bytes(ld), metric);
}

}  // namespace cozo
