// hnsw_codes.cuh — the compact uint8 copy of an index's f32 vectors and the exact lower bound on the L2 distance that
// lets the search reject a neighbour without fetching its f32 row.
//
// Layout: one code row per vector, code_row_bytes(ld) = 16 + round_up(ld, 16) bytes, so that a row is one
// cp.async.bulk (16-byte aligned, a multiple of 16 bytes long):
//   float lo, scale, err, 0      the row header
//   uint8 c[ld]                  one code per element of the f32 row, padding elements included; zero padded
// Element j dequantises to  x~_j = fmaf((float)c_j, scale, lo)  (code_value), which is exactly what the search
// computes.  err >= ||x - x~||_2 over all ld elements, computed in f64 from those very f32 values and rounded up;
// a row holding NaN or +-inf (or whose range overflows f32) gets err = +inf and is never pruned.
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

// Affine per-row quantisation of x[0..ld) into `out` (code_row_bytes(ld) bytes).
__host__ __device__ inline void quantize_row(const float* x, uint32_t ld, uint8_t* out) {
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
  double ss = 0.0;
  for (uint32_t j = 0; j < ld; ++j) {
    uint32_t cj = 0;
    if (scale > 0.f) {
      const float t = rintf((x[j] - lo) / scale);
      cj = t > 0.f ? (t < 255.f ? (uint32_t)t : 255u) : 0u;
    }
    c[j] = (uint8_t)cj;
    const double e = (double)x[j] - (double)code_value(cj, lo, scale);
    ss += e * e;
  }
  for (uint32_t j = ld; j < code_row_bytes(ld) - CODE_HDR; ++j) c[j] = 0;
  // ss carries at most (2 ld + 2) f64 roundings, far below the 2^-30 the two factors add
  float err = INFINITY;
  if (finite) {
    const double e = sqrt(ss * (1.0 + 0x1p-30)) * (1.0 + 0x1p-30);
    err = (float)e;
    if ((double)err < e) err = nextafterf(err, INFINITY);
  }
  float* hdr = reinterpret_cast<float*>(out);
  hdr[0] = lo;
  hdr[1] = scale;
  hdr[2] = err;
  hdr[3] = 0.f;
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

// Fills the code rows of vectors ids[i] (ids == nullptr: first + i) for i < count.  One thread per row: this runs
// once per write of the vectors, not per search.
static __global__ void quantize_rows_kernel(const float* vec, uint32_t ld, uint8_t* codes, const uint32_t* ids,
                                            uint32_t first, uint32_t count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const size_t r = ids ? ids[i] : first + i;
  quantize_row(vec + r * ld, ld, codes + r * code_row_bytes(ld));
}

}  // namespace cozo
