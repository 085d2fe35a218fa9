// codes_prune_emu.cpp — checks code_prunes / code_prune_radius of cozo_b200/csrc/hnsw_codes.cuh on the CPU: the per-row
// test the pruned search runs instead of comparing code_lower_bound with the worst distance.  Rows and queries are those
// of codes_bound_emu.cpp (random and adversarial: constant rows, rows on the code grid, magnitudes from 1e-38 to 3e38,
// subnormals, NaN, +-inf, dims that are not a multiple of 4), and the two f32 distances are summed in the search kernel's
// order.  For every pair and every worst distance the beam could hold (around d and the bound, d's float neighbours, 0,
// +inf, NaN), code_prunes must not prune when d < worst.
// Usage: codes_prune_emu <trials> <seed>; prints EMU_OK and a summary line.
#include "cuda_emu.hpp"

#include <algorithm>
#include <random>
#include <vector>

#include "../../cozo_b200/csrc/hnsw_codes.cuh"

using namespace cozo;

// the kernel's f32 L2 distance over ld elements: lane l owns float4 idx = l + 32 i
static float kernel_dist(const std::vector<float>& q, const std::vector<float>& x, uint32_t ld) {
  float part[32];
  for (int l = 0; l < 32; ++l) {
    float a = 0.f;
    for (uint32_t idx = l; idx < ld / 4; idx += 32)
      for (int e = 0; e < 4; ++e) {
        const float d = q[idx * 4 + e] - x[idx * 4 + e];
        a = fmaf(d, d, a);
      }
    part[l] = a;
  }
  for (int o = 16; o > 0; o >>= 1) {
    float nx[32];
    for (int l = 0; l < 32; ++l) nx[l] = part[l] + part[l ^ o];
    std::copy(nx, nx + 32, part);
  }
  return part[0];
}

int main(int argc, char** argv) {
  const long trials = argc > 1 ? atol(argv[1]) : 20000;
  std::mt19937_64 rng(argc > 2 ? atoll(argv[2]) : 1);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  auto pick = [&](uint32_t n) { return (uint32_t)(rng() % n); };
  const uint32_t dims[] = {1, 3, 4, 5, 17, 31, 64, 127, 128, 129, 255, 383, 768, 1023, 1536, 2048};
  long checked = 0, pruned_rows = 0;
  for (long t = 0; t < trials; ++t) {
    const uint32_t dim = dims[pick(sizeof(dims) / sizeof(dims[0]))];
    const uint32_t ld = (dim + 3) / 4 * 4;
    std::vector<float> x(ld, 0.f), q(ld, 0.f);  // padding stays zero, as in the index and in load_query
    const uint32_t kind = pick(12);
    const double mag = std::pow(10.0, (double)pick(77) - 38.0);  // 1e-38 .. 1e38
    for (uint32_t j = 0; j < dim; ++j) {
      double v;
      switch (kind) {
        case 0: v = U(rng); break;                                    // the benchmark's U[0,1)
        case 1: v = 0.25; break;                                      // constant row
        case 2: v = (U(rng) - 0.5) * mag; break;                      // any magnitude
        case 3: v = (U(rng) - 0.5) * 1e-40; break;                    // subnormals
        case 4: v = (j & 1 ? 3.0e38 : -3.0e38) * U(rng); break;       // the range overflows f32
        case 5: v = j == dim / 2 ? 1e6 : U(rng) * 1e-3; break;        // one outlier
        case 6: {                                                    // on the code grid: err is ~0
          const float lo = (float)(U(rng) - 0.5), sc = (float)(U(rng) * 0.01);
          v = fmaf((float)pick(256), sc, lo);
          break;
        }
        case 7: v = std::round(U(rng) * 4.0); break;                  // few distinct values
        default: v = std::ldexp(U(rng) - 0.5, (int)pick(40) - 20); break;
      }
      x[j] = (float)v;
    }
    if (kind == 8 && dim > 1) x[pick(dim)] = NAN;
    if (kind == 9 && dim > 1) x[pick(dim)] = pick(2) ? INFINITY : -INFINITY;
    std::vector<uint8_t> row(code_row_bytes(ld), 0xA5);
    quantize_row(x.data(), ld, row.data());
    float hdr[4];
    std::memcpy(hdr, row.data(), 16);
    for (uint32_t j = ld; j < code_row_bytes(ld) - CODE_HDR; ++j)
      if (row[CODE_HDR + j] != 0) { printf("code padding not zeroed\n"); return 1; }
    std::vector<float> xt(ld);
    for (uint32_t j = 0; j < ld; ++j) xt[j] = code_value(row[CODE_HDR + j], hdr[0], hdr[1]);
    bool row_finite = true;
    for (uint32_t j = 0; j < ld; ++j) row_finite = row_finite && code_finite(x[j]);
    if (!row_finite && !(hdr[2] == INFINITY)) { printf("non-finite row without err = inf\n"); return 1; }
    for (int r = 0; r < 8; ++r) {
      const uint32_t qk = pick(8);
      for (uint32_t j = 0; j < dim; ++j) {
        double v;
        switch (qk) {
          case 0: v = x[j]; break;                                              // d = 0
          case 1: v = xt[j]; break;                                             // d~ = 0
          case 2: v = x[j] + (U(rng) - 0.5) * 1e-6 * (std::fabs(x[j]) + 1e-30); break;
          case 3: v = x[j] * (1.0 + (U(rng) - 0.5) * 1e-3); break;
          case 4: v = (U(rng) - 0.5) * mag; break;
          case 5: v = j == 0 ? NAN : U(rng); break;
          default: v = U(rng); break;
        }
        q[j] = (float)v;
      }
      const float d = kernel_dist(q, x, ld);
      const float dt = kernel_dist(q, xt, ld);
      const double lb = code_lower_bound(dt, hdr[2]);
      ++checked;
      if (std::isnan(d)) {  // `d < worst` is false for NaN anyway; still, no bound may come out of it
        if (lb > 0.0 && !std::isnan(dt)) { printf("bound %g on a NaN distance (dt %g)\n", lb, dt); return 1; }
        continue;
      }
      if (!(lb <= (double)d)) {
        printf("BOUND VIOLATED: dim %u kind %u qk %u d %.9g dt %.9g err %.9g lb %.17g\n", dim, kind, qk, d, dt, hdr[2], lb);
        return 1;
      }
      // code_prunes (the per-row test of the search) may prune only where d < worst is false, for any worst the beam
      // can hold: around d and the bound, exact neighbours of d, 0, +inf and NaN
      const float worsts[] = {d, nextafterf(d, INFINITY), nextafterf(d, -INFINITY), (float)lb, nextafterf((float)lb, INFINITY),
                              (float)(lb * (1.0 + (U(rng) - 0.5) * 1e-4)), d * (float)U(rng), d * (float)(1.0 + U(rng)), 0.f,
                              INFINITY, NAN};
      for (const float worst : worsts) {
        const bool prunes = code_prunes(dt, hdr[2], code_prune_radius(worst));
        if (prunes && d < worst) {
          printf("PRUNE VIOLATED: dim %u kind %u qk %u d %.9g dt %.9g err %.9g worst %.9g\n", dim, kind, qk, d, dt, hdr[2], worst);
          return 1;
        }
        pruned_rows += prunes;
      }
    }
  }
  printf("checked %ld pairs, %ld (pair, worst) prunes\n", checked, pruned_rows);
  if (pruned_rows == 0) {  // the test must be able to prune at all
    printf("nothing pruned\n");
    return 1;
  }
  printf("EMU_OK\n");
  return 0;
}
