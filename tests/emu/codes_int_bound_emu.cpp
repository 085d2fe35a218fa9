// codes_int_bound_emu.cpp — checks the integer form of the code-row bound of cozo_b200/csrc/hnsw_codes.cuh on the CPU:
// code_query_prepare (the fixed-point query), the exact product S = sum a_j c_j, and code_int_prunes / code_int_radius,
// which the pruned search runs per row.  Rows are those of codes_prune_emu.cpp (random and adversarial: constant rows,
// rows on the code grid, magnitudes from 1e-38 to 3e38, subnormals, NaN, +-inf, dims that are not a multiple of 4, up to
// 2048); queries add NaN and +-inf elements and huge offsets.  The f32 distance d is summed in the search kernel's order.
// For every pair and every worst distance the beam could hold (around d and the bound, d's float neighbours, 0, +inf,
// NaN), code_int_prunes must not prune when d < worst.  The sums of the kernel's int32 products (per lane and in its
// shuffle tree) must stay inside int32, and on U[0,1) data the integer test must prune about as often as code_prunes.
// Usage: codes_int_bound_emu <trials> <seed>; prints EMU_OK and a summary line.
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

// S in the kernel's order (lane-strided code words, then the xor-shuffle tree), in int64 so that any partial outside
// int32 is seen; returns false if one is
static bool kernel_dot(const std::vector<int32_t>& a, const uint8_t* c, uint32_t ld, int64_t& S) {
  int64_t part[32];
  bool ok = true;
  for (int l = 0; l < 32; ++l) {
    int64_t s = 0;
    for (uint32_t idx = l; idx < ld / 4; idx += 32)
      for (int e = 0; e < 4; ++e) {
        s += (int64_t)a[idx * 4 + e] * c[idx * 4 + e];
        ok = ok && s >= INT32_MIN && s <= INT32_MAX;
      }
    part[l] = s;
  }
  for (int o = 16; o > 0; o >>= 1) {
    int64_t nx[32];
    for (int l = 0; l < 32; ++l) {
      nx[l] = part[l] + part[l ^ o];
      ok = ok && nx[l] >= INT32_MIN && nx[l] <= INT32_MAX;
    }
    std::copy(nx, nx + 32, part);
  }
  S = part[0];
  return ok;
}

int main(int argc, char** argv) {
  const long trials = argc > 1 ? atol(argv[1]) : 20000;
  std::mt19937_64 rng(argc > 2 ? atoll(argv[2]) : 1);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  auto pick = [&](uint32_t n) { return (uint32_t)(rng() % n); };
  const uint32_t dims[] = {1, 3, 4, 5, 17, 31, 64, 127, 128, 129, 255, 383, 514, 768, 1023, 1536, 2045, 2048};
  long checked = 0, pruned_rows = 0, u_old = 0, u_new = 0;
  for (long t = 0; t < trials; ++t) {
    const uint32_t dim = dims[pick(sizeof(dims) / sizeof(dims[0]))];
    const uint32_t ld = (dim + 3) / 4 * 4;
    std::vector<float> x(ld, 0.f), q(ld, 0.f);  // padding stays zero, as in the index and in load_query
    const uint32_t kind = pick(13);
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
        case 10: v = 1000.0 + U(rng); break;                          // an offset that dwarfs the spread
        case 11: v = (j & 1 ? 1.8e19 : -1.8e19) * U(rng); break;      // ||x^||^2 overflows f32
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
    const uint8_t* c = row.data() + CODE_HDR;
    std::vector<float> xt(ld);
    for (uint32_t j = 0; j < ld; ++j) xt[j] = code_value(c[j], hdr[0], hdr[1]);
    bool row_finite = true;
    for (uint32_t j = 0; j < ld; ++j) row_finite = row_finite && code_finite(x[j]);
    if (!row_finite && !(hdr[2] == INFINITY)) { printf("non-finite row without err = inf\n"); return 1; }
    if (!(hdr[3] >= 0.f && hdr[3] <= 3.40282347e38f)) { printf("X2 %g is not a finite f32 >= 0\n", hdr[3]); return 1; }
    for (int r = 0; r < 8; ++r) {
      const uint32_t qk = pick(11);
      const double off = qk == 8 ? std::pow(10.0, (double)pick(30)) : 0.0;
      for (uint32_t j = 0; j < dim; ++j) {
        double v;
        switch (qk) {
          case 0: v = x[j]; break;                                              // d = 0
          case 1: v = xt[j]; break;                                             // d~ = 0
          case 2: v = x[j] + (U(rng) - 0.5) * 1e-6 * (std::fabs(x[j]) + 1e-30); break;
          case 3: v = x[j] * (1.0 + (U(rng) - 0.5) * 1e-3); break;
          case 4: v = (U(rng) - 0.5) * mag; break;
          case 5: v = j == 0 ? NAN : U(rng); break;
          case 6: v = j == dim - 1 ? (pick(2) ? INFINITY : -INFINITY) : U(rng); break;
          case 7: v = x[j] + 1e4; break;                                        // a huge offset from the row
          case 8: v = off + U(rng); break;                                      // an offset of 1 .. 1e29
          default: v = U(rng); break;
        }
        q[j] = (float)v;
      }
      std::vector<int32_t> a(ld);
      const CodeQuery cq = code_query_prepare(q.data(), ld, a.data());
      const int32_t A = code_query_amax(ld);
      for (uint32_t j = 0; j < ld; ++j)
        if (a[j] < -A || a[j] > A || (j >= dim && a[j] != 0)) { printf("level %d out of range at %u\n", a[j], j); return 1; }
      int64_t S64;
      if (!kernel_dot(a, c, ld, S64)) { printf("int32 overflow: dim %u kind %u qk %u\n", dim, kind, qk); return 1; }
      const int32_t S = (int32_t)S64;
      bool q_finite = true;
      for (uint32_t j = 0; j < ld; ++j) q_finite = q_finite && code_finite(q[j]);
      if (!q_finite && !(cq.eq == INFINITY)) { printf("non-finite query without e_q = inf\n"); return 1; }
      const float d = kernel_dist(q, x, ld);
      const float dt = kernel_dist(q, xt, ld);
      const double lb = code_lower_bound(dt, hdr[2]);
      ++checked;
      const float worsts[] = {d, nextafterf(d, INFINITY), nextafterf(d, -INFINITY), (float)lb, nextafterf((float)lb, INFINITY),
                              (float)(lb * (1.0 + (U(rng) - 0.5) * 1e-4)), d * (float)U(rng), d * (float)(1.0 + U(rng)), 0.f,
                              1e-36f, INFINITY, NAN};
      for (const float worst : worsts) {
        const bool prunes = code_int_prunes(cq, S, hdr, code_int_radius(cq, worst));
        if (prunes && (std::isnan(d) || d < worst)) {
          printf("PRUNE VIOLATED: dim %u kind %u qk %u d %.9g worst %.9g err %.9g e_q %.9g X2 %.9g S %d\n", dim, kind, qk,
                 d, worst, hdr[2], cq.eq, hdr[3], S);
          return 1;
        }
        pruned_rows += prunes;
        if (kind == 0 && qk >= 9) {
          u_old += code_prunes(dt, hdr[2], code_prune_radius(worst));
          u_new += prunes;
        }
      }
    }
  }
  printf("checked %ld pairs, %ld (pair, worst) prunes; U[0,1) rows vs U[0,1) queries: %ld prunes (f32 test: %ld)\n",
         checked, pruned_rows, u_new, u_old);
  if (pruned_rows == 0) {  // the test must be able to prune at all
    printf("nothing pruned\n");
    return 1;
  }
  if (u_new < 0.97 * u_old) {  // and about as often as the f32 test where the benchmark runs
    printf("integer test prunes too rarely on U[0,1) data\n");
    return 1;
  }
  printf("EMU_OK\n");
  return 0;
}
