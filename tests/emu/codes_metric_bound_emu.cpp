// codes_metric_bound_emu.cpp — checks the Cosine and IP code-row bound of cozo_b200/csrc/hnsw_codes.cuh on the CPU:
// quantize_row with the metric's header (Xn), code_dot_query, code_dot_radius and code_dot_prunes, which the pruned
// search runs per row.  Rows are random and adversarial (those of codes_int_bound_emu.cpp: magnitudes from 1e-38 to 3e38,
// subnormals, NaN, +-inf, overflowing ranges, large offsets; plus normalised Gaussian rows, mixed-sign rows and zero
// rows); queries add NaN and +-inf elements, zero queries, opposite and normalised Gaussian ones.  The kernel's f32 dot
// product, sum of squares and query norm are summed in its lane order and finished as finish<METRIC> does.  For every
// pair, both metrics, and every worst distance around d, around the largest worst the test still prunes at, and the
// special values (0, 1, +-FLT_MAX, +-inf, NaN), a prune must imply d >= worst (d not NaN); rows with err = +inf, queries
// with e_q = +inf and Cosine queries with qnorm = 0 must never prune.  Then on U[0,1) and normalised Gaussian data at
// D = 768 the share of rows at least as far as the median distance that the test rejects is printed and must reach
// a floor.
// Usage: codes_metric_bound_emu <trials> <seed>; prints EMU_OK and the rates.
#include "cuda_emu.hpp"

#include <algorithm>
#include <random>
#include <vector>

#include "../../cozo_b200/csrc/hnsw_codes.cuh"

using namespace cozo;

// sum over the ld elements in the kernel's order: lane l owns float4 idx = l + 32 i, fmaf chains, then the xor tree
template <class F>
static float lane_sum(uint32_t ld, F term) {
  float part[32];
  for (int l = 0; l < 32; ++l) {
    float a = 0.f;
    for (uint32_t idx = l; idx < ld / 4; idx += 32)
      for (int e = 0; e < 4; ++e) a = term(idx * 4 + e, a);
    part[l] = a;
  }
  for (int o = 16; o > 0; o >>= 1) {
    float nx[32];
    for (int l = 0; l < 32; ++l) nx[l] = part[l] + part[l ^ o];
    std::copy(nx, nx + 32, part);
  }
  return part[0];
}

struct Sums {
  float a, b, qnorm;
};
static Sums kernel_sums(const std::vector<float>& q, const std::vector<float>& x, uint32_t ld) {
  Sums s;
  s.a = lane_sum(ld, [&](uint32_t j, float acc) { return fmaf(q[j], x[j], acc); });
  s.b = lane_sum(ld, [&](uint32_t j, float acc) { return fmaf(x[j], x[j], acc); });
  s.qnorm = lane_sum(ld, [&](uint32_t j, float acc) { return fmaf(q[j], q[j], acc); });
  return s;
}

// finish<METRIC> of hnsw_device.cuh
static float kernel_dist(int metric, const Sums& s) {
  if (metric == COZO_GPU_IP) return (float)(1.0 - (double)s.a);
  return (float)(1.0 - (double)s.a / sqrt((double)s.qnorm * (double)s.b));
}

static int64_t kernel_dot(const std::vector<int32_t>& a, const uint8_t* c, uint32_t ld) {
  int64_t S = 0;
  for (uint32_t j = 0; j < ld; ++j) S += (int64_t)a[j] * c[j];
  return S;  // exact; codes_int_bound_emu.cpp checks that the kernel's int32 partials do not overflow
}

struct Pair {
  std::vector<uint8_t> row;
  CodeQuery cq;
  int32_t S;
  Sums s;
};

static bool prunes(int metric, const Pair& p, const CodeDotQuery& cd, float worst) {
  const float* hdr = reinterpret_cast<const float*>(p.row.data());
  const double R = code_dot_radius(cd, worst);
  return metric == COZO_GPU_IP ? code_dot_prunes<COZO_GPU_IP>(cd, p.S, hdr, R)
                               : code_dot_prunes<COZO_GPU_COSINE>(cd, p.S, hdr, R);
}

static CodeDotQuery dot_query(int metric, const CodeQuery& cq, float qnorm) {
  return metric == COZO_GPU_IP ? code_dot_query<COZO_GPU_IP>(cq, qnorm) : code_dot_query<COZO_GPU_COSINE>(cq, qnorm);
}

// floats in their numeric order as unsigned keys, and back
static uint32_t fkey(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}
static float fval(uint32_t k) {
  const uint32_t u = (k & 0x80000000u) ? k & 0x7FFFFFFFu : ~k;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

// the largest finite worst at which the row still prunes (NaN if none): the test is monotone in worst
static float prune_threshold(int metric, const Pair& p, const CodeDotQuery& cd) {
  uint32_t lo = fkey(-3.40282347e38f), hi = fkey(3.40282347e38f);
  if (!prunes(metric, p, cd, fval(lo))) return NAN;
  if (prunes(metric, p, cd, fval(hi))) return fval(hi);
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    (prunes(metric, p, cd, fval(mid)) ? lo : hi) = mid;
  }
  return fval(lo);
}

static Pair make_pair(const std::vector<float>& q, const std::vector<float>& x, uint32_t ld, int metric) {
  Pair p;
  p.row.assign(code_row_bytes(ld), 0xA5);
  quantize_row(x.data(), ld, p.row.data(), metric);
  std::vector<int32_t> a(ld);
  p.cq = code_query_prepare(q.data(), ld, a.data());
  p.S = (int32_t)kernel_dot(a, p.row.data() + CODE_HDR, ld);
  p.s = kernel_sums(q, x, ld);
  return p;
}

int main(int argc, char** argv) {
  const long trials = argc > 1 ? atol(argv[1]) : 20000;
  std::mt19937_64 rng(argc > 2 ? atoll(argv[2]) : 1);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  std::normal_distribution<double> N(0.0, 1.0);
  auto pick = [&](uint32_t n) { return (uint32_t)(rng() % n); };
  auto gaussian_unit = [&](std::vector<float>& v, uint32_t dim) {
    double n2 = 0.0;
    std::vector<double> g(dim);
    for (uint32_t j = 0; j < dim; ++j) {
      g[j] = N(rng);
      n2 += g[j] * g[j];
    }
    for (uint32_t j = 0; j < dim; ++j) v[j] = (float)(g[j] / std::sqrt(n2));
  };
  const uint32_t dims[] = {1, 3, 4, 5, 17, 31, 64, 127, 128, 129, 255, 383, 514, 768, 1023, 1536, 2045, 2048};
  const int metrics[] = {COZO_GPU_IP, COZO_GPU_COSINE};
  long checked = 0, pruned = 0;
  for (long t = 0; t < trials; ++t) {
    const uint32_t dim = dims[pick(sizeof(dims) / sizeof(dims[0]))];
    const uint32_t ld = (dim + 3) / 4 * 4;
    std::vector<float> x(ld, 0.f), q(ld, 0.f);  // padding stays zero, as in the index and in load_query
    const uint32_t kind = pick(16);
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
        case 11: v = (j & 1 ? 1.8e19 : -1.8e19) * U(rng); break;      // ||x|| beyond the Xn range
        case 13: v = (U(rng) - 0.5) * std::ldexp(1.0, (int)pick(20) - 10); break;  // mixed sign
        case 14: v = 0.0; break;                                      // zero row
        default: v = std::ldexp(U(rng) - 0.5, (int)pick(40) - 20); break;
      }
      x[j] = (float)v;
    }
    if (kind == 12) gaussian_unit(x, dim);  // normalised Gaussian
    if (kind == 8 && dim > 1) x[pick(dim)] = NAN;
    if (kind == 9 && dim > 1) x[pick(dim)] = pick(2) ? INFINITY : -INFINITY;
    std::vector<float> xt(ld);
    {
      std::vector<uint8_t> row(code_row_bytes(ld));
      quantize_row(x.data(), ld, row.data(), COZO_GPU_IP);
      float hdr[4];
      std::memcpy(hdr, row.data(), 16);
      for (uint32_t j = 0; j < ld; ++j) xt[j] = code_value(row[CODE_HDR + j], hdr[0], hdr[1]);
      double n2 = 0.0;
      bool finite = true;
      for (uint32_t j = 0; j < ld; ++j) {
        n2 += (double)x[j] * (double)x[j];
        finite = finite && code_finite(x[j]);
      }
      if (!finite && !(hdr[2] == INFINITY)) { printf("non-finite row without err = inf\n"); return 1; }
      if (hdr[2] != INFINITY && !((double)hdr[3] >= std::sqrt(n2) && (double)hdr[3] <= std::sqrt(n2) * (1.0 + 0x1p-22))) {
        printf("Xn %.9g is not a tight upper bound of ||x|| = %.17g\n", hdr[3], std::sqrt(n2));
        return 1;
      }
      std::vector<uint8_t> l2a(code_row_bytes(ld)), l2b(code_row_bytes(ld));  // L2 rows: the metric changes nothing
      quantize_row(x.data(), ld, l2a.data());
      quantize_row(x.data(), ld, l2b.data(), COZO_GPU_L2);
      if (l2a != l2b || std::memcmp(l2a.data(), row.data(), 8) || std::memcmp(l2a.data() + 16, row.data() + 16, ld)) {
        printf("the metric changed lo, scale or the codes\n");
        return 1;
      }
    }
    for (int r = 0; r < 8; ++r) {
      const uint32_t qk = pick(14);
      const double off = qk == 8 ? std::pow(10.0, (double)pick(30)) : 0.0;
      for (uint32_t j = 0; j < dim; ++j) {
        double v;
        switch (qk) {
          case 0: v = x[j]; break;                                              // cos = 1
          case 1: v = xt[j]; break;
          case 2: v = x[j] + (U(rng) - 0.5) * 1e-6 * (std::fabs(x[j]) + 1e-30); break;
          case 3: v = x[j] * (1.0 + (U(rng) - 0.5) * 1e-3); break;
          case 4: v = (U(rng) - 0.5) * mag; break;
          case 5: v = j == 0 ? NAN : U(rng); break;
          case 6: v = j == dim - 1 ? (pick(2) ? INFINITY : -INFINITY) : U(rng); break;
          case 7: v = x[j] + 1e4; break;                                        // a huge offset from the row
          case 8: v = off + U(rng); break;                                      // an offset of 1 .. 1e29
          case 9: v = 0.0; break;                                               // zero query
          case 11: v = -x[j]; break;                                            // opposite: negative dot products
          case 12: v = U(rng) - 0.5; break;
          default: v = U(rng); break;
        }
        q[j] = (float)v;
      }
      if (qk == 10) gaussian_unit(q, dim);
      for (const int metric : metrics) {
        const Pair p = make_pair(q, x, ld, metric);
        const float* hdr = reinterpret_cast<const float*>(p.row.data());
        const float d = kernel_dist(metric, p.s);
        const CodeDotQuery cd = dot_query(metric, p.cq, p.s.qnorm);
        const bool never = hdr[2] == INFINITY || p.cq.eq == INFINITY || (metric == COZO_GPU_COSINE && !(p.s.qnorm > 0.f));
        const float thr = prune_threshold(metric, p, cd);
        const float worsts[] = {d, nextafterf(d, INFINITY), nextafterf(d, -INFINITY), thr, nextafterf(thr, INFINITY),
                                nextafterf(thr, -INFINITY), d * (float)U(rng), d * (float)(1.0 + U(rng)), 0.f, 1.f, -1.f,
                                2.f, 3.40282347e38f, -3.40282347e38f, INFINITY, -INFINITY, NAN};
        ++checked;
        for (const float worst : worsts) {
          const bool pr = prunes(metric, p, cd, worst);
          if (pr && (never || std::isnan(d) || d < worst)) {
            printf("PRUNE VIOLATED: metric %d dim %u kind %u qk %u d %.9g worst %.9g thr %.9g err %.9g e_q %.9g Xn %.9g "
                   "qnorm %.9g S %d\n",
                   metric, dim, kind, qk, d, worst, thr, hdr[2], p.cq.eq, hdr[3], p.s.qnorm, p.S);
            return 1;
          }
          pruned += pr;
        }
      }
    }
  }
  printf("checked %ld (pair, metric) cases, %ld (case, worst) prunes\n", checked, pruned);
  if (pruned == 0) {
    printf("nothing pruned\n");
    return 1;
  }

  // How often it prunes where it matters: per query, 400 rows of the same data; the worst distance is the median of
  // their distances (rows just beyond it are as close to the bound as a hop's neighbours often are), and the rate is the
  // share of the rows at least that far that the test rejects.
  const uint32_t D = 768, NR = 400;
  const char* names[] = {"U[0,1)", "normalised Gaussian"};
  const double floors[2][2] = {{0.5, 0.5}, {0.5, 0.5}};  // [data][IP, Cosine]
  bool low = false;
  for (int data = 0; data < 2; ++data) {
    for (int mi = 0; mi < 2; ++mi) {
      const int metric = metrics[mi];
      long far = 0, rej = 0;
      for (int qi = 0; qi < 20; ++qi) {
        std::vector<float> q(D);
        if (data == 0) for (auto& v : q) v = (float)U(rng);
        else gaussian_unit(q, D);
        std::vector<Pair> ps;
        std::vector<float> ds;
        for (uint32_t i = 0; i < NR; ++i) {
          std::vector<float> x(D);
          if (data == 0) for (auto& v : x) v = (float)U(rng);
          else gaussian_unit(x, D);
          ps.push_back(make_pair(q, x, D, metric));
          ds.push_back(kernel_dist(metric, ps.back().s));
        }
        std::vector<float> sorted = ds;
        std::sort(sorted.begin(), sorted.end());
        const float worst = sorted[NR / 2];
        for (uint32_t i = 0; i < NR; ++i) {
          if (!(ds[i] >= worst)) continue;
          const CodeDotQuery cd = dot_query(metric, ps[i].cq, ps[i].s.qnorm);
          const bool pr = prunes(metric, ps[i], cd, worst);
          ++far;
          rej += pr;
        }
      }
      const double rate = (double)rej / (double)far;
      printf("%s, %s: rejects %.3f of the rows at or beyond the worst distance (floor %.2f)\n", names[data],
             metric == COZO_GPU_IP ? "IP" : "Cosine", rate, floors[data][mi]);
      low = low || rate < floors[data][mi];
    }
  }
  if (low) {
    printf("the test prunes too rarely\n");
    return 1;
  }
  printf("EMU_OK\n");
  return 0;
}
