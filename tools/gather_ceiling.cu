// gather_ceiling.cu — how fast an H100 gathers random rows in the geometry of the warp-per-query HNSW search
// (hnsw_search_kernel): 4 CTAs x 4 warps per SM, `depth` rows in flight per warp.  Built and driven by
// tools/gather_ceiling.py; not part of libcozo_gpu.so.  Three ways to move a row:
//
// bulk: one cp.async.bulk + mbarrier per row, issued by one lane, into a per-warp shared-memory ring.  Each warp owns
// 14 KB of shared memory, the search kernel's per-warp budget at ef 200 and D = 768, so that 4 CTAs fit on an SM as they
// do in the search.  A row wider than that gets a warp region of one row buffer, and the grid is the CTAs that are
// resident at once (16 KB rows: 3 per SM, 12 warps).  A ring deeper than that many rows reuses row buffers: the rows are
// never read, only their arrival is waited for, so the copies still move every byte.
//
// ldg: every lane of the warp reads its words of the row with ld.global.nc.L1::no_allocate straight into registers, in
// the order the code scorer consumes them (word lane + 32 i, so one warp instruction covers one 128-byte span).  The
// warp keeps `depth` rows in flight as register sets and sums each row's words when it is consumed, so no load can be
// removed.  ldg128: the same with 16-byte loads (ld.global.nc.L1::no_allocate.v4, vector lane + 32 i), so a 784-byte row
// is 2 warp instructions instead of 7.  Rows of 784 B (7 words per lane with ldg, 8 with ldg128) and 3072 B (24) are
// supported, at most 96 words per lane in flight with ldg and 72 with ldg128 (its register quads spill at 96).
//
// With a visited bitmap (one per warp, ceil(nrows / 32) words), each row also costs one random atomicOr on it, as the search's
// visited test does.  Latency per request = clock64 when the row is usable (the wait's success, or the row's sum) minus
// clock64 at the issue (queueing included).
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr uint32_t WARP_SMEM = 14336;
constexpr uint32_t MAX_DEPTH = 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint64_t mix(uint64_t x) {  // splitmix64 finaliser: a random row per (warp, request)
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__device__ __forceinline__ uint32_t visit(uint32_t* visited, uint64_t gw, uint64_t nrows, uint64_t r) {
  if (!visited) return 0;
  return atomicOr(visited + gw * ((nrows + 31) / 32) + (r >> 5), 1u << (r & 31));
}

__global__ void __launch_bounds__(128, 4) gather_kernel(const uint8_t* rows, uint64_t nrows, uint32_t row_bytes,
                                                        uint32_t depth, uint32_t reqs, uint32_t warp_smem,
                                                        uint32_t* visited, unsigned long long* lat_sum,
                                                        unsigned long long* sink) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane != 0) return;  // one issuing lane per warp, as in the search
  // per warp: [mbarriers MAX_DEPTH][issue clocks MAX_DEPTH][row buffers]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)warp * warp_smem);
  long long* t_issue = reinterpret_cast<long long*>(bars + MAX_DEPTH);
  uint8_t* buf = reinterpret_cast<uint8_t*>(t_issue + MAX_DEPTH);
  const uint32_t nbuf = (warp_smem - 16 * MAX_DEPTH) / row_bytes;
  const uint64_t gw = (uint64_t)blockIdx.x * 4 + warp;
  for (uint32_t s = 0; s < depth; ++s)
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[s])) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  uint32_t phase = 0, acc = 0;
  unsigned long long lat = 0;
  auto issue = [&](uint32_t i) {
    const uint32_t s = i % depth;
    const uint64_t r = mix(gw * reqs + i) % nrows;
    acc ^= visit(visited, gw, nrows, r);
    t_issue[s] = clock64();
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bars[s])),
                 "r"(row_bytes)
                 : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(buf + (size_t)(s % nbuf) * row_bytes)),
        "l"(rows + r * row_bytes), "r"(row_bytes), "r"(smem_u32(&bars[s]))
        : "memory");
  };
  for (uint32_t i = 0; i < depth && i < reqs; ++i) issue(i);
  for (uint32_t i = 0; i < reqs; ++i) {
    const uint32_t s = i % depth;
    uint32_t ok = 0, spins = 0;
    while (!ok) {
      if (++spins > (1u << 26)) __trap();  // never hang the GPU on a protocol bug
      asm volatile(
          "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(ok)
          : "r"(smem_u32(&bars[s])), "r"((phase >> s) & 1u)
          : "memory");
    }
    phase ^= 1u << s;
    lat += (unsigned long long)(clock64() - t_issue[s]);
    if (i + depth < reqs) issue(i + depth);
  }
  atomicAdd(lat_sum, lat);
  atomicXor(sink, (unsigned long long)acc);
}

// clock64 read after `dep` is available: the fake input keeps the compiler from hoisting it above the row's sum.
__device__ __forceinline__ long long clock_after(uint32_t dep) {
  long long c;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) : "r"(dep) : "memory");
  return c;
}

__device__ __forceinline__ uint32_t ldg_word(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

__device__ __forceinline__ uint4 ldg_vec4(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

// VEC = words per load (1: ld.b32, 4: ld.v4.b32); NW = loads per lane and row
template <int DEPTH, int NW, int VEC>
__global__ void __launch_bounds__(128, 4) ldg_kernel(const uint8_t* rows, uint64_t nrows, uint32_t row_bytes,
                                                     uint32_t reqs, uint32_t* visited, unsigned long long* lat_sum,
                                                     unsigned long long* sink) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t gw = (uint64_t)blockIdx.x * 4 + warp;
  const uint32_t nvecs = row_bytes / (4 * VEC);
  uint32_t v[DEPTH][NW * VEC];
  long long t_issue[DEPTH];
  uint32_t sum = 0, acc = 0;
  unsigned long long lat = 0;
  auto issue = [&](int s, uint32_t i) {
    const uint64_t r = mix(gw * reqs + i) % nrows;
    if (lane == 0) acc ^= visit(visited, gw, nrows, r);
    t_issue[s] = clock64();
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      const uint32_t idx = lane + 32u * w;
      if constexpr (VEC == 1) {
        v[s][w] = idx < nvecs ? ldg_word(reinterpret_cast<const uint32_t*>(rows + r * row_bytes) + idx) : 0u;
      } else {
        const uint4 x = idx < nvecs ? ldg_vec4(reinterpret_cast<const uint4*>(rows + r * row_bytes) + idx)
                                    : make_uint4(0, 0, 0, 0);
        v[s][4 * w] = x.x;
        v[s][4 * w + 1] = x.y;
        v[s][4 * w + 2] = x.z;
        v[s][4 * w + 3] = x.w;
      }
    }
  };
#pragma unroll
  for (int s = 0; s < DEPTH; ++s)
    if ((uint32_t)s < reqs) issue(s, s);
  for (uint32_t base = 0; base < reqs; base += DEPTH) {
#pragma unroll
    for (int s = 0; s < DEPTH; ++s) {
      const uint32_t i = base + s;
      if (i < reqs) {
        uint32_t row = 0;
#pragma unroll
        for (int w = 0; w < NW * VEC; ++w) row += v[s][w];
        sum += row;
        lat += (unsigned long long)(clock_after(row) - t_issue[s]);
        if (i + DEPTH < reqs) issue(s, i + DEPTH);
      }
    }
  }
  sum = __reduce_add_sync(0xffffffffu, sum);
  if (lane == 0) {
    atomicAdd(lat_sum, lat);
    atomicXor(sink, (unsigned long long)(sum ^ acc));
  }
}

// words per lane in flight that fit a 128-register thread without spilling (ptxas -v)
constexpr int ldg_max_words(int vec) { return vec == 1 ? 96 : 72; }

template <int NW, int VEC, int DEPTH = 1>
cudaError_t launch_ldg(int depth, int ctas, const uint8_t* rows, uint64_t nrows, uint32_t row_bytes, uint32_t reqs,
                       uint32_t* visited, unsigned long long* lat, unsigned long long* sink) {
  if constexpr (DEPTH * NW * VEC > ldg_max_words(VEC) || DEPTH > 8) {
    return cudaErrorInvalidValue;
  } else {
    if (depth != DEPTH)
      return launch_ldg<NW, VEC, DEPTH + 1>(depth, ctas, rows, nrows, row_bytes, reqs, visited, lat, sink);
    ldg_kernel<DEPTH, NW, VEC><<<ctas, 128>>>(rows, nrows, row_bytes, reqs, visited, lat, sink);
    return cudaSuccess;
  }
}

}  // namespace

// Gathers `reqs` random rows per warp over sm_count x (resident CTAs per SM, at most 4) CTAs, with mode 0 (bulk),
// 1 (ldg) or 2 (ldg128); `visited` is null or a zeroed bitmap of warps x ceil(nrows / 32) words.  Returns 0, the elapsed ms, the summed
// per-request latency in cycles and the number of warps, or the CUDA error code.  ldg rejects depths whose register
// sets exceed 96 words per lane and row sizes other than 784 and 3072 B.
extern "C" int gather_run(int mode, const void* rows, uint64_t nrows, uint32_t row_bytes, uint32_t depth, uint32_t reqs,
                          uint32_t* visited, float* ms, unsigned long long* lat_cycles, uint32_t* warps) {
  const uint32_t warp_smem = row_bytes > WARP_SMEM - 16 * MAX_DEPTH ? (16 * MAX_DEPTH + row_bytes + 127) / 128 * 128
                                                                     : WARP_SMEM;
  if (depth < 1 || depth > MAX_DEPTH || row_bytes % 16 || 4 * warp_smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  if (mode < 0 || mode > 2 || (mode > 0 && row_bytes != 784 && row_bytes != 3072)) return (int)cudaErrorInvalidValue;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int smem = mode == 0 ? 4 * warp_smem : 0;
  cudaError_t e = cudaSuccess;
  int cps = 0;
  if (mode == 0) {
    if ((e = cudaFuncSetAttribute(gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)) != cudaSuccess)
      return (int)e;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, gather_kernel, 128, smem)) != cudaSuccess) return (int)e;
  } else {
    cps = 4;  // ldg / ldg128 need no shared memory; 4 CTAs of 128 threads at <= 128 registers fit
  }
  if (cps < 1) return (int)cudaErrorInvalidValue;
  const int ctas = sms * (cps < 4 ? cps : 4);
  *warps = (uint32_t)ctas * 4;
  unsigned long long* d_lat = nullptr;
  if ((e = cudaMalloc(&d_lat, 2 * sizeof(*d_lat))) != cudaSuccess) return (int)e;
  cudaMemset(d_lat, 0, 2 * sizeof(*d_lat));
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a);
  const uint8_t* r = static_cast<const uint8_t*>(rows);
  if (mode == 0)
    gather_kernel<<<ctas, 128, smem>>>(r, nrows, row_bytes, depth, reqs, warp_smem, visited, d_lat, d_lat + 1);
  else if (mode == 1)
    e = row_bytes == 784 ? launch_ldg<7, 1>((int)depth, ctas, r, nrows, row_bytes, reqs, visited, d_lat, d_lat + 1)
                         : launch_ldg<24, 1>((int)depth, ctas, r, nrows, row_bytes, reqs, visited, d_lat, d_lat + 1);
  else
    e = row_bytes == 784 ? launch_ldg<2, 4>((int)depth, ctas, r, nrows, row_bytes, reqs, visited, d_lat, d_lat + 1)
                         : launch_ldg<6, 4>((int)depth, ctas, r, nrows, row_bytes, reqs, visited, d_lat, d_lat + 1);
  cudaEventRecord(b);
  if (e == cudaSuccess) e = cudaEventSynchronize(b);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e == cudaSuccess) {
    cudaEventElapsedTime(ms, a, b);
    cudaMemcpy(lat_cycles, d_lat, sizeof(*d_lat), cudaMemcpyDeviceToHost);
  }
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  cudaFree(d_lat);
  return (int)e;
}
