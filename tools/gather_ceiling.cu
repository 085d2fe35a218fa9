// gather_ceiling.cu — how fast an H100 gathers random rows with cp.async.bulk + mbarrier in the geometry of the
// warp-per-query HNSW search (hnsw_search_kernel): 4 CTAs x 4 warps per SM, one issuing lane per warp, a per-warp ring of
// `depth` requests in flight.  Built and driven by tools/gather_ceiling.py; not part of libcozo_gpu.so.
//
// Each warp owns 14 KB of shared memory, the search kernel's per-warp budget at ef 200 and D = 768, so that 4 CTAs fit
// on an SM as they do in the search.  A row wider than that gets a warp region of one row buffer, and the grid is the
// CTAs that are resident at once (16 KB rows: 3 per SM, 12 warps).  A ring deeper than that many rows reuses row buffers: the rows are never read,
// only their arrival is waited for, so the copies still move every byte.  Latency per request = clock64 at the wait's success minus clock64 at the issue (queueing included).
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

__global__ void __launch_bounds__(128, 4) gather_kernel(const uint8_t* rows, uint64_t nrows, uint32_t row_bytes,
                                                        uint32_t depth, uint32_t reqs, uint32_t warp_smem,
                                                        unsigned long long* lat_sum) {
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
  uint32_t phase = 0;
  unsigned long long lat = 0;
  auto issue = [&](uint32_t i) {
    const uint32_t s = i % depth;
    const uint64_t r = mix(gw * reqs + i) % nrows;
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
}

}  // namespace

// Gathers `reqs` random rows per warp over sm_count x (resident CTAs per SM, at most 4) CTAs; returns 0, the elapsed
// ms, the summed per-request latency in cycles and the number of warps, or the CUDA error code.
extern "C" int gather_run(const void* rows, uint64_t nrows, uint32_t row_bytes, uint32_t depth, uint32_t reqs,
                          float* ms, unsigned long long* lat_cycles, uint32_t* warps) {
  const uint32_t warp_smem = row_bytes > WARP_SMEM - 16 * MAX_DEPTH ? (16 * MAX_DEPTH + row_bytes + 127) / 128 * 128
                                                                     : WARP_SMEM;
  if (depth < 1 || depth > MAX_DEPTH || row_bytes % 16 || 4 * warp_smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int smem = 4 * warp_smem;
  cudaError_t e = cudaFuncSetAttribute(gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  int cps = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, gather_kernel, 128, smem)) != cudaSuccess) return (int)e;
  if (cps < 1) return (int)cudaErrorInvalidValue;
  const int ctas = sms * (cps < 4 ? cps : 4);
  *warps = (uint32_t)ctas * 4;
  unsigned long long* d_lat = nullptr;
  if ((e = cudaMalloc(&d_lat, sizeof(*d_lat))) != cudaSuccess) return (int)e;
  cudaMemset(d_lat, 0, sizeof(*d_lat));
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a);
  gather_kernel<<<ctas, 128, smem>>>(static_cast<const uint8_t*>(rows), nrows, row_bytes, depth, reqs, warp_smem, d_lat);
  cudaEventRecord(b);
  e = cudaEventSynchronize(b);
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
