// graph.cu — FixedRule graph algorithms on an HBM-resident CSR:
//   PageRank              (fixed_rule/algos/pagerank.rs:29-56 -> graph::page_rank)
//   multi-source Dijkstra (fixed_rule/algos/shortest_path_dijkstra.rs:274-339)
//   ClosenessCentrality   (fixed_rule/algos/all_pairs_shortest_path.rs:97-143)
//   BetweennessCentrality (fixed_rule/algos/all_pairs_shortest_path.rs:29-95)
// The CSR is what GraphBuilder::csr_layout(Sorted) produces for the edge stream
// of as_directed_graph / as_directed_weighted_graph (fixed_rule/mod.rs:136-328).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

#include "graph_host.hpp"
#include "graph_kernels.cuh"

namespace cozo {

__global__ void edge_check_kernel(const uint32_t* src, const uint32_t* dst, const float* w, uint64_t m, uint32_t n,
                                  int* bad) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  if (src[e] >= n || dst[e] >= n) *bad = 1;
  if (w) {
    float x = w[e];
    if (!(x >= 0.f) || isinf(x)) *bad = 2;  // finite and non-negative (fixed_rule/mod.rs:258-286)
  }
}

__global__ void make_keys_kernel(const uint32_t* hi, const uint32_t* lo, uint64_t m, unsigned long long* keys,
                                 uint32_t* deg) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  keys[e] = ((unsigned long long)hi[e] << 32) | lo[e];
  atomicAdd(&deg[hi[e]], 1u);
}

__global__ void split_keys_kernel(const unsigned long long* keys, uint64_t m, uint32_t* lo) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  lo[e] = (uint32_t)(keys[e] & 0xFFFFFFFFull);
}

__global__ void gather_w_kernel(const float* w, const uint32_t* perm, uint64_t m, float* out) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  out[e] = w[perm[e]];
}

__global__ void iota_kernel(uint32_t* p, uint64_t m) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) p[e] = (uint32_t)e;
}

// the default SSSP kernel: a thin wrapper around sssp_body (graph_kernels.cuh)
template <bool FORB, bool SMEM>
__global__ void __launch_bounds__(256) sssp_kernel(const uint32_t* __restrict__ out_ptr,
                                                   const uint32_t* __restrict__ out_idx,
                                                   const float* __restrict__ out_w, uint32_t n,
                                                   const uint32_t* __restrict__ sources, uint32_t n_src,
                                                   unsigned long long* state, uint8_t* flags, size_t flags_stride,
                                                   ForbiddenSets fs) {
  extern __shared__ __align__(16) uint8_t sssp_smem[];
  sssp_body<FORB, SMEM>(out_ptr, out_idx, out_w, n, sources, n_src, state, flags, flags_stride, fs, sssp_smem);
}

// launch helper.  Default = the flag-scan kernel (shared-memory state when it fits).  Options, both off by default
// because neither form has run on a GPU yet: "sssp.frontier" = 1 -> compacted frontier queues (one CTA per source),
// "sssp.wide" = 1 -> many CTAs per source with one launch per round (host loop, capped at n + 2 rounds).
// "sssp.smem" = 0 keeps the flag-scan state in HBM even when it fits shared memory, so that tests reach the form every
// graph above ~23 k nodes takes with graphs small enough for exact references.
static size_t sssp_flags_stride(uint32_t n) { return ((size_t)n * 9 + 15) & ~(size_t)15; }
template <bool FORB>
static cudaError_t launch_sssp(cozo_gpu_graph_t* g, const uint32_t* d_sources, uint32_t n_src,
                               unsigned long long* state, uint8_t* flags, ForbiddenSets fs, cudaStream_t st) {
  const uint32_t n = g->n;
  const size_t need = (size_t)n * 10;
  const DeviceInfo& di = device_info();
  const size_t fstride = sssp_flags_stride(n);
  if (get_option("sssp.wide", 0) == 1) {
    if (n_src > 65535u) return cudaErrorInvalidValue;  // sources ride on gridDim.y; the wide form is meant for a handful
    uint32_t* counts = nullptr;
    cudaError_t e = cudaMalloc(&counts, (size_t)2 * n_src * 4);
    if (e != cudaSuccess) return e;
    const uint32_t ctas = std::max<uint32_t>(1, (uint32_t)di.sm_count * 4 / n_src);
    sssp_wide_init_kernel<<<dim3(std::min<uint32_t>(ctas, (n + 255) / 256), n_src), 256, 0, st>>>(
        n, d_sources, n_src, state, flags, fstride, counts);
    std::vector<uint32_t> h(n_src);
    uint32_t parity = 0;
    for (uint32_t round = 0; round < n + 2; ++round) {
      sssp_wide_round_kernel<FORB><<<dim3(ctas, n_src), 256, 0, st>>>(g->out_ptr, g->out_idx, g->out_w, n, n_src, state, flags,
                                                                     fstride, counts, parity, fs);
      sssp_wide_reset_kernel<<<(n_src + 255) / 256, 256, 0, st>>>(counts, n_src, parity);  // consumed: next "next"
      parity ^= 1u;
      e = cudaMemcpyAsync(h.data(), counts + (size_t)parity * n_src, (size_t)n_src * 4, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) break;
      bool any = false;
      for (uint32_t c : h) any |= c != 0;
      if (!any) break;
    }
    cudaFree(counts);
    return e != cudaSuccess ? e : cudaGetLastError();
  }
  if (get_option("sssp.frontier", 0) == 1) {
    sssp_queue_kernel<FORB><<<n_src, 256, 0, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                   fstride, fs);
    return cudaGetLastError();
  }
  if (need + 1024 <= di.smem_optin && get_option("sssp.smem", 1) != 0) {
    // raise the kernel's dynamic shared-memory limit, never lower it (concurrent callers with other graphs)
    static std::mutex mu;
    static size_t raised[2] = {0, 0};
    {
      std::lock_guard<std::mutex> lk(mu);
      if (need > raised[FORB ? 1 : 0]) {
        cudaError_t e = cudaFuncSetAttribute(sssp_kernel<FORB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
        if (e != cudaSuccess) return e;
        raised[FORB ? 1 : 0] = need;
      }
    }
    sssp_kernel<FORB, true><<<n_src, 256, need, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                      fstride, fs);
  } else {
    sssp_kernel<FORB, false><<<n_src, 256, 0, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                    fstride, fs);
  }
  return cudaGetLastError();
}

}  // namespace cozo

using namespace cozo;

extern "C" void cozo_gpu_graph_free(cozo_gpu_graph_t* g) {
  if (!g) return;
  void* ptrs[] = {g->out_ptr, g->out_idx, g->in_ptr, g->in_idx, g->out_w};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  pr_state_free(g->pr);
  delete g;
}

extern "C" int cozo_gpu_graph_stage(cozo_gpu_graph_t** out, uint32_t n, uint64_t m, const uint32_t* src,
                                    const uint32_t* dst, const float* w) {
  if (!out) return set_error(COZO_GPU_EINVAL, "null argument");
  *out = nullptr;
  int rc = ensure_init();
  if (rc) return rc;
  if (m && (!src || !dst)) return set_error(COZO_GPU_EINVAL, "null edge arrays");
  if (m >= 0xFFFFFFFFull) return set_error(COZO_GPU_EUNSUP, "more than 2^32-2 edges");
  auto* g = new cozo_gpu_graph();
  g->n = n;
  g->m = m;
  g->weighted = w != nullptr;
  auto fail = [&](int code) {
    cozo_gpu_graph_free(g);
    return code;
  };
#define G_CUDA(call)                                                                              \
  do {                                                                                            \
    cudaError_t _e = (call);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return fail(set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,    \
                            "%s failed: %s (line %d)", #call, cudaGetErrorString(_e), __LINE__)); \
  } while (0)
  const size_t np1 = (size_t)n + 1;
  const size_t mm = std::max<uint64_t>(m, 1);
  G_CUDA(cudaMalloc(&g->out_ptr, np1 * 4));
  G_CUDA(cudaMalloc(&g->in_ptr, np1 * 4));
  G_CUDA(cudaMalloc(&g->out_idx, mm * 4));
  G_CUDA(cudaMalloc(&g->in_idx, mm * 4));
  if (w) G_CUDA(cudaMalloc(&g->out_w, mm * 4));
  G_CUDA(cudaMemset(g->out_ptr, 0, np1 * 4));
  G_CUDA(cudaMemset(g->in_ptr, 0, np1 * 4));
  if (m) {
    DevBuf dsrc, ddst, dw, keys, keys2, perm, perm2, tmp, bad;
    G_CUDA(cudaMalloc(&dsrc.p, m * 4));
    G_CUDA(cudaMalloc(&ddst.p, m * 4));
    G_CUDA(cudaMalloc(&keys.p, m * 8));
    G_CUDA(cudaMalloc(&keys2.p, m * 8));
    G_CUDA(cudaMalloc(&bad.p, 4));
    G_CUDA(cudaMemset(bad.p, 0, 4));
    G_CUDA(cudaMemcpy(dsrc.p, src, m * 4, cudaMemcpyHostToDevice));
    G_CUDA(cudaMemcpy(ddst.p, dst, m * 4, cudaMemcpyHostToDevice));
    if (w) {
      G_CUDA(cudaMalloc(&dw.p, m * 4));
      G_CUDA(cudaMemcpy(dw.p, w, m * 4, cudaMemcpyHostToDevice));
    }
    const uint32_t tb = 256;
    const uint32_t gb = (uint32_t)((m + tb - 1) / tb);
    edge_check_kernel<<<gb, tb>>>(dsrc.as<uint32_t>(), ddst.as<uint32_t>(), dw.as<float>(), m, n, bad.as<int>());
    int hbad = 0;
    G_CUDA(cudaMemcpy(&hbad, bad.p, 4, cudaMemcpyDeviceToHost));
    if (hbad == 1) return fail(set_error(COZO_GPU_EINVAL, "edge endpoint out of range (n=%u)", n));
    if (hbad == 2) return fail(set_error(COZO_GPU_EINVAL, "edge weight must be finite and non-negative"));
    int end_bit = 32;
    while (end_bit < 64 && (n >> (end_bit - 32)) != 0) ++end_bit;  // bits of the row id
    size_t tmp_bytes = 0, tb2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys.as<unsigned long long>(), keys2.as<unsigned long long>(),
                                    (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, 0, end_bit);
    cub::DeviceScan::ExclusiveSum(nullptr, tb2, g->out_ptr, g->out_ptr, (int)np1);
    tmp_bytes = std::max(tmp_bytes, tb2);
    G_CUDA(cudaMalloc(&tmp.p, tmp_bytes));
    // out-CSR: sort by (src, dst); equal pairs keep input order (stable LSD radix sort)
    make_keys_kernel<<<gb, tb>>>(dsrc.as<uint32_t>(), ddst.as<uint32_t>(), m, keys.as<unsigned long long>(),
                                 g->out_ptr);
    if (w) {
      G_CUDA(cudaMalloc(&perm.p, m * 4));
      G_CUDA(cudaMalloc(&perm2.p, m * 4));
      iota_kernel<<<gb, tb>>>(perm.as<uint32_t>(), m);
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortPairs(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(),
                                      perm.as<uint32_t>(), perm2.as<uint32_t>(), (int)m, 0, end_bit);
      gather_w_kernel<<<gb, tb>>>(dw.as<float>(), perm2.as<uint32_t>(), m, g->out_w);
    } else {
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortKeys(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(), (int)m,
                                     0, end_bit);
    }
    split_keys_kernel<<<gb, tb>>>(keys2.as<unsigned long long>(), m, g->out_idx);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceScan::ExclusiveSum(tmp.p, t3, g->out_ptr, g->out_ptr, (int)np1);
    }
    // in-CSR: sort by (dst, src)
    make_keys_kernel<<<gb, tb>>>(ddst.as<uint32_t>(), dsrc.as<uint32_t>(), m, keys.as<unsigned long long>(),
                                 g->in_ptr);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortKeys(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(), (int)m,
                                     0, end_bit);
    }
    split_keys_kernel<<<gb, tb>>>(keys2.as<unsigned long long>(), m, g->in_idx);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceScan::ExclusiveSum(tmp.p, t3, g->in_ptr, g->in_ptr, (int)np1);
    }
    G_CUDA(cudaGetLastError());
    G_CUDA(cudaDeviceSynchronize());
  }
#undef G_CUDA
  *out = g;
  return 0;
}

extern "C" int cozo_gpu_graph_export(cozo_gpu_graph_t* g, uint32_t* out_ptr, uint32_t* out_idx, float* out_w,
                                     uint32_t* in_ptr, uint32_t* in_idx) {
  if (!g) return set_error(COZO_GPU_EINVAL, "null graph handle");
  const size_t np1 = (size_t)g->n + 1;
  if (out_ptr) COZO_CUDA(cudaMemcpy(out_ptr, g->out_ptr, np1 * 4, cudaMemcpyDeviceToHost));
  if (in_ptr) COZO_CUDA(cudaMemcpy(in_ptr, g->in_ptr, np1 * 4, cudaMemcpyDeviceToHost));
  if (out_idx && g->m) COZO_CUDA(cudaMemcpy(out_idx, g->out_idx, g->m * 4, cudaMemcpyDeviceToHost));
  if (in_idx && g->m) COZO_CUDA(cudaMemcpy(in_idx, g->in_idx, g->m * 4, cudaMemcpyDeviceToHost));
  if (out_w && g->m && g->out_w) COZO_CUDA(cudaMemcpy(out_w, g->out_w, g->m * 4, cudaMemcpyDeviceToHost));
  return 0;
}

namespace cozo {
// every call owns a stream: FixedRule::run is invoked concurrently from Rayon workers (query/eval.rs:199-202)
// and independent calls must not serialise on the legacy default stream
struct CallStream {
  cudaStream_t s = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  int init() {
    COZO_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    COZO_CUDA(cudaEventCreate(&e0));
    COZO_CUDA(cudaEventCreate(&e1));
    COZO_CUDA(cudaEventRecord(e0, s));
    return 0;
  }
  double stop() {
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
  }
  ~CallStream() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (s) cudaStreamDestroy(s);
  }
};

// shared driver of the SSSP family: runs sources in chunks that fit `budget` bytes.  "sssp.max_chunk_sources" = k > 0
// caps a chunk at k sources, so that tests run several chunks on small graphs.
template <class PerChunk>
static int sssp_chunks(cozo_gpu_graph_t* g, CallStream& cs, const uint32_t* sources_host, uint32_t n_src,
                       size_t extra_per_src, const volatile int* poison, PerChunk per_chunk) {
  const uint32_t n = g->n;
  const size_t fstride = sssp_flags_stride(n);
  const size_t per_src = (size_t)n * 8 + fstride + extra_per_src;
  size_t freeb = 0, totalb = 0;
  COZO_CUDA(cudaMemGetInfo(&freeb, &totalb));
  size_t budget = std::min<size_t>(freeb / 2, (size_t)8 << 30);
  uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(n_src, budget / std::max<size_t>(per_src, 1)));
  const int64_t max_chunk = get_option("sssp.max_chunk_sources", 0);
  if (max_chunk > 0) chunk = (uint32_t)std::min<int64_t>(chunk, max_chunk);
  DevBuf state, flags, dsrc;
  COZO_CUDA(cudaMalloc(&state.p, (size_t)chunk * n * 8));
  COZO_CUDA(cudaMalloc(&flags.p, (size_t)chunk * fstride));
  COZO_CUDA(cudaMalloc(&dsrc.p, (size_t)chunk * 4));
  int ret = 0;
  for (uint32_t s0 = 0; s0 < n_src && !ret; s0 += chunk) {
    if (poisoned(poison)) {
      ret = set_error(COZO_GPU_EKILLED, "Running query is killed before completion");
      break;
    }
    uint32_t c = std::min(chunk, n_src - s0);
    cudaMemcpyAsync(dsrc.p, sources_host + s0, (size_t)c * 4, cudaMemcpyHostToDevice, cs.s);
    cudaError_t le = launch_sssp<false>(g, dsrc.as<uint32_t>(), c, state.as<unsigned long long>(), flags.as<uint8_t>(),
                                        ForbiddenSets{}, cs.s);
    if (le != cudaSuccess) {
      ret = set_error(COZO_GPU_ECUDA, "sssp launch failed: %s", cudaGetErrorString(le));
      break;
    }
    ret = per_chunk(s0, c, state.as<unsigned long long>(), dsrc.as<uint32_t>());
    cudaError_t ce = cudaStreamSynchronize(cs.s);
    if (!ret && ce != cudaSuccess) ret = set_error(COZO_GPU_ECUDA, "sssp failed: %s", cudaGetErrorString(ce));
  }
  return ret;
}
}  // namespace cozo

extern "C" int cozo_gpu_sssp_multi(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, float* out_dist,
                                   uint32_t* out_pred, double* out_kernel_ms, const volatile int* poison) {
  if (!g || (n_src && (!sources || !out_dist))) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n_src == 0 || n == 0) return 0;
  for (uint32_t i = 0; i < n_src; ++i)
    if (sources[i] >= n) return set_error(COZO_GPU_EINVAL, "source %u out of range", sources[i]);
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf dd, dp;
  rc = sssp_chunks(g, cs, sources, n_src, (size_t)n * 8, poison,
                   [&](uint32_t s0, uint32_t c, unsigned long long* state, uint32_t*) -> int {
                     const uint64_t total = (uint64_t)c * n;
                     if (!dd.p) {
                       COZO_CUDA(cudaMalloc(&dd.p, total * 4));
                       COZO_CUDA(cudaMalloc(&dp.p, total * 4));
                     }
                     sssp_unpack_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, cs.s>>>(state, total, dd.as<float>(),
                                                                                          dp.as<uint32_t>());
                     COZO_CUDA(cudaMemcpyAsync(out_dist + (size_t)s0 * n, dd.p, total * 4, cudaMemcpyDeviceToHost, cs.s));
                     if (out_pred)
                       COZO_CUDA(cudaMemcpyAsync(out_pred + (size_t)s0 * n, dp.p, total * 4, cudaMemcpyDeviceToHost, cs.s));
                     return 0;
                   });
  const double ms = cs.stop();
  if (out_kernel_ms) *out_kernel_ms = ms;
  return rc;
}

extern "C" int cozo_gpu_closeness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms,
                                  const volatile int* poison) {
  if (!g || !out) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;  // all_pairs_shortest_path.rs:111-113
  std::vector<uint32_t> sources(n);
  for (uint32_t i = 0; i < n; ++i) sources[i] = i;
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf dout;
  COZO_CUDA(cudaMalloc(&dout.p, (size_t)n * 4));
  rc = sssp_chunks(g, cs, sources.data(), n, 0, poison,
                   [&](uint32_t s0, uint32_t c, unsigned long long* state, uint32_t*) -> int {
                     closeness_kernel<<<c, 256, 0, cs.s>>>(state, n, c, s0, dout.as<float>());
                     return 0;
                   });
  const double ms = cs.stop();
  if (out_kernel_ms) *out_kernel_ms = ms;
  if (rc) return rc;
  COZO_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaStreamSynchronize(cs.s));
  return 0;
}

extern "C" int cozo_gpu_betweenness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms,
                                    const volatile int* poison) {
  if (!g || !out) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;  // all_pairs_shortest_path.rs:43-46
  std::vector<uint32_t> sources(n);
  for (uint32_t i = 0; i < n; ++i) sources[i] = i;
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf bc, bcf, sig, del, cyc;
  COZO_CUDA(cudaMalloc(&bc.p, (size_t)n * 8));
  COZO_CUDA(cudaMemsetAsync(bc.p, 0, (size_t)n * 8, cs.s));
  COZO_CUDA(cudaMalloc(&bcf.p, (size_t)n * 4));
  COZO_CUDA(cudaMalloc(&cyc.p, 4));
  COZO_CUDA(cudaMemsetAsync(cyc.p, 0, 4, cs.s));
  size_t sig_cap = 0;
  rc = sssp_chunks(g, cs, sources.data(), n, (size_t)n * 32, poison,
                   [&](uint32_t, uint32_t c, unsigned long long* state, uint32_t* dsrc) -> int {
                     size_t need = (size_t)c * 2 * n * 8;
                     if (sig_cap < need) {
                       COZO_CUDA(cudaStreamSynchronize(cs.s));
                       if (sig.p) cudaFree(sig.p);
                       if (del.p) cudaFree(del.p);
                       sig.p = del.p = nullptr;
                       COZO_CUDA(cudaMalloc(&sig.p, need));
                       COZO_CUDA(cudaMalloc(&del.p, need));
                       sig_cap = need;
                     }
                     betweenness_kernel<<<c, 256, 0, cs.s>>>(g->out_ptr, g->out_idx, g->out_w, n, dsrc, c, state,
                                                            sig.as<double>(), del.as<double>(), cyc.as<int>());
                     betweenness_reduce_kernel<<<(n + 255) / 256, 256, 0, cs.s>>>(del.as<double>(), n, c, bc.as<double>());
                     return 0;
                   });
  int hcyc = 0;
  if (!rc) {
    f64_to_f32_kernel<<<(n + 255) / 256, 256, 0, cs.s>>>(bc.as<double>(), n, bcf.as<float>());
    cudaMemcpyAsync(&hcyc, cyc.p, 4, cudaMemcpyDeviceToHost, cs.s);
  }
  const double ms = cs.stop();
  if (out_kernel_ms) *out_kernel_ms = ms;
  if (rc) return rc;
  if (hcyc)
    return set_error(COZO_GPU_EUNSUP, "betweenness: a zero-weight cycle makes the set of tied shortest paths unbounded "
                                      "(the reference does not terminate on this input)");
  COZO_CUDA(cudaMemcpyAsync(out, bcf.p, (size_t)n * 4, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaStreamSynchronize(cs.s));
  return 0;
}

extern "C" int cozo_gpu_clustering(cozo_gpu_graph_t* g, double* out_cc, uint64_t* out_triangles, uint64_t* out_degree,
                                   double* out_kernel_ms, const volatile int* poison) {
  if (!g || !out_cc || !out_triangles || !out_degree) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;
  if (poisoned(poison)) return set_error(COZO_GPU_EKILLED, "Running query is killed before completion");
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf cc, nt, dg;
  COZO_CUDA(cudaMalloc(&cc.p, (size_t)n * 8));
  COZO_CUDA(cudaMalloc(&nt.p, (size_t)n * 8));
  COZO_CUDA(cudaMalloc(&dg.p, (size_t)n * 8));
  clustering_kernel<<<(n + 7) / 8, 256, 0, cs.s>>>(g->out_ptr, g->out_idx, n, cc.as<double>(),
                                                  nt.as<unsigned long long>(), dg.as<unsigned long long>());
  const double ms = cs.stop();
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_error(COZO_GPU_ECUDA, "clustering failed: %s", cudaGetErrorString(ce));
  COZO_CUDA(cudaMemcpyAsync(out_cc, cc.p, (size_t)n * 8, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaMemcpyAsync(out_triangles, nt.p, (size_t)n * 8, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaMemcpyAsync(out_degree, dg.p, (size_t)n * 8, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaStreamSynchronize(cs.s));
  if (out_kernel_ms) *out_kernel_ms = ms;
  return 0;
}

extern "C" int cozo_gpu_sssp_paths(cozo_gpu_graph_t* g, const uint32_t* sources, const uint32_t* goals, uint32_t n_src,
                                   const uint32_t* forb_node_ptr, const uint32_t* forb_nodes,
                                   const uint32_t* forb_edge_ptr, const uint32_t* forb_edge_src,
                                   const uint32_t* forb_edge_dst, uint32_t max_len, float* out_cost, uint32_t* out_len,
                                   uint32_t* out_paths, double* out_kernel_ms, const volatile int* poison) {
  if (!g || (n_src && (!sources || !goals || !out_cost || !out_len || !out_paths)))
    return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n_src == 0 || n == 0) return 0;
  if (max_len == 0) return set_error(COZO_GPU_EINVAL, "max_len must be positive");
  for (uint32_t i = 0; i < n_src; ++i)
    if (sources[i] >= n || goals[i] >= n) return set_error(COZO_GPU_EINVAL, "source/goal out of range");
  if (poisoned(poison)) return set_error(COZO_GPU_EKILLED, "Running query is killed before completion");
  const bool forb = forb_node_ptr && forb_edge_ptr;
  const uint32_t n_fn = forb ? forb_node_ptr[n_src] : 0, n_fe = forb ? forb_edge_ptr[n_src] : 0;
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  cudaStream_t st = cs.s;
  DevBuf state, flags, dsrc, dgoal, fnp, fnn, fep, fes, fed, dc, dl, dp;
  COZO_CUDA(cudaMalloc(&state.p, (size_t)n_src * n * 8));
  COZO_CUDA(cudaMalloc(&flags.p, (size_t)n_src * sssp_flags_stride(n)));
  COZO_CUDA(cudaMalloc(&dsrc.p, (size_t)n_src * 4));
  COZO_CUDA(cudaMalloc(&dgoal.p, (size_t)n_src * 4));
  COZO_CUDA(cudaMalloc(&dc.p, (size_t)n_src * 4));
  COZO_CUDA(cudaMalloc(&dl.p, (size_t)n_src * 4));
  COZO_CUDA(cudaMalloc(&dp.p, (size_t)n_src * max_len * 4));
  COZO_CUDA(cudaMemcpyAsync(dsrc.p, sources, (size_t)n_src * 4, cudaMemcpyHostToDevice, st));
  COZO_CUDA(cudaMemcpyAsync(dgoal.p, goals, (size_t)n_src * 4, cudaMemcpyHostToDevice, st));
  ForbiddenSets fs{};
  if (forb) {
    COZO_CUDA(cudaMalloc(&fnp.p, ((size_t)n_src + 1) * 4));
    COZO_CUDA(cudaMalloc(&fep.p, ((size_t)n_src + 1) * 4));
    COZO_CUDA(cudaMalloc(&fnn.p, std::max<size_t>(n_fn, 1) * 4));
    COZO_CUDA(cudaMalloc(&fes.p, std::max<size_t>(n_fe, 1) * 4));
    COZO_CUDA(cudaMalloc(&fed.p, std::max<size_t>(n_fe, 1) * 4));
    COZO_CUDA(cudaMemcpyAsync(fnp.p, forb_node_ptr, ((size_t)n_src + 1) * 4, cudaMemcpyHostToDevice, st));
    COZO_CUDA(cudaMemcpyAsync(fep.p, forb_edge_ptr, ((size_t)n_src + 1) * 4, cudaMemcpyHostToDevice, st));
    if (n_fn) COZO_CUDA(cudaMemcpyAsync(fnn.p, forb_nodes, (size_t)n_fn * 4, cudaMemcpyHostToDevice, st));
    if (n_fe) {
      COZO_CUDA(cudaMemcpyAsync(fes.p, forb_edge_src, (size_t)n_fe * 4, cudaMemcpyHostToDevice, st));
      COZO_CUDA(cudaMemcpyAsync(fed.p, forb_edge_dst, (size_t)n_fe * 4, cudaMemcpyHostToDevice, st));
    }
    fs = ForbiddenSets{fnp.as<uint32_t>(), fnn.as<uint32_t>(), fep.as<uint32_t>(), fes.as<uint32_t>(),
                       fed.as<uint32_t>()};
  }
  cudaError_t le = forb ? launch_sssp<true>(g, dsrc.as<uint32_t>(), n_src, state.as<unsigned long long>(),
                                            flags.as<uint8_t>(), fs, st)
                        : launch_sssp<false>(g, dsrc.as<uint32_t>(), n_src, state.as<unsigned long long>(),
                                             flags.as<uint8_t>(), fs, st);
  if (le != cudaSuccess) return set_error(COZO_GPU_ECUDA, "sssp launch failed: %s", cudaGetErrorString(le));
  sssp_path_kernel<<<(n_src + 127) / 128, 128, 0, st>>>(state.as<unsigned long long>(), n, dsrc.as<uint32_t>(),
                                                        dgoal.as<uint32_t>(), n_src, max_len, dc.as<float>(),
                                                        dl.as<uint32_t>(), dp.as<uint32_t>());
  const double ms = cs.stop();
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_error(COZO_GPU_ECUDA, "sssp_paths failed: %s", cudaGetErrorString(ce));
  COZO_CUDA(cudaMemcpyAsync(out_cost, dc.p, (size_t)n_src * 4, cudaMemcpyDeviceToHost, st));
  COZO_CUDA(cudaMemcpyAsync(out_len, dl.p, (size_t)n_src * 4, cudaMemcpyDeviceToHost, st));
  COZO_CUDA(cudaMemcpyAsync(out_paths, dp.p, (size_t)n_src * max_len * 4, cudaMemcpyDeviceToHost, st));
  COZO_CUDA(cudaStreamSynchronize(st));
  if (out_kernel_ms) *out_kernel_ms = ms;
  return 0;
}
