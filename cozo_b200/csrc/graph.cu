// graph.cu — FixedRule graph algorithms on an HBM-resident CSR:
//   PageRank              (fixed_rule/algos/pagerank.rs:29-56 -> graph::page_rank)
//   multi-source Dijkstra (fixed_rule/algos/shortest_path_dijkstra.rs:274-339)
//   ClosenessCentrality   (fixed_rule/algos/all_pairs_shortest_path.rs:97-143)
//   BetweennessCentrality (fixed_rule/algos/all_pairs_shortest_path.rs:29-95)
// and the staging of that CSR from dense ids (cozo_gpu_graph_stage) or from node keys (cozo_gpu_graph_stage_keys).
// The CSR is what GraphBuilder::csr_layout(Sorted) produces for the edge stream
// of as_directed_graph / as_directed_weighted_graph (fixed_rule/mod.rs:136-328).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <utility>
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

// the same search stopping once every goal is settled (cozo_gpu_sssp_goals); no forbidden sets
template <bool SMEM>
__global__ void __launch_bounds__(256) sssp_goal_kernel(const uint32_t* __restrict__ out_ptr,
                                                        const uint32_t* __restrict__ out_idx,
                                                        const float* __restrict__ out_w, uint32_t n,
                                                        const uint32_t* __restrict__ sources, uint32_t n_src,
                                                        unsigned long long* state, uint8_t* flags, size_t flags_stride,
                                                        GoalSet gs) {
  extern __shared__ __align__(16) uint8_t sssp_smem[];
  __shared__ float red[64];
  gs.red = red;
  sssp_body<false, SMEM, true>(out_ptr, out_idx, out_w, n, sources, n_src, state, flags, flags_stride, ForbiddenSets{},
                               sssp_smem, gs);
}

// launch helper.  Default = the flag-scan kernel (shared-memory state when it fits).  Options, both off by default
// because neither form has run on a GPU yet: "sssp.frontier" = 1 -> compacted frontier queues (one CTA per source),
// "sssp.wide" = 1 -> many CTAs per source with one launch per round (host loop, capped at n + 2 rounds).
// "sssp.smem" = 0 keeps the flag-scan state in HBM even when it fits shared memory, so that tests reach the form every
// graph above ~23 k nodes takes with graphs small enough for exact references.
// Goals (gs.goals != nullptr, FORB = false): the flag-scan form stops once they are settled; the other two forms run to
// the fixed point, which gives the same answers.
static size_t sssp_flags_stride(uint32_t n) { return ((size_t)n * 9 + 15) & ~(size_t)15; }
template <bool FORB>
static cudaError_t launch_sssp(cozo_gpu_graph_t* g, const uint32_t* d_sources, uint32_t n_src,
                               unsigned long long* state, uint8_t* flags, ForbiddenSets fs, cudaStream_t st,
                               GoalSet gs = GoalSet{}) {
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
    static size_t raised[3] = {0, 0, 0};
    const int slot = gs.goals ? 2 : FORB ? 1 : 0;
    {
      std::lock_guard<std::mutex> lk(mu);
      if (need > raised[slot]) {
        cudaError_t e = gs.goals ? cudaFuncSetAttribute(sssp_goal_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need)
                                 : cudaFuncSetAttribute(sssp_kernel<FORB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
        if (e != cudaSuccess) return e;
        raised[slot] = need;
      }
    }
    if (gs.goals)
      sssp_goal_kernel<true><<<n_src, 256, need, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                       fstride, gs);
    else
      sssp_kernel<FORB, true><<<n_src, 256, need, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                        fstride, fs);
  } else if (gs.goals) {
    sssp_goal_kernel<false><<<n_src, 256, 0, st>>>(g->out_ptr, g->out_idx, g->out_w, n, d_sources, n_src, state, flags,
                                                   fstride, gs);
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
  void* ptrs[] = {g->out_ptr, g->out_idx, g->in_ptr, g->in_idx, g->out_w, g->key_bytes, g->key_off, g->key_id,
                  g->node_first};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  pr_state_free(g->pr);
  delete g;
}

int cozo::graph_build_csr(cozo_gpu_graph_t* g, const uint32_t* dsrc, const uint32_t* ddst, const float* dw,
                          cudaStream_t st) {
#define G_CUDA(call)                                                                         \
  do {                                                                                       \
    cudaError_t _e = (call);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,    \
                       "%s failed: %s (line %d)", #call, cudaGetErrorString(_e), __LINE__); \
  } while (0)
  const uint32_t n = g->n;
  const uint64_t m = g->m;
  const size_t np1 = (size_t)n + 1;
  const size_t mm = std::max<uint64_t>(m, 1);
  G_CUDA(cudaMalloc(&g->out_ptr, np1 * 4));
  G_CUDA(cudaMalloc(&g->in_ptr, np1 * 4));
  G_CUDA(cudaMalloc(&g->out_idx, mm * 4));
  G_CUDA(cudaMalloc(&g->in_idx, mm * 4));
  if (g->weighted) G_CUDA(cudaMalloc(&g->out_w, mm * 4));
  G_CUDA(cudaMemsetAsync(g->out_ptr, 0, np1 * 4, st));
  G_CUDA(cudaMemsetAsync(g->in_ptr, 0, np1 * 4, st));
  if (m) {
    DevBuf keys, keys2, perm, perm2, tmp, bad;
    G_CUDA(cudaMalloc(&keys.p, m * 8));
    G_CUDA(cudaMalloc(&keys2.p, m * 8));
    G_CUDA(cudaMalloc(&bad.p, 4));
    G_CUDA(cudaMemsetAsync(bad.p, 0, 4, st));
    const uint32_t tb = 256;
    const uint32_t gb = (uint32_t)((m + tb - 1) / tb);
    edge_check_kernel<<<gb, tb, 0, st>>>(dsrc, ddst, dw, m, n, bad.as<int>());
    int hbad = 0;
    G_CUDA(cudaMemcpyAsync(&hbad, bad.p, 4, cudaMemcpyDeviceToHost, st));
    G_CUDA(cudaStreamSynchronize(st));
    if (hbad == 1) return set_error(COZO_GPU_EINVAL, "edge endpoint out of range (n=%u)", n);
    if (hbad == 2) return set_error(COZO_GPU_EINVAL, "edge weight must be finite and non-negative");
    int end_bit = 32;
    while (end_bit < 64 && (n >> (end_bit - 32)) != 0) ++end_bit;  // bits of the row id
    size_t tmp_bytes = 0, tb2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys.as<unsigned long long>(), keys2.as<unsigned long long>(),
                                    (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, 0, end_bit, st);
    cub::DeviceScan::ExclusiveSum(nullptr, tb2, g->out_ptr, g->out_ptr, (int)np1, st);
    tmp_bytes = std::max(tmp_bytes, tb2);
    G_CUDA(cudaMalloc(&tmp.p, tmp_bytes));
    // out-CSR: sort by (src, dst); equal pairs keep input order (stable LSD radix sort)
    make_keys_kernel<<<gb, tb, 0, st>>>(dsrc, ddst, m, keys.as<unsigned long long>(), g->out_ptr);
    if (dw) {
      G_CUDA(cudaMalloc(&perm.p, m * 4));
      G_CUDA(cudaMalloc(&perm2.p, m * 4));
      iota_kernel<<<gb, tb, 0, st>>>(perm.as<uint32_t>(), m);
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortPairs(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(),
                                      perm.as<uint32_t>(), perm2.as<uint32_t>(), (int)m, 0, end_bit, st);
      gather_w_kernel<<<gb, tb, 0, st>>>(dw, perm2.as<uint32_t>(), m, g->out_w);
    } else {
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortKeys(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(), (int)m,
                                     0, end_bit, st);
    }
    split_keys_kernel<<<gb, tb, 0, st>>>(keys2.as<unsigned long long>(), m, g->out_idx);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceScan::ExclusiveSum(tmp.p, t3, g->out_ptr, g->out_ptr, (int)np1, st);
    }
    // in-CSR: sort by (dst, src)
    make_keys_kernel<<<gb, tb, 0, st>>>(ddst, dsrc, m, keys.as<unsigned long long>(), g->in_ptr);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceRadixSort::SortKeys(tmp.p, t3, keys.as<unsigned long long>(), keys2.as<unsigned long long>(), (int)m,
                                     0, end_bit, st);
    }
    split_keys_kernel<<<gb, tb, 0, st>>>(keys2.as<unsigned long long>(), m, g->in_idx);
    {
      size_t t3 = tmp_bytes;
      cub::DeviceScan::ExclusiveSum(tmp.p, t3, g->in_ptr, g->in_ptr, (int)np1, st);
    }
    G_CUDA(cudaGetLastError());
  }
  G_CUDA(cudaStreamSynchronize(st));
#undef G_CUDA
  return 0;
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
  DevBuf dsrc, ddst, dw;
  if (m) {
    G_CUDA(cudaMalloc(&dsrc.p, m * 4));
    G_CUDA(cudaMalloc(&ddst.p, m * 4));
    G_CUDA(cudaMemcpy(dsrc.p, src, m * 4, cudaMemcpyHostToDevice));
    G_CUDA(cudaMemcpy(ddst.p, dst, m * 4, cudaMemcpyHostToDevice));
    if (w) {
      G_CUDA(cudaMalloc(&dw.p, m * 4));
      G_CUDA(cudaMemcpy(dw.p, w, m * 4, cudaMemcpyHostToDevice));
    }
  }
#undef G_CUDA
  // the legacy default stream, as before the dense path was shared with cozo_gpu_graph_stage_keys
  rc = graph_build_csr(g, dsrc.as<uint32_t>(), ddst.as<uint32_t>(), w ? dw.as<float>() : nullptr, 0);
  if (rc) return fail(rc);
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
// shared driver of the SSSP family: runs sources in chunks that fit `budget` bytes.  "sssp.max_chunk_sources" = k > 0
// caps a chunk at k sources, so that tests run several chunks on small graphs.
template <class PerChunk>
static int sssp_chunks(cozo_gpu_graph_t* g, CallStream& cs, const uint32_t* sources_host, uint32_t n_src,
                       size_t extra_per_src, const volatile int* poison, PerChunk per_chunk, GoalSet gs = GoalSet{}) {
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
                                        ForbiddenSets{}, cs.s, gs);
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

int cozo::sssp_goals_check(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                           uint32_t n_goals) {
  const uint32_t n = g->n;
  for (uint32_t i = 0; i < n_src; ++i)
    if (sources[i] >= n) return set_error(COZO_GPU_EINVAL, "source %u out of range", sources[i]);
  std::vector<uint32_t> sorted(goals, goals + n_goals);
  std::sort(sorted.begin(), sorted.end());
  for (uint32_t i = 0; i < n_goals; ++i) {
    if (sorted[i] >= n) return set_error(COZO_GPU_EINVAL, "goal %u out of range", sorted[i]);
    if (i && sorted[i] == sorted[i - 1]) return set_error(COZO_GPU_EINVAL, "goal %u given twice", sorted[i]);
  }
  return 0;
}

int cozo::sssp_goals_run(cozo_gpu_graph_t* g, CallStream& cs, const uint32_t* sources, uint32_t n_src,
                         const uint32_t* goals, uint32_t n_goals, bool keep_ties, float* out_cost, uint64_t* off_out,
                         uint64_t cap, const volatile int* poison, const GoalRowSink& sink) {
  const uint32_t n = g->n;
  DevBuf dgoal, dcost, dscan, dmark, drows, tmp;
  COZO_CUDA(cudaMalloc(&dgoal.p, (size_t)n_goals * 4));
  COZO_CUDA(cudaMemcpyAsync(dgoal.p, goals, (size_t)n_goals * 4, cudaMemcpyHostToDevice, cs.s));
  const GoalSet gs{dgoal.as<uint32_t>(), n_goals, nullptr};
  uint64_t base = 0, rows_cap = 0;  // rows so far; capacity of drows in rows (a path node, or one (v, p) pair)
  bool fits = true;
  size_t tmp_bytes = 0;
  return sssp_chunks(
      g, cs, sources, n_src, (size_t)n_goals * 12 + (keep_ties ? (size_t)n + 8 : 0), poison,
      [&](uint32_t s0, uint32_t c, unsigned long long* state, uint32_t* dsrc) -> int {
        const uint64_t pc = (uint64_t)c * n_goals;
        const uint64_t m = keep_ties ? (uint64_t)c : pc;  // entries scanned, plus the one that receives the total
        if (!dcost.p) {  // the first chunk is the largest
          COZO_CUDA(cudaMalloc(&dcost.p, pc * 4));
          COZO_CUDA(cudaMalloc(&dscan.p, (m + 1) * 8));
          if (keep_ties) COZO_CUDA(cudaMalloc(&dmark.p, (size_t)c * n));
          cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, dscan.as<uint64_t>(), dscan.as<uint64_t>(), (int64_t)m + 1,
                                        cs.s);
          COZO_CUDA(cudaMalloc(&tmp.p, std::max<size_t>(tmp_bytes, 16)));
        }
        uint64_t* scan = dscan.as<uint64_t>();
        sssp_goal_len_kernel<<<(uint32_t)((pc + 256) / 256), 256, 0, cs.s>>>(state, n, dsrc, gs.goals, n_goals, c,
                                                                            dcost.as<float>(), keep_ties ? nullptr : scan);
        if (keep_ties)
          sssp_tie_mark_kernel<<<c, 256, 0, cs.s>>>(g->out_ptr, g->out_idx, g->out_w, n, dsrc, gs, c, state,
                                                   dmark.as<uint8_t>(), scan);
        size_t t3 = tmp_bytes;
        cub::DeviceScan::ExclusiveSum(tmp.p, t3, scan, scan, (int64_t)m + 1, cs.s);
        COZO_CUDA(cudaGetLastError());
        COZO_CUDA(cudaMemcpyAsync(out_cost + (size_t)s0 * n_goals, dcost.p, pc * 4, cudaMemcpyDeviceToHost, cs.s));
        uint64_t* off = off_out + (keep_ties ? (uint64_t)s0 : (uint64_t)s0 * n_goals);
        COZO_CUDA(cudaMemcpyAsync(off, scan, (m + 1) * 8, cudaMemcpyDeviceToHost, cs.s));
        COZO_CUDA(cudaStreamSynchronize(cs.s));
        const uint64_t total = off[m];
        for (uint64_t i = 0; i <= m; ++i) off[i] += base;
        fits = fits && base + total <= cap;
        if (fits && total) {
          if (rows_cap < total) {
            if (drows.p) cudaFree(drows.p);
            drows.p = nullptr;
            COZO_CUDA(cudaMalloc(&drows.p, total * (keep_ties ? 8 : 4)));
            rows_cap = total;
          }
          if (keep_ties)
            sssp_tie_write_kernel<<<c, 256, 0, cs.s>>>(g->out_ptr, g->out_idx, g->out_w, n, dsrc, c, state,
                                                      dmark.as<uint8_t>(), scan, drows.as<uint32_t>());
          else
            sssp_goal_path_kernel<<<(uint32_t)((pc + 255) / 256), 256, 0, cs.s>>>(state, n, gs.goals, n_goals, c, scan,
                                                                                 drows.as<uint32_t>());
          COZO_CUDA(cudaGetLastError());
          const int rc = sink(drows.as<uint32_t>(), base, total);
          if (rc) return rc;
        }
        base += total;
        return 0;
      },
      gs);
}

extern "C" int cozo_gpu_sssp_goals(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                                   uint32_t n_goals, int32_t keep_ties, float* out_cost, uint64_t* out_path_off,
                                   uint32_t* out_paths, uint64_t paths_cap, uint64_t* out_tie_off,
                                   uint32_t* out_tie_edges, uint64_t ties_cap, double* out_kernel_ms,
                                   const volatile int* poison) {
  const uint64_t pairs = (uint64_t)n_src * n_goals;
  uint64_t* off_out = keep_ties ? out_tie_off : out_path_off;
  uint32_t* rows_out = keep_ties ? out_tie_edges : out_paths;
  const uint64_t cap = keep_ties ? ties_cap : paths_cap;
  if (!g || (n_src && !sources) || (n_goals && !goals) || (pairs && !out_cost) || !off_out || (cap && !rows_out))
    return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  rc = sssp_goals_check(g, sources, n_src, goals, n_goals);
  if (rc) return rc;
  // offsets per pair (paths) or per source (tied edges); a source with no goals has none of either
  const uint64_t n_off = keep_ties ? (uint64_t)n_src + 1 : pairs + 1;
  std::fill(off_out, off_out + n_off, 0);
  if (pairs == 0) return 0;
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  const uint64_t per_row = keep_ties ? 2 : 1;
  rc = sssp_goals_run(g, cs, sources, n_src, goals, n_goals, keep_ties != 0, out_cost, off_out, cap, poison,
                      [&](const uint32_t* drows, uint64_t base, uint64_t total) -> int {
                        COZO_CUDA(cudaMemcpyAsync(rows_out + base * per_row, drows, total * per_row * 4,
                                                  cudaMemcpyDeviceToHost, cs.s));
                        return 0;
                      });
  const double ms = cs.stop();
  if (out_kernel_ms) *out_kernel_ms = ms;
  return rc;
}

int cozo::closeness_run(cozo_gpu_graph_t* g, CallStream& cs, uint32_t lo, uint32_t hi, float* dout,
                        const volatile int* poison) {
  const uint32_t n = g->n;
  std::vector<uint32_t> sources(hi - lo);
  for (uint32_t i = lo; i < hi; ++i) sources[i - lo] = i;
  return sssp_chunks(g, cs, sources.data(), hi - lo, 0, poison,
                     [&](uint32_t s0, uint32_t c, unsigned long long* state, uint32_t*) -> int {
                       closeness_kernel<<<c, 256, 0, cs.s>>>(state, n, c, s0, dout);
                       return 0;
                     });
}

extern "C" int cozo_gpu_closeness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms,
                                  const volatile int* poison) {
  if (!g || !out) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;  // all_pairs_shortest_path.rs:111-113
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf dout;
  COZO_CUDA(cudaMalloc(&dout.p, (size_t)n * 4));
  rc = closeness_run(g, cs, 0, n, dout.as<float>(), poison);
  const double ms = cs.stop();
  if (out_kernel_ms) *out_kernel_ms = ms;
  if (rc) return rc;
  COZO_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaStreamSynchronize(cs.s));
  return 0;
}

int cozo::betweenness_run(cozo_gpu_graph_t* g, CallStream& cs, uint32_t lo, uint32_t hi, double* dbc, int* dcyc,
                          const volatile int* poison) {
  const uint32_t n = g->n;
  std::vector<uint32_t> sources(hi - lo);
  for (uint32_t i = lo; i < hi; ++i) sources[i - lo] = i;
  DevBuf sig, del;
  size_t sig_cap = 0;
  return sssp_chunks(g, cs, sources.data(), hi - lo, (size_t)n * 32, poison,
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
                                                              sig.as<double>(), del.as<double>(), dcyc);
                       betweenness_reduce_kernel<<<(n + 255) / 256, 256, 0, cs.s>>>(del.as<double>(), n, c, dbc);
                       return 0;
                     });
}

extern "C" int cozo_gpu_betweenness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms,
                                    const volatile int* poison) {
  if (!g || !out) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;  // all_pairs_shortest_path.rs:43-46
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  DevBuf bc, bcf, cyc;
  COZO_CUDA(cudaMalloc(&bc.p, (size_t)n * 8));
  COZO_CUDA(cudaMemsetAsync(bc.p, 0, (size_t)n * 8, cs.s));
  COZO_CUDA(cudaMalloc(&bcf.p, (size_t)n * 4));
  COZO_CUDA(cudaMalloc(&cyc.p, 4));
  COZO_CUDA(cudaMemsetAsync(cyc.p, 0, 4, cs.s));
  rc = betweenness_run(g, cs, 0, n, bc.as<double>(), cyc.as<int>(), poison);
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

// ---- cozo_gpu_graph_stage_keys: dense node ids from node KEYS, on the device ----
// as_directed_graph / as_directed_weighted_graph (fixed_rule/mod.rs:136-328) give every distinct node key a dense id in
// first-appearance order over the endpoints from_0, to_0, from_1, ... (mod.rs:164-179) through a BTreeMap<DataValue,
// u32>.  Here the keys arrive as byte strings (their memcmp encodings, data/memcmp.rs: equal bytes <=> equal values):
//   1. the 2m endpoints are grouped EXACTLY by refinement: a stable radix sort by length, then for every 8-byte
//      big-endian word r a stable sort by word r and a stable sort by group; a group splits where the word differs.
//      Rounds stop when no group holds two endpoints with bytes left to compare.  No hash is ever trusted.
//   2. stable sorts keep the members of a group in endpoint order, so a group's first member is the key's first
//      appearance; an exclusive scan of first-appearance flags in endpoint order ranks the groups: the dense ids.
//   3. the ids go back to the endpoints, edges are mirrored if asked, and the dense stream enters the CSR build of
//      cozo_gpu_graph_stage (graph_build_csr) without leaving the device.
//   4. the distinct keys stay on the handle in group order, i.e. sorted by (length, bytes), for binary-search lookups.
namespace cozo {

constexpr uint32_t KTB = 256;
static uint32_t kblocks(uint64_t n) { return (uint32_t)((n + KTB - 1) / KTB); }
static int bit_width(unsigned long long x) {
  int b = 0;
  while (b < 64 && (x >> b) != 0) ++b;
  return std::max(b, 1);
}
static void release(DevBuf& b) {
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
}

// refinement word r of key e: r = 0 is the length, r >= 1 the bytes [8(r-1), 8r) big-endian, zero past the end
__device__ __forceinline__ unsigned long long key_word(const uint8_t* bytes, const uint64_t* off, uint32_t e,
                                                       uint32_t r) {
  const uint64_t b = off[e], len = off[e + 1] - b;
  if (r == 0) return len;
  const uint64_t s = (uint64_t)(r - 1) * 8;
  unsigned long long w = 0;
  for (uint32_t i = 0; i < 8; ++i) w = (w << 8) | (s + i < len ? bytes[b + s + i] : 0u);
  return w;
}

// offsets must not decrease; the OR of all lengths has the bit width of the longest one
__global__ void key_off_check_kernel(const uint64_t* off, uint64_t E, int* bad, unsigned long long* len_or) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long len = 0;
  if (e < E) {
    const uint64_t a = off[e], b = off[e + 1];
    if (b < a) *bad = 1;
    else len = b - a;
  }
  for (int o = 16; o > 0; o >>= 1) len |= __shfl_xor_sync(0xffffffffu, len, o);
  if ((threadIdx.x & 31) == 0 && len) atomicOr(len_or, len);
}

__global__ void key_iota_kernel(uint32_t* p, uint64_t E) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < E) p[i] = (uint32_t)i;
}

__global__ void key_word_kernel(const uint8_t* bytes, const uint64_t* off, const uint32_t* perm, uint64_t E, uint32_t r,
                                unsigned long long* w) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < E) w[p] = key_word(bytes, off, perm[p], r);
}

__global__ void key_gather_group_kernel(const uint32_t* grp, const uint32_t* perm, uint64_t E, uint32_t* out) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < E) out[p] = grp[perm[p]];
}

// in sorted order: a new group starts where the old group or word r changes
__global__ void key_heads_kernel(const uint8_t* bytes, const uint64_t* off, const uint32_t* perm, const uint32_t* grp,
                                 uint64_t E, uint32_t r, uint32_t* head) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= E) return;
  if (p == 0) {
    head[0] = 1;
    return;
  }
  const uint32_t a = perm[p - 1], b = perm[p];
  head[p] = grp[a] != grp[b] || key_word(bytes, off, a, r) != key_word(bytes, off, b, r);
}

// group id = exclusive scan of the heads + head - 1.  state[0] = 1 while some group holds two endpoints whose keys are
// longer than the `compared` bytes already looked at; state[1] = number of groups.
__global__ void key_assign_kernel(const uint64_t* off, const uint32_t* perm, const uint32_t* head, const uint32_t* excl,
                                  uint64_t E, uint64_t compared, uint32_t* grp, uint32_t* state) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= E) return;
  const uint32_t e = perm[p];
  grp[e] = excl[p] + head[p] - 1;
  if (!head[p] && off[e + 1] - off[e] > compared) state[0] = 1;
  if (p == E - 1) state[1] = excl[p] + head[p];
}

// the first member of every group (smallest endpoint index): flag it and remember it per group
__global__ void key_first_kernel(const uint32_t* perm, const uint32_t* head, const uint32_t* grp, uint64_t E,
                                 uint32_t* is_first, uint32_t* gfirst) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= E || !head[p]) return;
  const uint32_t e = perm[p];
  is_first[e] = 1;
  gfirst[grp[e]] = e;
}

// dense id of group g = rank of its first appearance among all first appearances
__global__ void key_rank_kernel(const uint32_t* gfirst, const uint32_t* rank, const uint64_t* off, uint32_t n,
                                uint32_t* gid, uint32_t* node_first, uint64_t* klen) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n) return;
  if (g == n) {
    klen[n] = 0;
    return;
  }
  const uint32_t e = gfirst[g], id = rank[e];
  gid[g] = id;
  node_first[id] = e;
  klen[g] = off[e + 1] - off[e];
}

__global__ void key_copy_kernel(const uint8_t* bytes, const uint64_t* off, const uint32_t* gfirst, const uint64_t* koff,
                                uint32_t n, uint8_t* kbytes) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const uint64_t s = off[gfirst[g]], d = koff[g], len = koff[g + 1] - d;
  for (uint64_t i = 0; i < len; ++i) kbytes[d + i] = bytes[s + i];
}

// the dense edge stream of as_directed_graph: edge e = (id of endpoint 2e, id of endpoint 2e+1), its mirror right
// after it when undirected (mod.rs:187-191)
__global__ void key_edges_kernel(const uint32_t* grp, const uint32_t* gid, const float* w, uint64_t m, int undirected,
                                 uint32_t* src, uint32_t* dst, float* w2) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= m) return;
  const uint32_t a = gid[grp[2 * e]], b = gid[grp[2 * e + 1]];
  if (undirected) {
    src[2 * e] = a;
    dst[2 * e] = b;
    src[2 * e + 1] = b;
    dst[2 * e + 1] = a;
    if (w) w2[2 * e] = w2[2 * e + 1] = w[e];
  } else {
    src[e] = a;
    dst[e] = b;
    if (w) w2[e] = w[e];
  }
}

// binary search of every query key among the distinct keys, ordered by (length, bytes)
__global__ void key_lookup_kernel(const uint8_t* kbytes, const uint64_t* koff, const uint32_t* kid, uint32_t n,
                                  const uint8_t* qbytes, const uint64_t* qoff, uint32_t count, uint32_t* out) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= count) return;
  const uint8_t* a = qbytes + qoff[q];
  const uint64_t la = qoff[q + 1] - qoff[q];
  uint32_t lo = 0, hi = n, res = NONE;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    const uint64_t lb = koff[mid + 1] - koff[mid];
    int c = la < lb ? -1 : (la > lb ? 1 : 0);
    for (uint64_t i = 0; c == 0 && i < la; ++i) {
      const uint8_t x = a[i], y = kbytes[koff[mid] + i];
      c = x < y ? -1 : (x > y ? 1 : 0);
    }
    if (c == 0) {
      res = kid[mid];
      break;
    }
    if (c < 0) hi = mid;
    else lo = mid + 1;
  }
  out[q] = res;
}

}  // namespace cozo

using namespace cozo;

extern "C" int cozo_gpu_graph_stage_keys(cozo_gpu_graph_t** out, uint64_t m, const uint8_t* key_bytes,
                                         const uint64_t* key_off, const float* w, int32_t undirected,
                                         uint32_t* out_n) {
  if (!out || !out_n) return set_error(COZO_GPU_EINVAL, "null argument");
  *out = nullptr;
  *out_n = 0;
  int rc = ensure_init();
  if (rc) return rc;
  if (m && (!key_bytes || !key_off)) return set_error(COZO_GPU_EINVAL, "null key arrays");
  const uint64_t m2 = undirected ? 2 * m : m;
  if (m >= 0x7FFFFFFFull || m2 >= 0xFFFFFFFFull)
    return set_error(COZO_GPU_EUNSUP, "more than 2^32-2 edges after mirroring or 2^32-2 endpoints");
  const uint64_t E = 2 * m;  // also bounds the distinct keys below 2^32-2
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  cudaStream_t st = cs.s;
  auto* g = new cozo_gpu_graph();
  g->m = m2;
  g->weighted = w != nullptr;
  g->keyed = true;
  auto fail = [&](int code) {
    cozo_gpu_graph_free(g);
    return code;
  };
  size_t need = 0;  // the refinement's peak, reported when an allocation fails
#define K_CUDA(call)                                                                                              \
  do {                                                                                                            \
    cudaError_t _e = (call);                                                                                      \
    if (_e == cudaErrorMemoryAllocation)                                                                          \
      return fail(set_error(COZO_GPU_ENOMEM, "stage_keys: %s failed: out of device memory (the call needs about %zu " \
                                             "bytes for %llu endpoints)", #call, need, (unsigned long long)E));   \
    if (_e != cudaSuccess)                                                                                        \
      return fail(set_error(COZO_GPU_ECUDA, "%s failed: %s (line %d)", #call, cudaGetErrorString(_e), __LINE__)); \
  } while (0)
  if (m == 0) {
    rc = graph_build_csr(g, nullptr, nullptr, nullptr, st);
    if (rc) return fail(rc);
    *out = g;
    return 0;
  }
  const uint32_t gbE = kblocks(E);
  DevBuf doff, dbytes, dw, state;
  K_CUDA(cudaMalloc(&doff.p, (E + 1) * 8));
  K_CUDA(cudaMalloc(&state.p, 32));
  K_CUDA(cudaMemsetAsync(state.p, 0, 32, st));
  K_CUDA(cudaMemcpyAsync(doff.p, key_off, (E + 1) * 8, cudaMemcpyHostToDevice, st));
  int* dbad = state.as<int>() + 4;
  unsigned long long* dlen_or = reinterpret_cast<unsigned long long*>(state.as<uint8_t>() + 24);
  key_off_check_kernel<<<gbE, KTB, 0, st>>>(doff.as<uint64_t>(), E, dbad, dlen_or);
  uint32_t hstate[8] = {};
  K_CUDA(cudaMemcpyAsync(hstate, state.p, 32, cudaMemcpyDeviceToHost, st));
  K_CUDA(cudaStreamSynchronize(st));
  if (hstate[4]) return fail(set_error(COZO_GPU_EINVAL, "key offsets decrease"));
  unsigned long long len_or = 0;
  std::memcpy(&len_or, hstate + 6, 8);
  const uint64_t B = key_off[E];  // offsets checked: the last one bounds every key

  // CUB scratch for the largest call of each kind, then the peak (DESIGN.md §3.6)
  size_t tmp_bytes = 0, t = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)E, 0, 64, st);
  tmp_bytes = std::max(tmp_bytes, t);
  cub::DeviceRadixSort::SortPairs(nullptr, t, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int64_t)E, 0, 32, st);
  tmp_bytes = std::max(tmp_bytes, t);
  cub::DeviceScan::ExclusiveSum(nullptr, t, (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)E, st);
  tmp_bytes = std::max(tmp_bytes, t);
  cub::DeviceScan::ExclusiveSum(nullptr, t, (uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)E + 1, st);
  tmp_bytes = std::max(tmp_bytes, t);
  need = (size_t)B + (E + 1) * 8 + E * 28 + tmp_bytes + (w ? m * 4 : 0) + 64;
  {
    size_t freeb = 0, totalb = 0;
    K_CUDA(cudaMemGetInfo(&freeb, &totalb));
    if (need > freeb)
      return fail(set_error(COZO_GPU_ENOMEM,
                            "stage_keys needs about %zu bytes of device memory for %llu endpoints and %llu key bytes; "
                            "%zu are free",
                            need, (unsigned long long)E, (unsigned long long)B, freeb));
  }
  K_CUDA(cudaMalloc(&dbytes.p, std::max<uint64_t>(B, 1)));
  if (B) K_CUDA(cudaMemcpyAsync(dbytes.p, key_bytes, B, cudaMemcpyHostToDevice, st));
  if (w) {
    K_CUDA(cudaMalloc(&dw.p, m * 4));
    K_CUDA(cudaMemcpyAsync(dw.p, w, m * 4, cudaMemcpyHostToDevice, st));
  }
  const uint8_t* bytes = dbytes.as<uint8_t>();
  const uint64_t* off = doff.as<uint64_t>();

  // ---- 1. exact refinement ----
  // K: the sort keys of a round (words: 2 x E u64), reused as group keys (2 x E u32) and, once those are sorted,
  // as heads + their scan (2 x E u32)
  DevBuf K, perm, perm2, grp, tmp;
  K_CUDA(cudaMalloc(&K.p, E * 16));
  K_CUDA(cudaMalloc(&perm.p, E * 4));
  K_CUDA(cudaMalloc(&perm2.p, E * 4));
  K_CUDA(cudaMalloc(&grp.p, E * 4));
  K_CUDA(cudaMalloc(&tmp.p, std::max<size_t>(tmp_bytes, 16)));
  unsigned long long* W = K.as<unsigned long long>();
  unsigned long long* W2 = W + E;
  uint32_t* G = K.as<uint32_t>();
  uint32_t* G2 = G + E;
  uint32_t* head = G + 2 * E;
  uint32_t* excl = G + 3 * E;
  uint32_t* P = perm.as<uint32_t>();
  uint32_t* P2 = perm2.as<uint32_t>();
  uint32_t* grp_of = grp.as<uint32_t>();
  uint32_t* hst = state.as<uint32_t>();
  key_iota_kernel<<<gbE, KTB, 0, st>>>(P, E);
  K_CUDA(cudaMemsetAsync(grp_of, 0, E * 4, st));  // round 0 starts from one group
  uint32_t n_groups = 1;
  for (uint32_t r = 0;; ++r) {
    size_t t3 = tmp_bytes;
    key_word_kernel<<<gbE, KTB, 0, st>>>(bytes, off, P, E, r, W);
    cub::DeviceRadixSort::SortPairs(tmp.p, t3, W, W2, P, P2, (int64_t)E, 0, r == 0 ? bit_width(len_or) : 64, st);
    if (n_groups > 1) {  // stable by group: the groups stay contiguous, word-sorted inside
      key_gather_group_kernel<<<gbE, KTB, 0, st>>>(grp_of, P2, E, G);
      t3 = tmp_bytes;
      cub::DeviceRadixSort::SortPairs(tmp.p, t3, G, G2, P2, P, (int64_t)E, 0, bit_width(n_groups - 1), st);
    } else {
      std::swap(P, P2);
    }
    key_heads_kernel<<<gbE, KTB, 0, st>>>(bytes, off, P, grp_of, E, r, head);
    t3 = tmp_bytes;
    cub::DeviceScan::ExclusiveSum(tmp.p, t3, head, excl, (int64_t)E, st);
    K_CUDA(cudaMemsetAsync(hst, 0, 4, st));
    key_assign_kernel<<<gbE, KTB, 0, st>>>(off, P, head, excl, E, (uint64_t)r * 8, grp_of, hst);
    K_CUDA(cudaMemcpyAsync(hstate, hst, 8, cudaMemcpyDeviceToHost, st));
    K_CUDA(cudaStreamSynchronize(st));
    K_CUDA(cudaGetLastError());
    n_groups = hstate[1];
    if (!hstate[0] || n_groups == E) break;
  }
  const uint32_t n = n_groups;
  g->n = n;

  // ---- 2. first appearances -> dense ids ----
  DevBuf gfirst, klen;
  uint32_t* is_first = G;  // heads stay in place: [2E, 3E)
  uint32_t* rank = G + E;
  K_CUDA(cudaMemsetAsync(is_first, 0, E * 4, st));
  K_CUDA(cudaMalloc(&gfirst.p, (size_t)n * 4));
  K_CUDA(cudaMalloc(&g->key_id, (size_t)n * 4));
  K_CUDA(cudaMalloc(&g->node_first, (size_t)n * 4));
  K_CUDA(cudaMalloc(&klen.p, ((size_t)n + 1) * 8));
  key_first_kernel<<<gbE, KTB, 0, st>>>(P, head, grp_of, E, is_first, gfirst.as<uint32_t>());
  {
    size_t t3 = tmp_bytes;
    cub::DeviceScan::ExclusiveSum(tmp.p, t3, is_first, rank, (int64_t)E, st);
  }
  key_rank_kernel<<<kblocks((uint64_t)n + 1), KTB, 0, st>>>(gfirst.as<uint32_t>(), rank, off, n, g->key_id,
                                                             g->node_first, klen.as<uint64_t>());
  K_CUDA(cudaStreamSynchronize(st));
  release(K);
  release(perm);
  release(perm2);

  // ---- 3. the distinct keys for lookups, in group order ----
  K_CUDA(cudaMalloc(&g->key_off, ((size_t)n + 1) * 8));
  {
    size_t t3 = tmp_bytes;
    cub::DeviceScan::ExclusiveSum(tmp.p, t3, klen.as<uint64_t>(), g->key_off, (int64_t)n + 1, st);
  }
  uint64_t kb = 0;
  K_CUDA(cudaMemcpyAsync(&kb, g->key_off + n, 8, cudaMemcpyDeviceToHost, st));
  K_CUDA(cudaStreamSynchronize(st));
  K_CUDA(cudaMalloc(&g->key_bytes, std::max<uint64_t>(kb, 1)));
  key_copy_kernel<<<kblocks(n), KTB, 0, st>>>(bytes, off, gfirst.as<uint32_t>(), g->key_off, n, g->key_bytes);
  K_CUDA(cudaStreamSynchronize(st));
  release(dbytes);
  release(doff);
  release(gfirst);
  release(klen);
  release(tmp);

  // ---- 4. the dense edge stream -> the CSR of cozo_gpu_graph_stage ----
  DevBuf dsrc, ddst, dw2;
  K_CUDA(cudaMalloc(&dsrc.p, m2 * 4));
  K_CUDA(cudaMalloc(&ddst.p, m2 * 4));
  if (w) K_CUDA(cudaMalloc(&dw2.p, m2 * 4));
  key_edges_kernel<<<kblocks(m), KTB, 0, st>>>(grp_of, g->key_id, dw.as<float>(), m, undirected ? 1 : 0,
                                               dsrc.as<uint32_t>(), ddst.as<uint32_t>(), dw2.as<float>());
  K_CUDA(cudaGetLastError());
  K_CUDA(cudaStreamSynchronize(st));
  release(grp);
  release(dw);
#undef K_CUDA
  rc = graph_build_csr(g, dsrc.as<uint32_t>(), ddst.as<uint32_t>(), dw2.as<float>(), st);
  if (rc) return fail(rc);
  *out_n = n;
  *out = g;
  return 0;
}

extern "C" int cozo_gpu_graph_node_endpoints(cozo_gpu_graph_t* g, uint64_t* out_first) {
  if (!g || (g->n && !out_first)) return set_error(COZO_GPU_EINVAL, "null argument");
  if (!g->keyed) return set_error(COZO_GPU_EINVAL, "the graph was not staged from keys");
  if (g->n == 0) return 0;
  std::vector<uint32_t> h(g->n);
  COZO_CUDA(cudaMemcpy(h.data(), g->node_first, (size_t)g->n * 4, cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < g->n; ++i) out_first[i] = h[i];
  return 0;
}

extern "C" int cozo_gpu_graph_lookup_keys(cozo_gpu_graph_t* g, const uint8_t* key_bytes, const uint64_t* key_off,
                                          uint32_t count, uint32_t* out_ids) {
  if (!g || (count && (!key_bytes || !key_off || !out_ids))) return set_error(COZO_GPU_EINVAL, "null argument");
  if (!g->keyed) return set_error(COZO_GPU_EINVAL, "the graph was not staged from keys");
  if (count == 0) return 0;
  for (uint32_t i = 0; i < count; ++i)
    if (key_off[i + 1] < key_off[i]) return set_error(COZO_GPU_EINVAL, "key offsets decrease");
  if (g->n == 0) {
    std::fill(out_ids, out_ids + count, NONE);
    return 0;
  }
  int rc = ensure_init();
  if (rc) return rc;
  CallStream cs;
  rc = cs.init();
  if (rc) return rc;
  const uint64_t B = key_off[count];
  DevBuf qb, qo, qi;
  COZO_CUDA(cudaMalloc(&qb.p, std::max<uint64_t>(B, 1)));
  COZO_CUDA(cudaMalloc(&qo.p, ((size_t)count + 1) * 8));
  COZO_CUDA(cudaMalloc(&qi.p, (size_t)count * 4));
  if (B) COZO_CUDA(cudaMemcpyAsync(qb.p, key_bytes, B, cudaMemcpyHostToDevice, cs.s));
  COZO_CUDA(cudaMemcpyAsync(qo.p, key_off, ((size_t)count + 1) * 8, cudaMemcpyHostToDevice, cs.s));
  key_lookup_kernel<<<kblocks(count), KTB, 0, cs.s>>>(g->key_bytes, g->key_off, g->key_id, g->n, qb.as<uint8_t>(),
                                                      qo.as<uint64_t>(), count, qi.as<uint32_t>());
  COZO_CUDA(cudaGetLastError());
  COZO_CUDA(cudaMemcpyAsync(out_ids, qi.p, (size_t)count * 4, cudaMemcpyDeviceToHost, cs.s));
  COZO_CUDA(cudaStreamSynchronize(cs.s));
  return 0;
}
