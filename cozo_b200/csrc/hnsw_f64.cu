// hnsw_f64.cu — batched k-NN search on an F64 vector index (manifest.dtype == VecElementType::F64).
//
// The reference computes distances of F64 vectors in f64 throughout (runtime/hnsw.rs:73-76, 86-93, 102-107) and
// casts the query to the index dtype first (hnsw.rs:879-884).  This is hnsw_search_level / hnsw_knn (hnsw.rs:539-587,
// 869-1012) on `double`: one warp per query, the query and the sorted found/candidate array (f64 keys) in shared
// memory, rows read with coalesced 8-byte loads.  The beam routines and the epilogue walk are the f32 search's
// (hnsw_device.cuh); the scoring (dist64), the params and the result store are its own, so the f32 kernels' register
// and shared-memory budget stay untouched.  It shares the graph layout, the visited bitmaps and the workspace pool with
// the f32 path.  F64 indexes are search-only on the device (maintenance re-stages).
#include <algorithm>

#include "hnsw_host.hpp"

namespace cozo {

struct Search64Params {
  const double* queries;
  const double* vec64;  // [n x ld64]
  uint32_t ld64;
  uint32_t B, k, ef;
  int has_radius;
  double radius;
  uint32_t* out_ids;
  double* out_dist;
  uint32_t* out_count;
  uint32_t* qstats;
  uint32_t* counter;
  uint32_t* vis;
  uint32_t nwords;
  uint32_t* vlog;
  uint32_t logcap;
  uint32_t warp_smem, off_fi, off_pend, off_q;
  const uint32_t* filter_mask;
  // fused exchange of the sharded corpus, as in SearchParams: besides (or instead of) out_ids/out_dist the top-k of
  // query qi is stored into every destination's [n_slots][B][k] gather buffer at slot `slot`
  uint32_t n_dest, slot;
  uint32_t* dest_ids[COZO_GPU_MAX_PEERS];
  double* dest_dist[COZO_GPU_MAX_PEERS];
};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// VectorCache::dist for (F64, F64) operands
template <int METRIC>
__device__ __forceinline__ double dist64(const double* q, const double* __restrict__ row, uint32_t dim, int lane,
                                         double qnorm) {
  double a = 0.0, b = 0.0;
#pragma unroll 4
  for (uint32_t i = lane; i < dim; i += 32) {
    const double x = q[i], y = __ldg(row + i);
    if (METRIC == COZO_GPU_L2) {
      const double d = x - y;
      a = fma(d, d, a);
    } else {
      a = fma(x, y, a);
      if (METRIC == COZO_GPU_COSINE) b = fma(y, y, b);
    }
  }
  a = warp_sum_f64(a);
  if (METRIC == COZO_GPU_L2) return a;
  if (METRIC == COZO_GPU_IP) return 1.0 - a;
  b = warp_sum_f64(b);
  return 1.0 - a / sqrt(qnorm * b);
}

template <int METRIC>
__device__ __forceinline__ void search_level64(const HnswDev& g, const Search64Params& p, WarpCtx& w, double* fd,
                                               const double* q, double qnorm, uint32_t ef, uint32_t level, int lane) {
  seed_visited(w, lane);
  const uint32_t stride = level == 0 ? g.s0 : g.su;
  for (;;) {
    uint32_t cand;
    if (!pop_candidate(g, w, level, lane, cand)) break;
    const uint32_t* row = neighbour_row(g, cand, level);
    for (uint32_t nb = 0; nb < stride; nb += 32) {
      uint32_t id = __ldg(row + nb + lane);
      uint32_t validmask = __ballot_sync(0xffffffffu, id != NONE);
      if (!validmask) break;
      w.nbr_reads += __popc(validmask);
      const uint32_t cnt = take_unvisited(w, id, lane, w.pend);
      __syncwarp();
      for (uint32_t c = 0; c < cnt; ++c) {
        const uint32_t nid = w.pend[c];
        const double d = dist64<METRIC>(q, p.vec64 + (size_t)nid * p.ld64, g.dim, lane, qnorm);
        __syncwarp();
        admit(w, fd, ef, d, nid, lane);
      }
      __syncwarp();
    }
  }
  visit_clear(w, lane);
}

// result i of query qi: into out_ids/out_dist, and into every destination's gather buffer.  out_ids/out_dist are
// always written: testing them for null next to the destination loop makes ptxas spill.
__device__ __forceinline__ void store64(const Search64Params& p, uint32_t qi, uint32_t i, uint32_t oid, double od) {
  p.out_ids[(size_t)qi * p.k + i] = oid;
  p.out_dist[(size_t)qi * p.k + i] = od;
  const size_t at = ((size_t)p.slot * p.B + qi) * p.k + i;
  for (uint32_t d = 0; d < p.n_dest; ++d) {  // the all-gather, fused into the epilogue
    p.dest_ids[d][at] = oid;
    p.dest_dist[d][at] = od;
  }
}

template <int METRIC>
__global__ void __launch_bounds__(128) hnsw_search_f64_kernel(HnswDev g, Search64Params p) {
  extern __shared__ __align__(16) uint8_t smem64[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpc = blockDim.x >> 5;
  uint8_t* base = smem64 + (size_t)warp * p.warp_smem;
  double* fd = reinterpret_cast<double*>(base);
  double* q = reinterpret_cast<double*>(base + p.off_q);
  WarpCtx w;
  w.fd = nullptr;
  w.fi = reinterpret_cast<uint32_t*>(base + p.off_fi);
  w.pend = reinterpret_cast<uint32_t*>(base + p.off_pend);
  w.bars = nullptr;
  w.ring = nullptr;
  const size_t slot = (size_t)blockIdx.x * wpc + warp;
  w.vis = p.vis + slot * p.nwords;
  w.nwords = p.nwords;
  w.vlog = p.vlog + slot * p.logcap;
  w.logcap = p.logcap;
  w.ns = 0;
  w.nlog = 0;
  w.head = 0;
  w.phase = 0;
  for (;;) {
    uint32_t qi = 0;
    if (lane == 0) qi = atomicAdd(p.counter, 1u);
    qi = __shfl_sync(0xffffffffu, qi, 0);
    if (qi >= p.B) break;
    double qn = 0.0;
    for (uint32_t i = lane; i < g.dim; i += 32) {
      const double x = p.queries[(size_t)qi * g.dim + i];
      q[i] = x;
      qn = fma(x, x, qn);
    }
    qn = warp_sum_f64(qn);
    __syncwarp();
    w.len = 0;
    w.cursor = 0;
    w.dist_evals = w.nodes_expanded = w.nbr_reads = 0;
    if (g.entry != NONE) {  // empty index => no rows (hnsw.rs:903-909)
      const double d = dist64<METRIC>(q, p.vec64 + (size_t)g.entry * p.ld64, g.dim, lane, qn);
      w.dist_evals = 1;
      if (lane == 0) {
        fd[0] = d;
        w.fi[0] = g.entry;
      }
      w.len = 1;
      __syncwarp();
      for (uint32_t lvl = g.top_level; lvl >= 1; --lvl) search_level64<METRIC>(g, p, w, fd, q, qn, 1, lvl, lane);
      search_level64<METRIC>(g, p, w, fd, q, qn, p.ef, 0, lane);
    }
    const uint32_t found = emit_results(p, w, fd, lane, g.entry != NONE,
                                        [&](uint32_t i, uint32_t oid, double od) { store64(p, qi, i, oid, od); });
    if (lane == 0) {
      if (p.out_count) p.out_count[qi] = found;
      if (p.qstats) reinterpret_cast<uint4*>(p.qstats)[qi] = make_uint4(w.dist_evals, w.nodes_expanded, w.nbr_reads, 0);
    }
    __syncwarp();
  }
}

}  // namespace cozo

int cozo::hnsw_launch_search_f64(cozo_gpu_hnsw* h, HnswWorkspace* ws, const double* d_q, uint32_t B, uint32_t k,
                                  uint32_t ef, double radius, uint32_t* d_ids, double* d_dist, uint32_t* d_count,
                                  uint32_t* d_qstats, cudaStream_t st, const ScatterDest64* scatter,
                                  const uint32_t* d_filter_mask) {
  const DeviceInfo& di = device_info();
  const HnswDev& g = h->dev;
  Search64Params p{};
  const uint32_t efcap = round_up(ef, 32);
  p.off_fi = efcap * 8;
  p.off_pend = p.off_fi + efcap * 4;
  p.off_q = round_up(p.off_pend + 128, 16);
  p.warp_smem = round_up(p.off_q + g.dim * 8, 16);
  uint32_t wpc = 4;
  size_t smem = (size_t)p.warp_smem * wpc;
  while (smem > di.smem_optin && wpc > 1) {
    wpc >>= 1;
    smem = (size_t)p.warp_smem * wpc;
  }
  if (smem > di.smem_optin)
    return set_error(COZO_GPU_EUNSUP, "ef=%u / dim=%u need %zu B of shared memory per warp (limit %zu)", ef, g.dim, smem,
                     di.smem_optin);
  using K64 = void (*)(HnswDev, Search64Params);
  K64 fn = g.metric == COZO_GPU_L2       ? (K64)hnsw_search_f64_kernel<COZO_GPU_L2>
           : g.metric == COZO_GPU_COSINE ? (K64)hnsw_search_f64_kernel<COZO_GPU_COSINE>
                                         : (K64)hnsw_search_f64_kernel<COZO_GPU_IP>;
  COZO_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)di.smem_optin));
  int cps = 0;
  COZO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, fn, wpc * 32, smem));
  if (cps < 1) return set_error(COZO_GPU_ECUDA, "F64 search kernel does not fit on an SM");
  uint32_t grid = std::min<uint32_t>((uint32_t)di.sm_count * (uint32_t)cps, (B + wpc - 1) / wpc);
  const uint32_t nwords = round_up((g.n + 31) / 32, 4);
  const uint32_t logcap = std::min<uint32_t>(65536u, std::max<uint32_t>(4096u, 64u * ef));
  const size_t slots = (size_t)grid * wpc;
  int rc = hnsw_ws_reserve(ws, slots * nwords, slots * logcap, st);
  if (rc) return rc;
  p.queries = d_q;
  p.vec64 = h->d_vec64;
  p.ld64 = h->ld64;
  p.B = B;
  p.k = k;
  p.ef = ef;
  p.has_radius = radius >= 0.0;
  p.radius = radius;
  p.out_ids = d_ids;
  p.out_dist = d_dist;
  p.out_count = d_count;
  p.qstats = d_qstats;
  p.counter = ws->counter;
  p.vis = ws->vis;
  p.nwords = nwords;
  p.vlog = ws->vlog;
  p.logcap = logcap;
  p.filter_mask = d_filter_mask;
  if (scatter) {
    p.n_dest = scatter->n_dest;
    p.slot = scatter->slot;
    for (uint32_t d = 0; d < scatter->n_dest; ++d) {
      p.dest_ids[d] = scatter->ids[d];
      p.dest_dist[d] = scatter->dist[d];
    }
  }
  COZO_CUDA(cudaMemsetAsync(ws->counter, 0, 4, st));
  fn<<<grid, wpc * 32, smem, st>>>(g, p);
  COZO_CUDA(cudaGetLastError());
  return 0;
}

using namespace cozo;

extern "C" int cozo_gpu_hnsw_search_f64(cozo_gpu_hnsw_t* h, const double* queries, uint32_t B, uint32_t k, uint32_t ef,
                                        double radius, const uint32_t* row_mask, uint32_t* out_ids, double* out_dist,
                                        uint32_t* out_count, CozoGpuSearchStats* stats) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  if (!h->f64) return set_error(COZO_GPU_EINVAL, "not an F64 index: use cozo_gpu_hnsw_search");
  if (k == 0) return set_error(COZO_GPU_EINVAL, "k must be positive");
  if (ef == 0) return set_error(COZO_GPU_EINVAL, "ef must be positive");
  int rc = ensure_init();
  if (rc) return rc;
  return hnsw_search_host(h, queries, B, k, ef, radius, row_mask, out_ids, out_dist, out_count, stats);
}
