// hnsw.cu — staging, batched k-NN search and export of the HBM-resident HNSW
// index.  Replaces SessionTx::hnsw_knn (runtime/hnsw.rs:869-1012) behind
// HnswSearchRA::iter (query/ra.rs:1085-1121); see include/cozo_gpu.h.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "hnsw_host.hpp"

namespace cozo {

struct SearchParams {
  const float* queries;
  uint32_t B, k, ef;
  int has_radius;
  double radius;
  uint32_t* out_ids;
  float* out_dist;
  uint32_t* out_count;
  uint32_t* qstats;
  uint32_t* counter;
  uint32_t* vis;
  uint32_t nwords;
  uint32_t* vlog;
  uint32_t logcap;
  uint32_t ns;
  uint32_t warp_smem;  // bytes of shared memory per warp
  uint32_t off_fi, off_pend, off_bars, off_ring;
  uint32_t cns, off_cbars, off_cring;  // code ring of the pruned search (cns = 0: none)
  // fused exchange of the sharded corpus: besides (or instead of) out_ids/out_dist the top-k of
  // query qi is stored into every destination's [n_slots][B][k] gather buffer at slot `slot`;
  // destinations are peer GPUs' buffers mapped over NVLink (plain st.global on peer pointers).
  // per-row filter verdicts (bit id = the row passes): applied to the final beam BEFORE the trim to k,
  // like the filter bytecode of hnsw_knn (hnsw.rs:943-947, 997-1006); nullptr = no filter
  const uint32_t* filter_mask;
  uint32_t n_dest, slot;
  uint32_t* dest_ids[COZO_GPU_MAX_PEERS];
  float* dest_dist[COZO_GPU_MAX_PEERS];
  uint32_t off_qcodes;  // the pruned search's fixed-point query (QueryCodes::a)
  uint32_t off_query;   // wide kernels (NV = 0): the query, zero padded to ld (per warp; per CTA in the cooperative one)
};


// hnsw_knn's tail (hnsw.rs:943-956, 997-1006) for the query of this warp: walk the beam nearest first, drop
// `dist > radius` and rows the filter rejects, keep the first k, pad the rest.  Without a filter the beam is cut to k
// before the radius test, and without either the kept entries are a prefix of the sorted array.  A radius does not
// keep a prefix: NaN keys sort last and pass it (`NaN > r` is false).  Returns the number of results.
__device__ __forceinline__ uint32_t emit_results(const SearchParams& p, const WarpCtx& w, uint32_t qi, int lane,
                                                 bool searched) {
  auto store = [&](uint32_t i, uint32_t oid, float od) {
    if (p.out_ids) {
      p.out_ids[(size_t)qi * p.k + i] = oid;
      p.out_dist[(size_t)qi * p.k + i] = od;
    }
    const size_t at = ((size_t)p.slot * p.B + qi) * p.k + i;
    for (uint32_t d = 0; d < p.n_dest; ++d) {  // the all-gather, fused into the epilogue
      p.dest_ids[d][at] = oid;
      p.dest_dist[d][at] = od;
    }
  };
  uint32_t found = 0;
  if (searched && !p.filter_mask && !p.has_radius) {
    found = w.len < p.k ? w.len : p.k;
    for (uint32_t i = lane; i < found; i += 32) store(i, w.fi[i] & IDMASK, w.fd[i]);
  } else if (searched) {
    const uint32_t lim = p.filter_mask || w.len < p.k ? w.len : p.k;
    for (uint32_t base_i = 0; base_i < lim && found < p.k; base_i += 32) {
      const uint32_t i = base_i + lane;
      bool ok = i < lim;
      uint32_t id = 0;
      float d = 0.f;
      if (ok) {
        id = w.fi[i] & IDMASK;
        d = w.fd[i];
        ok = (!p.filter_mask || ((p.filter_mask[id >> 5] >> (id & 31)) & 1u)) && !(p.has_radius && (double)d > p.radius);
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, ok);
      const uint32_t pos = found + __popc(bal & ((1u << lane) - 1));
      if (ok && pos < p.k) store(pos, id, d);
      found += __popc(bal);
    }
    if (found > p.k) found = p.k;
  }
  for (uint32_t i = found + lane; i < p.k; i += 32) store(i, NONE, INFINITY);
  return found;
}

#ifdef COZO_HOP_CLOCKS
// tools/hop_clocks.py: the per-phase totals of every warp of the warp-per-query search since the last read
__device__ unsigned long long g_hop_clocks[HC_N];
extern "C" int cozo_gpu_hop_clocks(unsigned long long* out) {
  COZO_CUDA(cudaMemcpyFromSymbol(out, g_hop_clocks, sizeof(g_hop_clocks)));
  static const unsigned long long zero[HC_N] = {};
  COZO_CUDA(cudaMemcpyToSymbol(g_hop_clocks, zero, sizeof(zero)));
  return 0;
}
#endif

// One warp per query, persistent CTAs pulling query indices from a counter.
// MINB = resident CTAs per SM the register allocation is capped for (4 warps per CTA).
template <int NV, int METRIC, bool BULK, int MINB>
__global__ void __launch_bounds__(128, MINB) hnsw_search_kernel(HnswDev g, SearchParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpc = blockDim.x >> 5;
  uint8_t* base = smem + (size_t)warp * p.warp_smem;
  WarpCtx w;
  w.fd = reinterpret_cast<float*>(base);
  w.fi = reinterpret_cast<uint32_t*>(base + p.off_fi);
  w.pend = reinterpret_cast<uint32_t*>(base + p.off_pend);
  w.bars = reinterpret_cast<uint64_t*>(base + p.off_bars);
  w.ring = reinterpret_cast<float*>(base + p.off_ring);
  const size_t slot = (size_t)blockIdx.x * wpc + warp;
  w.vis = p.vis + slot * p.nwords;
  w.nwords = p.nwords;
  w.vlog = p.vlog + slot * p.logcap;
  w.logcap = p.logcap;
  w.ns = p.ns;
  w.nlog = 0;
  w.head = 0;
  w.phase = 0;
  w.cring = base + p.off_cring;
  w.cbars = reinterpret_cast<uint64_t*>(base + p.off_cbars);
  w.cns = p.cns;
  w.chead = 0;
  w.cphase = 0;
#ifdef COZO_HOP_CLOCKS
  for (int k = 0; k < HC_N; ++k) w.clk[k] = 0;
#endif
  if (BULK) {
    if (lane == 0) {
      for (uint32_t s = 0; s < p.ns; ++s) mbar_init(&w.bars[s], 1);
      for (uint32_t s = 0; s < p.cns; ++s) mbar_init(&w.cbars[s], 1);
      mbar_fence_init();
    }
    __syncwarp();
  }
  const int nvec4 = g.ld >> 2;
  // at run time: only if g.codes is set (then p.cns > 0); wide rows carry no codes
  constexpr bool PRUNE = BULK && METRIC == COZO_GPU_L2 && NV > 0;

  for (;;) {
    uint32_t qi = 0;
    if (lane == 0) qi = atomicAdd(p.counter, 1u);
    qi = __shfl_sync(0xffffffffu, qi, 0);
    if (qi >= p.B) break;
    typename QueryOf<NV>::type q;
    float qnorm;
    if constexpr (NV == 0)
      load_query_wide(p.queries + (size_t)qi * g.dim, g.dim, lane, reinterpret_cast<float4*>(base + p.off_query), true,
                      q, qnorm);
    else
      load_query<NV>(p.queries + (size_t)qi * g.dim, g.dim, lane, q, qnorm);
    QueryCodes qc;
    qc.a = reinterpret_cast<QueryPair*>(base + p.off_qcodes);
    if constexpr (PRUNE) {
      if (g.codes) load_query_codes<NV>(q, g.ld, lane, qc);
    }
    w.len = 0;
    w.cursor = 0;
    w.dist_evals = w.nodes_expanded = w.nbr_reads = w.pruned = 0;
    uint32_t found = 0;
    if (g.entry != NONE) {  // empty index => no rows (hnsw.rs:903-909)
      // entry point distance (hnsw.rs:915-918)
      float d = dist_ldg1<NV, METRIC>(q, reinterpret_cast<const float4*>(g.vec + (size_t)g.entry * g.ld), lane, nvec4,
                                      qnorm);
      w.dist_evals = 1;
      if (lane == 0) {
        w.fd[0] = d;
        w.fi[0] = g.entry;
      }
      w.len = 1;
      __syncwarp();
      for (uint32_t lvl = g.top_level; lvl >= 1; --lvl)  // hnsw.rs:919-929
        search_level<NV, METRIC, BULK, PRUNE>(g, w, q, qnorm, 1, lvl, lane, &qc);
      search_level<NV, METRIC, BULK, PRUNE>(g, w, q, qnorm, p.ef, 0, lane, &qc);  // hnsw.rs:930-938
    }
    found = emit_results(p, w, qi, lane, g.entry != NONE);
    if (lane == 0) {
      if (p.out_count) p.out_count[qi] = found;
      if (p.qstats) {
        uint4 s = make_uint4(w.dist_evals, w.nodes_expanded, w.nbr_reads, w.dist_evals - w.pruned);
        reinterpret_cast<uint4*>(p.qstats)[qi] = s;
      }
    }
    __syncwarp();
  }
#ifdef COZO_HOP_CLOCKS
  if (lane == 0)
    for (int k = 0; k < HC_N; ++k) atomicAdd(&g_hop_clocks[k], w.clk[k]);
#endif
}

using KernelFn = void (*)(HnswDev, SearchParams);

// Cooperative form: one CTA (4 warps) per query; see coop_search_level.  Shared memory per CTA:
// [fd ef][fi ef][pend 32][pdist 32][ctrl 8] then per warp [bars ns][ring ns rows].  The wide form (NV = 0) keeps its
// query between the two: [ctrl 8][query ld][per warp ...].
template <int NV, int METRIC>
__global__ void __launch_bounds__(128, 4) hnsw_search_coop_kernel(HnswDev g, SearchParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  WarpCtx w;
  w.fd = reinterpret_cast<float*>(smem);
  w.fi = reinterpret_cast<uint32_t*>(smem + p.off_fi);
  w.pend = nullptr;
  CoopShared cs;
  cs.pend = reinterpret_cast<uint32_t*>(smem + p.off_pend);
  cs.pdist = reinterpret_cast<float*>(smem + p.off_pend + 128);
  cs.ctrl = reinterpret_cast<uint32_t*>(smem + p.off_pend + 256);
  uint8_t* wbase = smem + p.off_bars + (size_t)warp * p.warp_smem;  // off_bars = start of the per-warp region
  w.bars = reinterpret_cast<uint64_t*>(wbase);
  w.ring = reinterpret_cast<float*>(wbase + p.off_ring);            // off_ring = ring offset inside the region
  const size_t slot = blockIdx.x;
  w.vis = p.vis + slot * p.nwords;
  w.nwords = p.nwords;
  w.vlog = p.vlog + slot * p.logcap;
  w.logcap = p.logcap;
  w.ns = p.ns;
  w.nlog = 0;
  w.head = 0;
  w.phase = 0;
  w.len = 0;
  w.cursor = 0;
  if (lane == 0) {
    for (uint32_t s = 0; s < p.ns; ++s) mbar_init(&w.bars[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  const int nvec4 = g.ld >> 2;
  for (;;) {
    if (threadIdx.x == 0) cs.ctrl[1] = atomicAdd(p.counter, 1u);
    __syncthreads();
    const uint32_t qi = cs.ctrl[1];
    __syncthreads();
    if (qi >= p.B) break;
    typename QueryOf<NV>::type q;
    float qnorm;
    if constexpr (NV == 0)  // one copy per CTA, written by warp 0; every warp sums the norm itself
      load_query_wide(p.queries + (size_t)qi * g.dim, g.dim, lane, reinterpret_cast<float4*>(smem + p.off_query),
                      warp == 0, q, qnorm);
    else
      load_query<NV>(p.queries + (size_t)qi * g.dim, g.dim, lane, q, qnorm);
    w.len = 0;
    w.cursor = 0;
    w.dist_evals = w.nodes_expanded = w.nbr_reads = 0;
    uint32_t found = 0;
    if (g.entry != NONE) {
      if (warp == 0) {
        float d = dist_ldg1<NV, METRIC>(q, reinterpret_cast<const float4*>(g.vec + (size_t)g.entry * g.ld), lane,
                                        nvec4, qnorm);
        w.dist_evals = 1;
        if (lane == 0) {
          w.fd[0] = d;
          w.fi[0] = g.entry;
        }
        w.len = 1;
      }
      __syncthreads();
      for (uint32_t lvl = g.top_level; lvl >= 1; --lvl)
        coop_search_level<NV, METRIC>(g, w, cs, q, qnorm, 1, lvl, lane, warp);
      coop_search_level<NV, METRIC>(g, w, cs, q, qnorm, p.ef, 0, lane, warp);
    }
    if (warp == 0) {
      found = emit_results(p, w, qi, lane, g.entry != NONE);
      if (lane == 0) {
        if (p.out_count) p.out_count[qi] = found;
        if (p.qstats)  // every evaluated row is fetched: the fourth word equals dist_evals
          reinterpret_cast<uint4*>(p.qstats)[qi] = make_uint4(w.dist_evals, w.nodes_expanded, w.nbr_reads, w.dist_evals);
      }
    }
    __syncthreads();
  }
}

template <int NV>
static KernelFn pick_coop_metric(int metric) {
  switch (metric) {
    case COZO_GPU_L2: return hnsw_search_coop_kernel<NV, COZO_GPU_L2>;
    case COZO_GPU_COSINE: return hnsw_search_coop_kernel<NV, COZO_GPU_COSINE>;
    default: return hnsw_search_coop_kernel<NV, COZO_GPU_IP>;
  }
}
static KernelFn pick_coop_kernel(uint32_t ld, int metric) {
  uint32_t need = (ld / 4 + 31) / 32;
  if (need <= 1) return pick_coop_metric<1>(metric);
  if (need <= 2) return pick_coop_metric<2>(metric);
  if (need <= 4) return pick_coop_metric<4>(metric);
  if (need <= 6) return pick_coop_metric<6>(metric);
  if (need <= 8) return pick_coop_metric<8>(metric);
  if (need <= 16) return pick_coop_metric<16>(metric);
  return pick_coop_metric<0>(metric);
}



template <int NV, int MINB>
static KernelFn pick_metric(int metric, bool bulk) {
  switch (metric) {
    case COZO_GPU_L2:
      return bulk ? hnsw_search_kernel<NV, COZO_GPU_L2, true, MINB> : hnsw_search_kernel<NV, COZO_GPU_L2, false, 4>;
    case COZO_GPU_COSINE:
      return bulk ? hnsw_search_kernel<NV, COZO_GPU_COSINE, true, MINB>
                  : hnsw_search_kernel<NV, COZO_GPU_COSINE, false, 4>;
    default:
      return bulk ? hnsw_search_kernel<NV, COZO_GPU_IP, true, MINB> : hnsw_search_kernel<NV, COZO_GPU_IP, false, 4>;
  }
}

template <int MINB>
static KernelFn pick_nv(uint32_t need, int metric, bool bulk) {
  if (need <= 1) return pick_metric<1, MINB>(metric, bulk);
  if (need <= 2) return pick_metric<2, MINB>(metric, bulk);
  if (need <= 4) return pick_metric<4, MINB>(metric, bulk);
  if (need <= 6) return pick_metric<6, MINB>(metric, bulk);
  if (need <= 8) return pick_metric<8, MINB>(metric, bulk);
  if (need <= 16) return pick_metric<16, MINB>(metric, bulk);
  return pick_metric<0, MINB>(metric, bulk);
}

// 4 CTAs x 4 warps per SM (<= 128 registers).  The batch is bandwidth-bound; builds capped for more resident
// warps buy occupancy with tighter register budgets, which cost instructions (tools/sweep.py compares them).
static KernelFn pick_kernel(uint32_t ld, int metric, bool bulk) {
  uint32_t need = (ld / 4 + 31) / 32;
  return pick_nv<4>(need, metric, bulk);
}

static HnswWorkspace* new_ws();
void hnsw_prewarm_pool(cozo_gpu_hnsw* h, size_t vis_words, size_t vlog_words);

// `stream` is the stream the next kernel using this workspace is launched on: a fresh bitmap is zeroed
// there, i.e. ordered before that kernel (the legacy default stream does not order work of a
// cudaStreamNonBlocking stream).
int hnsw_ws_reserve(HnswWorkspace* ws, size_t vis_words, size_t vlog_words, cudaStream_t stream) {
  if (ws->vis_words < vis_words) {
    if (ws->vis) {
      COZO_CUDA(cudaStreamSynchronize(stream));  // nothing may still read the old bitmap
      cudaFree(ws->vis);
    }
    ws->vis = nullptr;
    ws->vis_words = 0;
    COZO_CUDA(cudaMalloc(&ws->vis, vis_words * 4));
    COZO_CUDA(cudaMemsetAsync(ws->vis, 0, vis_words * 4, stream));
    ws->vis_words = vis_words;
  }
  if (ws->vlog_words < vlog_words) {
    if (ws->vlog) cudaFree(ws->vlog);
    ws->vlog = nullptr;
    ws->vlog_words = 0;
    COZO_CUDA(cudaMalloc(&ws->vlog, vlog_words * 4));
    ws->vlog_words = vlog_words;
  }
  return 0;
}

// Each in-flight search owns one workspace (visited bitmaps are n/8 bytes per resident warp).
// At most "hnsw.max_workspaces" (default 3) exist per index; further callers wait for a
// release instead of allocating hundreds of MB inside the hot path.
HnswWorkspace* hnsw_acquire_ws(cozo_gpu_hnsw* h) {
  {
    std::unique_lock<std::mutex> lk(h->mu);
    const uint32_t cap = (uint32_t)std::max<int64_t>(1, get_option("hnsw.max_workspaces", 3));
    h->cv.wait(lk, [&] { return !h->pool.empty() || h->n_workspaces < cap; });
    if (!h->pool.empty()) {
      HnswWorkspace* ws = h->pool.back();
      h->pool.pop_back();
      return ws;
    }
    h->n_workspaces++;
  }
  HnswWorkspace* ws = new_ws();
  if (!ws) {
    std::lock_guard<std::mutex> lk(h->mu);
    h->n_workspaces--;
    h->cv.notify_one();
    return nullptr;
  }
  return ws;
}

static HnswWorkspace* new_ws() {
  auto* ws = new HnswWorkspace();
  if (cudaStreamCreateWithFlags(&ws->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&ws->e0) != cudaSuccess || cudaEventCreate(&ws->e1) != cudaSuccess ||
      cudaMalloc(&ws->counter, 256) != cudaSuccess) {
    set_error(COZO_GPU_ECUDA, "workspace creation failed: %s", cudaGetErrorString(cudaGetLastError()));
    delete ws;
    return nullptr;
  }
  return ws;
}

// Create the remaining workspaces of the pool with the sizes the first search needed, so that
// back-to-back asynchronous calls never allocate (cudaMalloc/cudaMemset serialise the device).
void hnsw_prewarm_pool(cozo_gpu_hnsw* h, size_t vis_words, size_t vlog_words) {
  const uint32_t cap = (uint32_t)std::max<int64_t>(1, get_option("hnsw.max_workspaces", 3));
  for (;;) {
    {
      std::lock_guard<std::mutex> lk(h->mu);
      if (h->n_workspaces >= cap) return;
      h->n_workspaces++;
    }
    HnswWorkspace* ws = new_ws();
    // zeroed on the workspace's own stream and waited for: whichever stream uses it later sees zeros
    if (!ws || hnsw_ws_reserve(ws, vis_words, vlog_words, ws->stream) != 0 ||
        cudaStreamSynchronize(ws->stream) != cudaSuccess) {
      if (ws) hnsw_release_ws(h, ws);  // usable, just not pre-sized
      else {
        std::lock_guard<std::mutex> lk(h->mu);
        h->n_workspaces--;
      }
      return;
    }
    hnsw_release_ws(h, ws);
  }
}

void hnsw_release_ws(cozo_gpu_hnsw* h, HnswWorkspace* ws) {
  {
    std::lock_guard<std::mutex> lk(h->mu);
    h->pool.push_back(ws);
  }
  h->cv.notify_one();
}

static void free_ws(HnswWorkspace* ws) {
  if (ws->vis) cudaFree(ws->vis);
  if (ws->vlog) cudaFree(ws->vlog);
  if (ws->counter) cudaFree(ws->counter);
  if (ws->q) cudaFree(ws->q);
  if (ws->ids) cudaFree(ws->ids);
  if (ws->dist) cudaFree(ws->dist);
  if (ws->count) cudaFree(ws->count);
  if (ws->qstats) cudaFree(ws->qstats);
  if (ws->mask) cudaFree(ws->mask);
  if (ws->e0) cudaEventDestroy(ws->e0);
  if (ws->e1) cudaEventDestroy(ws->e1);
  if (ws->stream) cudaStreamDestroy(ws->stream);
  delete ws;
}

static void codes_drop(cozo_gpu_hnsw* h) {
  if (h->d_codes) cudaFree(h->d_codes);
  h->d_codes = nullptr;
  h->codes_rows = 0;
  h->codes_failed = true;
  h->dev.codes = nullptr;
}

// Room for `rows` code rows, keeping rows [0, n).  Only L2 f32 indexes with CODES_MIN_LD <= ld <= 2048 carry codes.  A failed
// allocation leaves
// the index without codes: it is then searched without pruning, with the same results.
void hnsw_codes_reserve(cozo_gpu_hnsw* h, uint32_t rows) {
  HnswDev& g = h->dev;
  // the pruning bound (hnsw_codes.cuh) is argued for ld <= REG_QUERY_MAX_LD, and the wide kernels do not prune
  if (h->f64 || g.metric != COZO_GPU_L2 || g.ld < CODES_MIN_LD || g.ld > REG_QUERY_MAX_LD || h->codes_failed ||
      rows <= h->codes_rows)
    return;
  uint8_t* nc = nullptr;
  if (cudaMalloc(&nc, (size_t)rows * g.code_ld) != cudaSuccess) {
    cudaGetLastError();  // not sticky: clear it
    codes_drop(h);
    return;
  }
  if (h->d_codes && g.n && cudaMemcpy(nc, h->d_codes, (size_t)g.n * g.code_ld, cudaMemcpyDeviceToDevice) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(nc);
    codes_drop(h);
    return;
  }
  if (h->d_codes) cudaFree(h->d_codes);
  h->d_codes = nc;
  h->codes_rows = rows;
  g.codes = nc;
}

// Re-quantise the code rows of the vector rows just written (ids = nullptr: rows first .. first+count-1), on the
// default stream, after the writes to d_vec.
void hnsw_codes_fill(cozo_gpu_hnsw* h, uint32_t first, uint32_t count, const uint32_t* d_ids) {
  const HnswDev& g = h->dev;
  if (!g.codes || !count) return;
  quantize_rows_kernel<<<(count + 127) / 128, 128>>>(h->d_vec, g.ld, h->d_codes, d_ids, first, count);
  if (cudaGetLastError() != cudaSuccess) codes_drop(h);
}

int hnsw_launch_search(cozo_gpu_hnsw* h, HnswWorkspace* ws, const float* d_q, uint32_t B, uint32_t k, uint32_t ef,
                       double radius, uint32_t* d_ids, float* d_dist, uint32_t* d_count, uint32_t* d_qstats,
                       cudaStream_t stream, const ScatterDest* scatter, const uint32_t* d_filter_mask) {
  const DeviceInfo& di = device_info();
  const HnswDev& g = h->dev;
  if (B == 0) return 0;
  // mode 0: plain ld.global rows, 1: warp per query + TMA ring, 2: CTA per query (cooperative),
  // -1 (default): cooperative when the batch cannot give every resident warp slot a query
  int64_t mode = get_option("hnsw.mode", -1);
  uint32_t ns = (uint32_t)get_option("hnsw.stages", 4);
  if (ns < 1) ns = 1;
  if (ns > 32) ns = 32;
  // the cooperative kernel wins while the batch is below about 1.5 waves of its CTAs (4 resident per SM), the
  // warp-per-query kernel beyond (tools/sweep_batch.py measures the crossover)
  const uint32_t coop_below = (uint32_t)get_option("hnsw.coop_below", (int64_t)di.sm_count * 6);
  const bool auto_mode = mode < 0;
  if (auto_mode) mode = B < coop_below ? 2 : 1;
  SearchParams p{};
  uint32_t efcap = round_up(ef, 32);
  KernelFn fn = nullptr;
  uint32_t wpc = 4, grid = 0;
  size_t smem = 0;
  // Rows wider than the register query (NV = 0 kernels) hold the query in shared memory and start from a ring of
  // WIDE_RING_BYTES per warp; stages are dropped, down to one, only when nothing else makes the block fit.  The
  // cooperative CTA needs the query and a stage for each of its 4 warps (up to ld ~11 500 at ef 200); the default mode
  // takes the warp-per-query kernel (query and one stage: up to ld ~28 000) for wider rows.
  const bool wide = g.ld > REG_QUERY_MAX_LD;
  const uint32_t row_bytes = g.ld * 4, query_bytes = wide ? round_up(row_bytes, 128) : 0;
  if (wide) ns = std::max<uint32_t>(1, std::min<uint32_t>(ns, WIDE_RING_BYTES / row_bytes));
  auto wide_unsup = [&](size_t need) {
    return set_error(COZO_GPU_EUNSUP, "vec_dim %u at ef=%u needs %zu B of shared memory (limit %zu)", g.dim, ef, need,
                     di.smem_optin);
  };
  if (mode == 2) {
    fn = pick_coop_kernel(g.ld, g.metric);
    uint32_t cns = std::min<uint32_t>(ns, 3);  // rows in flight per warp; 4 warps share a query
    p.off_fi = efcap * 4;
    p.off_pend = p.off_fi + efcap * 4;                 // pend | pdist | ctrl : 128 + 128 + 32 bytes
    p.off_query = round_up(p.off_pend + 288, 128);
    p.off_bars = p.off_query + query_bytes;            // start of the per-warp regions
    for (;;) {
      p.off_ring = round_up(cns * 8, 128);               // ring offset inside a warp's region
      p.warp_smem = round_up(p.off_ring + cns * row_bytes, 128);
      smem = (size_t)p.off_bars + (size_t)p.warp_smem * COOP_WARPS;
      if (smem <= di.smem_optin || !wide || cns == 1) break;
      --cns;
    }
    if (smem > di.smem_optin && wide && auto_mode) {
      mode = 1;  // the warp-per-query kernel below
    } else {
      ns = cns;
      if (smem > di.smem_optin) {
        if (wide) return wide_unsup(smem);
        return set_error(COZO_GPU_EUNSUP, "ef=%u needs %zu B of shared memory per CTA (limit %zu)", ef, smem,
                         di.smem_optin);
      }
      // always the device maximum: concurrent callers with different ef / stages never lower each other's limit
      COZO_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)di.smem_optin));
      int cps = 0;
      COZO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, fn, 128, smem));
      if (cps < 1) return set_error(COZO_GPU_ECUDA, "search kernel does not fit on an SM");
      grid = std::min<uint32_t>((uint32_t)di.sm_count * (uint32_t)cps, B);
      wpc = 1;  // one visited bitmap / log per CTA
    }
  }
  if (mode != 2) {
    const bool bulk = mode != 0;
    wpc = (uint32_t)get_option("hnsw.warps_per_cta", 4);
    if (wpc < 1) wpc = 1;
    if (wpc > 4) wpc = 4;  // __launch_bounds__(128, ..)
    if (!bulk) ns = 0;
    fn = pick_kernel(g.ld, g.metric, bulk);
    p.off_fi = efcap * 4;
    p.off_pend = p.off_fi + efcap * 4;
    p.off_bars = p.off_pend + 32 * 4;
    p.off_ring = round_up(p.off_bars + ns * 8, 128);
    p.warp_smem = round_up(p.off_ring + ns * g.ld * 4, 128);
    if (wide) {  // [fd][fi][pend][bars ns][query][ring ns]
      p.off_query = p.off_ring;
      p.off_ring += query_bytes;
      p.warp_smem += query_bytes;
    }
    if (bulk && g.codes) {
      // pruned search (prune_chunk): most rows of a hop never reach the f32 ring, so it keeps at most 2 stages and
      // the code ring takes the rest of the same per-warp budget; the CTAs resident per SM stay what they were.
      // The fixed-point query (QueryCodes, 256 B per 128 elements) is taken from the code ring: at config 2 (D = 768,
      // ef 200) that leaves 2 f32 + 5 code stages (7 before); hnsw.stages=1 (1 + 2) measured 0.9 % slower
      // (tools/sweep.py).
      // [fd][fi][pend][bars ns][code bars <= 16][fixed-point query][f32 ring ns][code ring cns]
      const uint32_t budget = p.warp_smem;
      ns = std::min<uint32_t>(ns, 2);
      p.off_cbars = p.off_bars + ns * 8;
      p.off_qcodes = p.off_cbars + 16 * 8;
      p.off_ring = round_up(p.off_qcodes + (g.ld / 4 + 31) / 32 * 256, 128);
      p.off_cring = p.off_ring + ns * g.ld * 4;  // a multiple of 16: ld is a multiple of 4
      const uint32_t room = budget > p.off_cring ? budget - p.off_cring : 0;
      p.cns = std::min<uint32_t>(16, std::max<uint32_t>(2, room / g.code_ld));
      p.warp_smem = round_up(p.off_cring + p.cns * g.code_ld, 128);
    }
    smem = (size_t)p.warp_smem * wpc;
    while (smem > di.smem_optin && wpc > 1) {
      wpc >>= 1;
      smem = (size_t)p.warp_smem * wpc;
    }
    while (wide && smem > di.smem_optin && ns > 1) {  // one warp: give up ring stages
      --ns;
      p.warp_smem = round_up(p.off_ring + ns * row_bytes, 128);
      smem = p.warp_smem;
    }
    if (wide && smem > di.smem_optin) return wide_unsup(smem);
    if (smem > di.smem_optin)
      return set_error(COZO_GPU_EUNSUP, "ef=%u needs %zu B of shared memory per warp (limit %zu)", ef, smem,
                       di.smem_optin);
    COZO_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)di.smem_optin));
    int ctas_per_sm = 0;
    COZO_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, fn, wpc * 32, smem));
    if (ctas_per_sm < 1) return set_error(COZO_GPU_ECUDA, "search kernel does not fit on an SM");
    int64_t cap = get_option("hnsw.max_ctas_per_sm", 0);
    if (cap > 0 && ctas_per_sm > cap) ctas_per_sm = (int)cap;
    grid = (uint32_t)di.sm_count * (uint32_t)ctas_per_sm;
    uint32_t need = (B + wpc - 1) / wpc;
    if (grid > need) grid = need;
  }
  const uint32_t block_threads = mode == 2 ? 128 : wpc * 32;

  uint32_t nwords = round_up((g.n + 31) / 32, 4);
  uint32_t logcap = std::min<uint32_t>(65536u, std::max<uint32_t>(4096u, 64u * ef));
  size_t slots = (size_t)grid * wpc;
  int rc = hnsw_ws_reserve(ws, slots * nwords, slots * logcap, stream);
  if (rc) return rc;
  hnsw_prewarm_pool(h, slots * nwords, slots * logcap);  // first call only: no allocation in later calls

  p.queries = d_q;
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
  p.ns = ns;
  p.filter_mask = d_filter_mask;
  p.n_dest = 0;
  p.slot = 0;
  if (scatter) {
    p.n_dest = scatter->n_dest;
    p.slot = scatter->slot;
    for (uint32_t d = 0; d < scatter->n_dest; ++d) {
      p.dest_ids[d] = scatter->ids[d];
      p.dest_dist[d] = scatter->dist[d];
    }
  }
  COZO_CUDA(cudaMemsetAsync(ws->counter, 0, 4, stream));
  fn<<<grid, block_threads, smem, stream>>>(g, p);
  COZO_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace cozo

using namespace cozo;

// ---------------------------------------------------------------------------
extern "C" int cozo_gpu_hnsw_stage(cozo_gpu_hnsw_t** out, const CozoGpuHnswStageDesc* d) {
  if (!out || !d) return set_error(COZO_GPU_EINVAL, "null argument");
  *out = nullptr;
  int rc = ensure_init();
  if (rc) return rc;
  if (d->dim == 0 || d->n_levels == 0 || !d->levels || (d->n_vectors && !d->vectors))
    return set_error(COZO_GPU_EINVAL, "bad stage descriptor");
  if (d->metric < 0 || d->metric > 2) return set_error(COZO_GPU_EINVAL, "unknown distance %d", d->metric);
  if (d->n_vectors >= 0x7FFFFFFFu) return set_error(COZO_GPU_EUNSUP, "more than 2^31-1 vectors in one shard");
  if (d->n_levels > 200) return set_error(COZO_GPU_EINVAL, "too many layers");
  const uint32_t n = d->n_vectors;
  if (d->levels[0].n_nodes != n) return set_error(COZO_GPU_EINVAL, "layer 0 must cover all %u vectors", n);
  if (d->entry_point != COZO_GPU_NONE && d->entry_point >= n)
    return set_error(COZO_GPU_EINVAL, "entry point out of range");

  auto* h = new cozo_gpu_hnsw();
  h->n_levels = d->n_levels;
  h->m_max0 = d->m_max0;
  h->m_max = d->m_max;
  h->live.assign(d->n_vectors, 1);
  h->n_live = d->n_vectors;
  HnswDev& g = h->dev;
  g.n = n;
  g.dim = d->dim;
  g.ld = round_up(d->dim, 4);
  g.metric = d->metric;
  g.entry = d->entry_point;
  g.top_level = d->n_levels - 1;

  // strides: observed max degree, at least the manifest bound
  // (row pointers come from the caller: a decreasing pair would wrap into an absurd stride below)
  constexpr uint32_t kMaxStagedDegree = 65536;
  uint32_t maxdeg0 = d->m_max0;
  {
    const CozoGpuHnswLevel& l0 = d->levels[0];
    for (uint32_t i = 0; i < n; ++i) {
      if (l0.row_ptr[i + 1] < l0.row_ptr[i] || l0.row_ptr[i + 1] - l0.row_ptr[i] > kMaxStagedDegree) {
        delete h;
        return set_error(COZO_GPU_EINVAL, "layer 0: row_ptr must be non-decreasing with at most %u neighbours per row (row %u)",
                         kMaxStagedDegree, i);
      }
      maxdeg0 = std::max<uint32_t>(maxdeg0, (uint32_t)(l0.row_ptr[i + 1] - l0.row_ptr[i]));
    }
  }
  uint32_t maxdegu = d->m_max;
  for (uint32_t L = 1; L < d->n_levels; ++L) {
    const CozoGpuHnswLevel& lv = d->levels[L];
    if (!lv.node_ids) {
      delete h;
      return set_error(COZO_GPU_EINVAL, "layer -%u needs node_ids", L);
    }
    for (uint32_t i = 0; i < lv.n_nodes; ++i) {
      if (lv.row_ptr[i + 1] < lv.row_ptr[i] || lv.row_ptr[i + 1] - lv.row_ptr[i] > kMaxStagedDegree) {
        delete h;
        return set_error(COZO_GPU_EINVAL, "layer -%u: row_ptr must be non-decreasing with at most %u neighbours per row (row %u)", L,
                         kMaxStagedDegree, i);
      }
      maxdegu = std::max<uint32_t>(maxdegu, (uint32_t)(lv.row_ptr[i + 1] - lv.row_ptr[i]));
    }
  }
  g.s0 = round_up(std::max(maxdeg0, 1u), 32);
  g.su = round_up(std::max(maxdegu, 1u), 32);

  // node -> top layer
  h->node_level.assign(n, 0);
  for (uint32_t L = 1; L < d->n_levels; ++L) {
    const CozoGpuHnswLevel& lv = d->levels[L];
    for (uint32_t i = 0; i < lv.n_nodes; ++i) {
      uint32_t id = lv.node_ids[i];
      if (id >= n || h->node_level[id] != L - 1) {
        delete h;
        return set_error(COZO_GPU_EINVAL, "node %u on layer -%u is missing from layer -%u", id, L, L - 1);
      }
      h->node_level[id] = (uint8_t)L;
    }
  }
  if (g.entry != NONE && h->node_level[g.entry] != g.top_level) {
    delete h;
    return set_error(COZO_GPU_EINVAL, "entry point must live on the top layer");
  }
  std::vector<uint32_t> upper_off(n, NONE);
  uint64_t up_rows = 0;
  for (uint32_t i = 0; i < n; ++i)
    if (h->node_level[i]) {
      upper_off[i] = (uint32_t)up_rows;
      up_rows += h->node_level[i];
    }
  h->up_rows = up_rows;

  auto fail = [&](int code) {
    cozo_gpu_hnsw_free(h);
    return code;
  };
#define STAGE_CUDA(call)                                                                              \
  do {                                                                                                \
    cudaError_t _e = (call);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      return fail(set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,        \
                            "%s failed: %s", #call, cudaGetErrorString(_e)));                         \
  } while (0)

  // vectors
  if (d->vec_dtype != 0 && d->vec_dtype != 1) return fail(set_error(COZO_GPU_EINVAL, "unknown vec_dtype %d", d->vec_dtype));
  if (d->vec_dtype == 1) {  // VecElementType::F64: f64 payloads, searched in f64 (hnsw.rs:73-76, 86-93, 102-107)
    h->f64 = true;
    h->ld64 = round_up(d->dim, 2);
    if (n) {
      STAGE_CUDA(cudaMalloc(&h->d_vec64, (size_t)n * h->ld64 * 8));
      if (h->ld64 != g.dim) STAGE_CUDA(cudaMemset(h->d_vec64, 0, (size_t)n * h->ld64 * 8));
      STAGE_CUDA(cudaMemcpy2D(h->d_vec64, (size_t)h->ld64 * 8, d->vectors, (size_t)g.dim * 8, (size_t)g.dim * 8, n,
                              d->vectors_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    }
  } else if (n) {
    STAGE_CUDA(cudaMalloc(&h->d_vec, (size_t)n * g.ld * 4));
    if (g.ld != g.dim) STAGE_CUDA(cudaMemset(h->d_vec, 0, (size_t)n * g.ld * 4));
    STAGE_CUDA(cudaMemcpy2D(h->d_vec, (size_t)g.ld * 4, d->vectors, (size_t)g.dim * 4, (size_t)g.dim * 4, n,
                            d->vectors_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  }
  g.vec = h->d_vec;
  g.code_ld = code_row_bytes(g.ld);
  hnsw_codes_reserve(h, n);
  hnsw_codes_fill(h, 0, n);
  // layer 0 adjacency
  {
    std::vector<uint32_t> adj((size_t)n * g.s0, NONE);
    const CozoGpuHnswLevel& l0 = d->levels[0];
    for (uint32_t i = 0; i < n; ++i) {
      uint64_t b = l0.row_ptr[i], e = l0.row_ptr[i + 1];
      for (uint64_t kx = b; kx < e; ++kx) {
        uint32_t t = l0.col_idx[kx];
        if (t >= n) return fail(set_error(COZO_GPU_EINVAL, "layer 0 edge %u->%u out of range", i, t));
        adj[(size_t)i * g.s0 + (kx - b)] = t;
      }
    }
    if (n) {
      STAGE_CUDA(cudaMalloc(&h->d_adj0, adj.size() * 4));
      STAGE_CUDA(cudaMemcpy(h->d_adj0, adj.data(), adj.size() * 4, cudaMemcpyHostToDevice));
    }
    g.adj0 = h->d_adj0;
  }
  // upper layers
  {
    std::vector<uint32_t> adj((size_t)std::max<uint64_t>(up_rows, 1) * g.su, NONE);
    for (uint32_t L = 1; L < d->n_levels; ++L) {
      const CozoGpuHnswLevel& lv = d->levels[L];
      for (uint32_t i = 0; i < lv.n_nodes; ++i) {
        uint32_t id = lv.node_ids[i];
        uint64_t b = lv.row_ptr[i], e = lv.row_ptr[i + 1];
        size_t row = (size_t)upper_off[id] + (L - 1);
        for (uint64_t kx = b; kx < e; ++kx) {
          uint32_t t = lv.col_idx[kx];
          if (t >= n || h->node_level[t] < L)
            return fail(set_error(COZO_GPU_EINVAL, "layer -%u edge %u->%u leaves the layer", L, id, t));
          adj[row * g.su + (kx - b)] = t;
        }
      }
    }
    STAGE_CUDA(cudaMalloc(&h->d_adj_up, adj.size() * 4));
    STAGE_CUDA(cudaMemcpy(h->d_adj_up, adj.data(), adj.size() * 4, cudaMemcpyHostToDevice));
    STAGE_CUDA(cudaMalloc(&h->d_upper_off, (size_t)std::max(n, 1u) * 4));
    if (n) STAGE_CUDA(cudaMemcpy(h->d_upper_off, upper_off.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    g.adj_up = h->d_adj_up;
    g.upper_off = h->d_upper_off;
  }
#undef STAGE_CUDA
  *out = h;
  return 0;
}

extern "C" void cozo_gpu_hnsw_free(cozo_gpu_hnsw_t* h) {
  if (!h) return;
  for (auto* ws : h->pool) free_ws(ws);
  const auto arrays = row_arrays(h);
  for (size_t i = 0; i < arrays.size(); ++i)
    if (arrays[i].ptr && (i != kVecArray || h->vec_owned)) cudaFree(arrays[i].ptr);
  if (h->d_vec64) cudaFree(h->d_vec64);
  delete h;
}

static int check_search_args(cozo_gpu_hnsw_t* h, uint32_t k, uint32_t ef) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  if (h->f64) return set_error(COZO_GPU_EINVAL, "F64 index: use cozo_gpu_hnsw_search_f64");
  // SearchInput::normalize_hnsw rejects k<=0 / ef<=0 (data/program.rs:1341-1569)
  if (k == 0) return set_error(COZO_GPU_EINVAL, "k must be positive");
  if (ef == 0) return set_error(COZO_GPU_EINVAL, "ef must be positive");
  return 0;
}

int cozo::hnsw_search_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k, uint32_t ef,
                          double radius, uint32_t* out_ids_dev, float* out_dist_dev, uint32_t* out_count_dev,
                          uint32_t* per_query_stats_dev, void* stream, const ScatterDest* scatter,
                          const uint32_t* filter_mask_dev) {
  int rc = check_search_args(h, k, ef);
  if (rc) return rc;
  if (B && !queries_dev) return set_error(COZO_GPU_EINVAL, "null buffer");
  if (B && !scatter && (!out_ids_dev || !out_dist_dev)) return set_error(COZO_GPU_EINVAL, "null buffer");
  if ((out_ids_dev == nullptr) != (out_dist_dev == nullptr)) return set_error(COZO_GPU_EINVAL, "ids/dist must come together");
  HnswWorkspace* ws = hnsw_acquire_ws(h);
  if (!ws) return COZO_GPU_ECUDA;
  rc = hnsw_launch_search(h, ws, queries_dev, B, k, ef, radius, out_ids_dev, out_dist_dev, out_count_dev,
                          per_query_stats_dev, (cudaStream_t)stream, scatter, filter_mask_dev);
  // The workspace (visited bitmaps) stays in use until the kernel ends: hand it
  // back to the pool from a host callback ordered after the kernel on `stream`,
  // which keeps this call asynchronous.
  struct Rel {
    cozo_gpu_hnsw* h;
    HnswWorkspace* ws;
  };
  if (rc == 0) {
    auto* r = new Rel{h, ws};
    cudaError_t e = cudaLaunchHostFunc(
        (cudaStream_t)stream,
        [](void* u) {
          auto* r = static_cast<Rel*>(u);
          hnsw_release_ws(r->h, r->ws);
          delete r;
        },
        r);
    if (e != cudaSuccess) {
      delete r;
      cudaStreamSynchronize((cudaStream_t)stream);
      hnsw_release_ws(h, ws);
      return set_error(COZO_GPU_ECUDA, "cudaLaunchHostFunc failed: %s", cudaGetErrorString(e));
    }
    return 0;
  }
  hnsw_release_ws(h, ws);
  return rc;
}

extern "C" int cozo_gpu_hnsw_search_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k,
                                        uint32_t ef, double radius, uint32_t* out_ids_dev, float* out_dist_dev,
                                        uint32_t* out_count_dev, uint32_t* per_query_stats_dev, void* stream) {
  return hnsw_search_dev(h, queries_dev, B, k, ef, radius, out_ids_dev, out_dist_dev, out_count_dev,
                         per_query_stats_dev, stream, nullptr, nullptr);
}

extern "C" int cozo_gpu_hnsw_search_scatter_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k,
                                                uint32_t ef, double radius, uint32_t n_dest,
                                                const uint64_t* dest_ids_ptrs, const uint64_t* dest_dist_ptrs,
                                                uint32_t slot, uint32_t* per_query_stats_dev, void* stream) {
  if (n_dest == 0 || n_dest > COZO_GPU_MAX_PEERS || !dest_ids_ptrs || !dest_dist_ptrs)
    return set_error(COZO_GPU_EINVAL, "n_dest must be in [1,%d]", COZO_GPU_MAX_PEERS);
  ScatterDest sc{};
  sc.n_dest = n_dest;
  sc.slot = slot;
  for (uint32_t d = 0; d < n_dest; ++d) {
    sc.ids[d] = reinterpret_cast<uint32_t*>(dest_ids_ptrs[d]);
    sc.dist[d] = reinterpret_cast<float*>(dest_dist_ptrs[d]);
    if (!sc.ids[d] || !sc.dist[d]) return set_error(COZO_GPU_EINVAL, "null destination buffer");
  }
  return hnsw_search_dev(h, queries_dev, B, k, ef, radius, nullptr, nullptr, nullptr, per_query_stats_dev, stream, &sc,
                         nullptr);
}

static int search_host_impl(cozo_gpu_hnsw_t* h, const float* queries, uint32_t B, uint32_t k, uint32_t ef, double radius,
                            const uint32_t* row_mask, uint32_t* out_ids, float* out_dist, uint32_t* out_count,
                            CozoGpuSearchStats* stats) {
  int rc = check_search_args(h, k, ef);
  if (rc) return rc;
  if (B && (!queries || !out_ids || !out_dist)) return set_error(COZO_GPU_EINVAL, "null buffer");
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return 0;
  HnswWorkspace* ws = hnsw_acquire_ws(h);
  if (!ws) return COZO_GPU_ECUDA;
  auto done = [&](int code) {
    hnsw_release_ws(h, ws);
    return code;
  };
#define S_CUDA(call)                                                                              \
  do {                                                                                            \
    cudaError_t _e = (call);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      return done(set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,    \
                            "%s failed: %s", #call, cudaGetErrorString(_e)));                     \
  } while (0)
  const uint32_t dim = h->dev.dim;
  size_t qf = (size_t)B * dim;
  if (ws->q_floats < qf) {
    if (ws->q) cudaFree(ws->q);
    ws->q = nullptr;
    ws->q_floats = 0;
    S_CUDA(cudaMalloc(&ws->q, qf * 4));
    ws->q_floats = qf;
  }
  if (ws->out_rows < B || ws->out_k < k) {
    if (ws->ids) cudaFree(ws->ids);
    if (ws->dist) cudaFree(ws->dist);
    if (ws->count) cudaFree(ws->count);
    if (ws->qstats) cudaFree(ws->qstats);
    ws->ids = nullptr;
    ws->dist = nullptr;
    ws->count = nullptr;
    ws->qstats = nullptr;
    ws->out_rows = ws->out_k = 0;
    size_t rows = std::max<size_t>(B, ws->out_rows), kk = std::max<size_t>(k, ws->out_k);
    S_CUDA(cudaMalloc(&ws->ids, rows * kk * 4));
    S_CUDA(cudaMalloc(&ws->dist, rows * kk * 4));
    S_CUDA(cudaMalloc(&ws->count, rows * 4));
    S_CUDA(cudaMalloc(&ws->qstats, rows * 16));
    ws->out_rows = rows;
    ws->out_k = kk;
  }
  cudaStream_t st = ws->stream;
  if (row_mask) {
    const size_t words = ((size_t)h->dev.n + 31) / 32;
    if (ws->mask_words < words) {
      if (ws->mask) cudaFree(ws->mask);
      ws->mask = nullptr;
      ws->mask_words = 0;
      S_CUDA(cudaMalloc(&ws->mask, std::max<size_t>(words, 1) * 4));
      ws->mask_words = words;
    }
    S_CUDA(cudaMemcpyAsync(ws->mask, row_mask, words * 4, cudaMemcpyHostToDevice, st));
  }
  S_CUDA(cudaMemcpyAsync(ws->q, queries, qf * 4, cudaMemcpyHostToDevice, st));
  S_CUDA(cudaEventRecord(ws->e0, st));
  rc = hnsw_launch_search(h, ws, ws->q, B, k, ef, radius, ws->ids, ws->dist, ws->count, ws->qstats, st, nullptr,
                          row_mask ? ws->mask : nullptr);
  if (rc) return done(rc);
  S_CUDA(cudaEventRecord(ws->e1, st));
  S_CUDA(cudaMemcpyAsync(out_ids, ws->ids, (size_t)B * k * 4, cudaMemcpyDeviceToHost, st));
  S_CUDA(cudaMemcpyAsync(out_dist, ws->dist, (size_t)B * k * 4, cudaMemcpyDeviceToHost, st));
  if (out_count) S_CUDA(cudaMemcpyAsync(out_count, ws->count, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  std::vector<uint32_t> qs;
  if (stats) {
    qs.resize((size_t)B * 4);
    S_CUDA(cudaMemcpyAsync(qs.data(), ws->qstats, (size_t)B * 16, cudaMemcpyDeviceToHost, st));
  }
  S_CUDA(cudaStreamSynchronize(st));
  if (stats) {
    float ms = 0;
    cudaEventElapsedTime(&ms, ws->e0, ws->e1);
    stats->n_queries = B;
    stats->kernel_ms = ms;
    for (uint32_t i = 0; i < B; ++i) {
      stats->dist_evals += qs[(size_t)i * 4 + 0];
      stats->nodes_expanded += qs[(size_t)i * 4 + 1];
      stats->nbr_reads += qs[(size_t)i * 4 + 2];
    }
  }
#undef S_CUDA
  return done(0);
}

extern "C" int cozo_gpu_hnsw_search(cozo_gpu_hnsw_t* h, const float* queries, uint32_t B, uint32_t k, uint32_t ef,
                                    double radius, uint32_t* out_ids, float* out_dist, uint32_t* out_count,
                                    CozoGpuSearchStats* stats) {
  return search_host_impl(h, queries, B, k, ef, radius, nullptr, out_ids, out_dist, out_count, stats);
}

extern "C" int cozo_gpu_hnsw_search_filtered(cozo_gpu_hnsw_t* h, const float* queries, uint32_t B, uint32_t k,
                                             uint32_t ef, double radius, const uint32_t* row_mask, uint32_t* out_ids,
                                             float* out_dist, uint32_t* out_count, CozoGpuSearchStats* stats) {
  if (h && h->dev.n && !row_mask) return set_error(COZO_GPU_EINVAL, "null row mask");
  return search_host_impl(h, queries, B, k, ef, radius, row_mask, out_ids, out_dist, out_count, stats);
}

extern "C" int cozo_gpu_hnsw_search_filtered_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k,
                                                 uint32_t ef, double radius, const uint32_t* row_mask_dev,
                                                 uint32_t* out_ids_dev, float* out_dist_dev, uint32_t* out_count_dev,
                                                 uint32_t* per_query_stats_dev, void* stream) {
  if (!row_mask_dev) return set_error(COZO_GPU_EINVAL, "null row mask");
  return hnsw_search_dev(h, queries_dev, B, k, ef, radius, out_ids_dev, out_dist_dev, out_count_dev,
                         per_query_stats_dev, stream, nullptr, row_mask_dev);
}

extern "C" int cozo_gpu_hnsw_info(cozo_gpu_hnsw_t* h, uint32_t* n_vectors, uint32_t* dim, uint32_t* n_levels,
                                  uint32_t* entry_point) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  if (n_vectors) *n_vectors = h->dev.n;
  if (dim) *dim = h->dev.dim;
  if (n_levels) *n_levels = h->n_levels;
  if (entry_point) *entry_point = h->dev.entry;
  return 0;
}

extern "C" const float* cozo_gpu_hnsw_vectors_dev(cozo_gpu_hnsw_t* h, uint32_t* row_stride) {
  if (!h) return nullptr;
  if (row_stride) *row_stride = h->dev.ld;
  return h->dev.vec;
}

// download one layer as CSR with rows sorted ascending (key order)
static int fetch_level(cozo_gpu_hnsw_t* h, uint32_t level, std::vector<uint32_t>& node_ids,
                       std::vector<uint64_t>& row_ptr, std::vector<uint32_t>& col_idx,
                       std::vector<float>* dist = nullptr) {
  const HnswDev& g = h->dev;
  if (level >= h->n_levels) return set_error(COZO_GPU_EINVAL, "layer %u does not exist", level);
  node_ids.clear();
  row_ptr.assign(1, 0);
  col_idx.clear();
  if (dist) dist->clear();
  const uint32_t stride = level == 0 ? g.s0 : g.su;
  const size_t rows = level == 0 ? (size_t)g.n : (size_t)std::max<uint64_t>(h->up_rows, 1);
  std::vector<uint32_t> adj(rows * stride);
  std::vector<float> adj_d;
  std::vector<uint32_t> off;
  if (!adj.empty())
    COZO_CUDA(cudaMemcpy(adj.data(), level == 0 ? g.adj0 : g.adj_up, adj.size() * 4, cudaMemcpyDeviceToHost));
  if (dist) {
    const float* src = level == 0 ? h->d_adj0_dist : h->d_adj_up_dist;
    if (!src) return set_error(COZO_GPU_EINVAL, "edge distances are not materialised");
    adj_d.resize(adj.size());
    if (!adj_d.empty()) COZO_CUDA(cudaMemcpy(adj_d.data(), src, adj_d.size() * 4, cudaMemcpyDeviceToHost));
  }
  if (level > 0) {
    off.resize(g.n);
    if (g.n) COZO_CUDA(cudaMemcpy(off.data(), g.upper_off, (size_t)g.n * 4, cudaMemcpyDeviceToHost));
  }
  std::vector<std::pair<uint32_t, float>> tmp;
  for (uint32_t i = 0; i < g.n; ++i) {
    if (h->node_level[i] < level) continue;
    node_ids.push_back(i);
    const size_t row = level == 0 ? (size_t)i : (size_t)off[i] + level - 1;
    tmp.clear();
    for (uint32_t j = 0; j < stride; ++j) {
      uint32_t t = adj[row * stride + j];
      if (t == NONE) break;
      tmp.push_back({t, dist ? adj_d[row * stride + j] : 0.f});
    }
    std::sort(tmp.begin(), tmp.end(), [](const auto& a, const auto& b) { return a.first < b.first; });  // key order
    for (auto& e : tmp) {
      col_idx.push_back(e.first);
      if (dist) dist->push_back(e.second);
    }
    row_ptr.push_back(col_idx.size());
  }
  return 0;
}

extern "C" int cozo_gpu_hnsw_level_size(cozo_gpu_hnsw_t* h, uint32_t level, uint32_t* n_nodes, uint64_t* n_edges) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  std::vector<uint32_t> ni, ci;
  std::vector<uint64_t> rp;
  int rc = fetch_level(h, level, ni, rp, ci);
  if (rc) return rc;
  if (n_nodes) *n_nodes = (uint32_t)ni.size();
  if (n_edges) *n_edges = ci.size();
  return 0;
}

extern "C" int cozo_gpu_hnsw_export_level(cozo_gpu_hnsw_t* h, uint32_t level, uint32_t* node_ids, uint64_t* row_ptr,
                                          uint32_t* col_idx) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  std::vector<uint32_t> ni, ci;
  std::vector<uint64_t> rp;
  int rc = fetch_level(h, level, ni, rp, ci);
  if (rc) return rc;
  if (node_ids) std::copy(ni.begin(), ni.end(), node_ids);
  if (row_ptr) std::copy(rp.begin(), rp.end(), row_ptr);
  if (col_idx) std::copy(ci.begin(), ci.end(), col_idx);
  return 0;
}

// Stored `dist` of every edge of a layer (the index relation's value column, relation.rs:1064-1126),
// aligned with the col_idx order of cozo_gpu_hnsw_export_level.
extern "C" int cozo_gpu_hnsw_export_level_dist(cozo_gpu_hnsw_t* h, uint32_t level, float* dist) {
  if (!h || !dist) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = hnsw_ensure_build_state(h);
  if (rc) return rc;
  std::vector<uint32_t> ni, ci;
  std::vector<uint64_t> rp;
  std::vector<float> d;
  rc = fetch_level(h, level, ni, rp, ci, &d);
  if (rc) return rc;
  std::copy(d.begin(), d.end(), dist);
  return 0;
}

// 1 for every id that is still indexed (0 after cozo_gpu_hnsw_remove)
extern "C" int cozo_gpu_hnsw_export_live(cozo_gpu_hnsw_t* h, uint8_t* live) {
  if (!h || !live) return set_error(COZO_GPU_EINVAL, "null argument");
  for (uint32_t i = 0; i < h->dev.n; ++i) live[i] = i < h->live.size() ? h->live[i] : 1;
  return 0;
}
