// hnsw_build.cu — index construction on the device.
//
// Batched variant of SessionTx::hnsw_put_vector (runtime/hnsw.rs:155-375):
// nodes are inserted in id order like create_hnsw_index's bulk insert
// (runtime/relation.rs:1176-1185), a batch at a time.  Every node of a batch
//   K1  searches the graph as it stood before the batch: ef=1 on the layers
//       above its own (hnsw.rs:219-229), ef_construction on its own layers
//       (hnsw.rs:242-256; found_nn carries over between layers);
//   K2  picks neighbours with hnsw_select_neighbours_heuristic (hnsw.rs:470-538),
//       capped at m_max(layer) (hnsw.rs:243-247), writes its own adjacency row
//       (the out edges, hnsw.rs:281-298) and queues the in edges (hnsw.rs:300-318);
//   K3  sorts the queued in edges by (layer, target);
//   K4  appends them to the target rows, shrinking an over-full row with the
//       same heuristic over the stored distances (hnsw_shrink_neighbour,
//       hnsw.rs:376-469).
// Differences from the reference, all consequences of batching: nodes of one
// batch do not see each other during K1, and a row that receives several in
// edges in one batch is shrunk once per chunk of 32 arrivals rather than once
// per arrival.  Soft-deleted (`ignore_link`) rows are not materialised: the
// staged layout only holds what hnsw_get_neighbours would return.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "hnsw_host.hpp"
#include "hnsw_build_kernels.cuh"

namespace cozo {

// thin __global__ wrappers around the bodies in hnsw_build_kernels.cuh
template <int NV, int METRIC>
__global__ void __launch_bounds__(128, 4) build_search_kernel(HnswDev g, BuildDev b, BatchParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  build_search_body<NV, METRIC>(g, b, p, smem);
}
template <int NV, int METRIC>
__global__ void __launch_bounds__(128) build_select_kernel(HnswDev g, BuildDev b, BatchParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  build_select_body<NV, METRIC>(g, b, p, smem);
}
template <int NV, int METRIC>
__global__ void __launch_bounds__(128) build_link_kernel(HnswDev g, BuildDev b, const unsigned long long* keys,
                                                         const uint32_t* perm, const uint32_t* req_src,
                                                         const float* req_d, uint32_t nreq, const uint32_t* heads,
                                                         uint32_t nheads) {
  extern __shared__ __align__(128) uint8_t smem[];
  build_link_body<NV, METRIC>(g, b, keys, perm, req_src, req_d, nreq, heads, nheads, smem);
}

using K1Fn = void (*)(HnswDev, BuildDev, BatchParams);
using K4Fn = void (*)(HnswDev, BuildDev, const unsigned long long*, const uint32_t*, const uint32_t*, const float*,
                      uint32_t, const uint32_t*, uint32_t);
using KdFn = void (*)(HnswDev, BuildDev, const uint32_t*, uint32_t, int);

template <int NV>
struct BuildKernels {
  static void get(int metric, K1Fn& k1, K1Fn& k2, K4Fn& k4, KdFn& kd) {
    switch (metric) {
      case COZO_GPU_L2:
        k1 = build_search_kernel<NV, COZO_GPU_L2>;
        k2 = build_select_kernel<NV, COZO_GPU_L2>;
        k4 = build_link_kernel<NV, COZO_GPU_L2>;
        kd = build_edge_dist_kernel<NV, COZO_GPU_L2>;
        break;
      case COZO_GPU_COSINE:
        k1 = build_search_kernel<NV, COZO_GPU_COSINE>;
        k2 = build_select_kernel<NV, COZO_GPU_COSINE>;
        k4 = build_link_kernel<NV, COZO_GPU_COSINE>;
        kd = build_edge_dist_kernel<NV, COZO_GPU_COSINE>;
        break;
      default:
        k1 = build_search_kernel<NV, COZO_GPU_IP>;
        k2 = build_select_kernel<NV, COZO_GPU_IP>;
        k4 = build_link_kernel<NV, COZO_GPU_IP>;
        kd = build_edge_dist_kernel<NV, COZO_GPU_IP>;
    }
  }
};

static int pick_build_kernels(const HnswDev& g, K1Fn& k1, K1Fn& k2, K4Fn& k4, KdFn& kd) {
  uint32_t need = (g.ld / 4 + 31) / 32;
  if (need <= 1) BuildKernels<1>::get(g.metric, k1, k2, k4, kd);
  else if (need <= 2) BuildKernels<2>::get(g.metric, k1, k2, k4, kd);
  else if (need <= 4) BuildKernels<4>::get(g.metric, k1, k2, k4, kd);
  else if (need <= 6) BuildKernels<6>::get(g.metric, k1, k2, k4, kd);
  else if (need <= 8) BuildKernels<8>::get(g.metric, k1, k2, k4, kd);
  else if (need <= 16) BuildKernels<16>::get(g.metric, k1, k2, k4, kd);
  else BuildKernels<0>::get(g.metric, k1, k2, k4, kd);
  return 0;
}

struct SplitMix64 {
  uint64_t s;
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

#define H_CUDA(call)                                                                                \
  do {                                                                                              \
    cudaError_t _e = (call);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,           \
                       "%s failed: %s (line %d)", #call, cudaGetErrorString(_e), __LINE__);          \
  } while (0)

// grow one device array to `new_bytes`, keeping `old_bytes`, filling the tail with `fill`; a borrowed array is not freed
static int grow(void*& p, size_t old_bytes, size_t new_bytes, int fill_byte, bool owned = true) {
  uint8_t* np = nullptr;
  H_CUDA(cudaMalloc(&np, std::max<size_t>(new_bytes, 1)));
  if (old_bytes && p) H_CUDA(cudaMemcpy(np, p, old_bytes, cudaMemcpyDeviceToDevice));
  if (new_bytes > old_bytes) H_CUDA(cudaMemset(np + old_bytes, fill_byte, new_bytes - old_bytes));
  if (p && owned) cudaFree(p);
  p = np;
  return 0;
}

// capacity management: rows [0,n) / [0,up_rows) are live, the rest is pre-initialised slack
int hnsw_reserve(cozo_gpu_hnsw* h, uint32_t need_n, uint64_t need_up) {
  HnswDev& g = h->dev;
  const auto arrays = row_arrays(h);
  if (need_n > h->cap_n) {
    uint32_t nc = std::max<uint32_t>(need_n, (uint32_t)std::min<uint64_t>(0x7FFFFFFEull, (uint64_t)h->cap_n * 3 / 2));
    for (size_t i = 0; i < arrays.size(); ++i) {
      const RowArray& a = arrays[i];
      int rc = 0;
      if (a.upper) continue;
      if (i == kCodesArray) {
        hnsw_codes_reserve(h, nc);
      } else if (i == kVecArray && !h->vec_owned) {
        if (need_n > h->borrowed_rows) {  // borrowed vectors cannot grow in place: take a private copy
          rc = grow(a.ptr, (size_t)g.n * a.row_bytes, (size_t)nc * a.row_bytes, a.fill, false);
          if (!rc) h->vec_owned = true;
        }
      } else {
        rc = grow(a.ptr, (size_t)h->cap_n * a.row_bytes, (size_t)nc * a.row_bytes, a.fill);
      }
      if (rc) return rc;
    }
    h->cap_n = nc;
  }
  if (need_up > h->cap_up || !h->d_adj_up) {
    uint64_t uc = std::max<uint64_t>(std::max<uint64_t>(need_up, 1), h->cap_up * 3 / 2);
    for (const RowArray& a : arrays) {
      if (!a.upper) continue;
      int rc = grow(a.ptr, (size_t)h->cap_up * a.row_bytes, (size_t)uc * a.row_bytes, a.fill);
      if (rc) return rc;
    }
    h->cap_up = uc;
  }
  g.vec = h->d_vec;
  g.adj0 = h->d_adj0;
  g.adj_up = h->d_adj_up;
  g.upper_off = h->d_upper_off;
  return 0;
}

// never write into a borrowed vector buffer: take a private copy first
static int own_vectors(cozo_gpu_hnsw* h) {
  return h->vec_owned ? 0 : hnsw_reserve(h, h->borrowed_rows + 1, h->up_rows);
}

static BuildDev build_dev(cozo_gpu_hnsw* h) {
  BuildDev b{};
  b.adj0 = h->d_adj0;
  b.adj0_d = h->d_adj0_dist;
  b.deg0 = h->d_deg0;
  b.adj_up = h->d_adj_up;
  b.adj_up_d = h->d_adj_up_dist;
  b.deg_up = h->d_deg_up;
  b.node_level = h->d_node_level;
  b.m_max0 = h->m_max0;
  b.m_max = h->m_max;
  b.keep_pruned = h->keep_pruned;
  b.extend = 0;
  b.upper_off = h->d_upper_off;
  return b;
}

// An index staged from host CSR carries no degrees / edge distances: derive them once.
int hnsw_ensure_build_state(cozo_gpu_hnsw* h) {
  if (h->f64)
    return set_error(COZO_GPU_EUNSUP, "F64 indexes are search-only on the device: re-stage after a mutation");
  if (h->build_state_ready) return 0;
  HnswDev& g = h->dev;
  // staging allocated exactly n rows; move to the growable layout
  if (h->cap_n == 0) {
    h->cap_n = g.n;
    // capacity == live rows exactly: the arrays staging made have no slack, and hnsw_reserve's grow() treats
    // everything below the capacity as initialised (a capacity of 1 with 0 live upper rows would carry one
    // row of uninitialised ids and degrees into the grown arrays)
    h->cap_up = h->up_rows;
    // staging made vec, codes, adj0, upper_off and adj_up; the builder's arrays start as unused capacity
    const auto arrays = row_arrays(h);
    for (size_t i = 0; i < arrays.size(); ++i) {
      const RowArray& a = arrays[i];
      if (a.ptr || i == kVecArray || i == kCodesArray) continue;
      const size_t bytes = std::max<size_t>(a.upper ? h->cap_up : h->cap_n, 1) * a.row_bytes;
      H_CUDA(cudaMalloc(&a.ptr, bytes));
      H_CUDA(cudaMemset(a.ptr, a.fill, bytes));
    }
    if (g.n) H_CUDA(cudaMemcpy(h->d_node_level, h->node_level.data(), g.n, cudaMemcpyHostToDevice));
    std::vector<uint32_t> owner;
    for (uint32_t i = 0; i < g.n; ++i)
      for (uint32_t L = 0; L < h->node_level[i]; ++L) owner.push_back(i);
    if (!owner.empty()) H_CUDA(cudaMemcpy(h->d_up_owner, owner.data(), owner.size() * 4, cudaMemcpyHostToDevice));
    h->live.assign(g.n, 1);
    h->n_live = g.n;
  }
  K1Fn k1, k2;
  K4Fn k4;
  KdFn kd;
  int rc = pick_build_kernels(g, k1, k2, k4, kd);
  if (rc) return rc;
  BuildDev b = build_dev(h);
  if (g.n) kd<<<(g.n + 3) / 4, 128>>>(g, b, nullptr, g.n, 0);
  if (h->up_rows) kd<<<(uint32_t)((h->up_rows + 3) / 4), 128>>>(g, b, h->d_up_owner, (uint32_t)h->up_rows, 1);
  H_CUDA(cudaGetLastError());
  H_CUDA(cudaDeviceSynchronize());
  h->build_state_ready = true;
  return 0;
}

// f32 row stages per warp of the K1 search.  Wide rows start from the search's WIDE_RING_BYTES ring and give up stages,
// down to one, while one warp (its query included) does not fit the shared-memory opt-in.
static uint32_t build_stages(uint32_t ld, uint32_t ef_c) {
  uint32_t ns = std::min(32u, std::max(1u, (uint32_t)get_option("hnsw.stages", 4)));
  if (ld > REG_QUERY_MAX_LD) {
    ns = std::max(1u, std::min(ns, WIDE_RING_BYTES / (ld * 4)));
    while (ns > 1 && make_layout(ef_c, ns, ld).warp_bytes > device_info().smem_optin) --ns;
  }
  return ns;
}

// the error of a K1 layout that does not fit even one warp
static int build_smem_unsup(const HnswDev& g, uint32_t ef_c, size_t need) {
  if (g.ld > REG_QUERY_MAX_LD)
    return set_error(COZO_GPU_EUNSUP, "vec_dim %u at ef_construction=%u needs %zu B of shared memory (limit %zu)", g.dim,
                     ef_c, need, device_info().smem_optin);
  return set_error(COZO_GPU_EUNSUP, "ef_construction=%u does not fit shared memory", ef_c);
}

// The batched insertion loop for the nodes `ids` (ascending) whose vectors, levels and upper_off are in place, linked in
// list order.  min_entry: after each batch the entry is the smallest id on the top layer (a node inserted at a key
// before the entry's, on the entry's layer, takes over, hnsw.rs:184-199); otherwise only a higher layer re-points it.
static int hnsw_insert_ids(cozo_gpu_hnsw* h, const std::vector<uint32_t>& ids, uint32_t max_batch, bool min_entry) {
  const DeviceInfo& di = device_info();
  HnswDev& g = h->dev;
  const uint32_t total = (uint32_t)ids.size();
  if (total == 0) return 0;
  K1Fn k1, k2;
  K4Fn k4;
  KdFn kd;
  int rc = pick_build_kernels(g, k1, k2, k4, kd);
  if (rc) return rc;
  BuildDev b = build_dev(h);
  const uint32_t ef_c = h->ef_construction;
  const bool extend = h->extend_candidates != 0;
  if (!max_batch) max_batch = 8192;
  // extend_candidates reads the rows of OTHER nodes while selecting, so its result depends on the order in which
  // the reference links the new node's neighbours: one node per batch, in-edges linked one at a time in selection order
  if (extend) max_batch = 1;
  uint32_t wpc = (uint32_t)get_option("hnsw.warps_per_cta", 4);
  wpc = std::min(4u, std::max(1u, wpc));
  const uint32_t ns = build_stages(g.ld, ef_c);
  SmemLayout lay = make_layout(ef_c, ns, g.ld);
  size_t smem1 = (size_t)lay.warp_bytes * wpc;
  while (smem1 > di.smem_optin && wpc > 1) {
    wpc >>= 1;
    smem1 = (size_t)lay.warp_bytes * wpc;
  }
  if (smem1 > di.smem_optin) return build_smem_unsup(g, ef_c, smem1);
  H_CUDA(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)di.smem_optin));
  int cps = 0;
  H_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, k1, wpc * 32, smem1));
  if (cps < 1) return set_error(COZO_GPU_ECUDA, "build kernel does not fit on an SM");
  const uint32_t max_grid1 = (uint32_t)di.sm_count * (uint32_t)cps;
  const uint32_t mcap = std::max(h->m_max0, h->m_max);
  const size_t smem2 = (size_t)4 * 2 * mcap * 4;
  const size_t smem4 = (size_t)4 * (4 * (mcap + 32) + 2 * mcap) * 4;

  struct Scratch {
    uint32_t *coff = nullptr, *list_node = nullptr, *list_level = nullptr;
    float* cand_d = nullptr;
    uint32_t *cand_id = nullptr, *cand_cnt = nullptr;
    unsigned long long *req_key = nullptr, *req_key2 = nullptr;
    uint32_t *req_src = nullptr, *perm = nullptr, *perm2 = nullptr, *heads = nullptr, *counters = nullptr;
    float* req_d = nullptr;
    void* cub_tmp = nullptr;
    unsigned long long* ext_keys = nullptr;
    float* ext_d = nullptr;
    uint32_t* ext_id = nullptr;
    cozo_gpu_hnsw* h = nullptr;
    HnswWorkspace* ws = nullptr;
    ~Scratch() {
      void* ptrs[] = {coff, list_node, list_level, cand_d, cand_id, cand_cnt, req_key, req_key2,
                      req_src, perm, perm2, heads, counters, req_d, cub_tmp, ext_keys, ext_d, ext_id};
      for (void* p : ptrs)
        if (p) cudaFree(p);
      if (ws) hnsw_release_ws(h, ws);
    }
  } sc;
  sc.h = h;
  sc.ws = hnsw_acquire_ws(h);
  if (!sc.ws) return COZO_GPU_ECUDA;
  HnswWorkspace* ws = sc.ws;
  cudaStream_t st = ws->stream;
  const uint32_t nwords = round_up((g.n + 31) / 32, 4);  // the search may visit ANY indexed id, not only ids < end
  const uint32_t logcap = std::min<uint32_t>(65536u, std::max<uint32_t>(4096u, 64u * ef_c));
  {
    size_t slots = (size_t)max_grid1 * wpc;
    rc = hnsw_ws_reserve(ws, slots * nwords, slots * logcap, st);
    if (rc) return rc;
  }
  max_batch = std::min<uint32_t>(max_batch, total);
  uint32_t max_lvl = 0;
  for (uint32_t id : ids) max_lvl = std::max<uint32_t>(max_lvl, h->node_level[id]);
  const uint32_t Tcap = (uint32_t)std::min<uint64_t>((uint64_t)max_batch * (max_lvl + 1), (uint64_t)max_batch + h->up_rows + 16);
  const uint64_t req_cap = std::max<uint64_t>((uint64_t)Tcap * mcap, 1);
  H_CUDA(cudaMalloc(&sc.coff, ((size_t)max_batch + 1) * 4));
  H_CUDA(cudaMalloc(&sc.list_node, (size_t)Tcap * 4));
  H_CUDA(cudaMalloc(&sc.list_level, (size_t)Tcap * 4));
  H_CUDA(cudaMalloc(&sc.cand_d, (size_t)Tcap * ef_c * 4));
  H_CUDA(cudaMalloc(&sc.cand_id, (size_t)Tcap * ef_c * 4));
  H_CUDA(cudaMalloc(&sc.cand_cnt, (size_t)Tcap * 4));
  H_CUDA(cudaMalloc(&sc.req_key, req_cap * 8));
  H_CUDA(cudaMalloc(&sc.req_key2, req_cap * 8));
  H_CUDA(cudaMalloc(&sc.req_src, req_cap * 4));
  H_CUDA(cudaMalloc(&sc.req_d, req_cap * 4));
  H_CUDA(cudaMalloc(&sc.perm, req_cap * 4));
  H_CUDA(cudaMalloc(&sc.perm2, req_cap * 4));
  H_CUDA(cudaMalloc(&sc.heads, req_cap * 4));
  H_CUDA(cudaMalloc(&sc.counters, 64));
  if (extend) {
    uint32_t cap = 32;
    const uint32_t need = std::max(ef_c, mcap + 32) * (1 + std::max(g.s0, g.su));
    while (cap < need) cap <<= 1;
    b.extend = 1;
    b.ext_cap = cap;
    const size_t slices = std::max<size_t>(Tcap, 4);  // K2: one slice per task; the sequential link step uses slice 0
    H_CUDA(cudaMalloc(&sc.ext_keys, slices * cap * 8));
    H_CUDA(cudaMalloc(&sc.ext_d, slices * cap * 4));
    H_CUDA(cudaMalloc(&sc.ext_id, slices * cap * 4));
    b.ext_keys = sc.ext_keys;
    b.ext_d = sc.ext_d;
    b.ext_id = sc.ext_id;
  }
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, sc.req_key, sc.req_key2, sc.perm, sc.perm2, (int)req_cap, 0, 40,
                                  st);
  H_CUDA(cudaMalloc(&sc.cub_tmp, cub_bytes));
  {
    std::vector<uint32_t> iota(req_cap);
    for (uint64_t i = 0; i < req_cap; ++i) iota[i] = (uint32_t)i;
    H_CUDA(cudaMemcpy(sc.perm, iota.data(), req_cap * 4, cudaMemcpyHostToDevice));
  }

  uint32_t inserted = 0;  // position in `ids`
  if (g.entry == NONE) {  // first vector: fresh self-loops only (hnsw.rs:360-373)
    g.entry = ids[0];
    g.top_level = h->node_level[ids[0]];
    inserted = 1;
    h->n_live += 1;
  }
  std::vector<uint32_t> coff, lnode, llevel;
  while (inserted < total) {
    // a batch never exceeds 1/16 of what is already linked, so that batch members (which do not see
    // each other) stay a small fraction of every neighbourhood
    uint32_t bs = std::min<uint32_t>(std::min<uint32_t>(max_batch, std::max<uint32_t>(1u, h->n_live / 16)), total - inserted);
    const uint32_t top = g.top_level;
    coff.assign(bs + 1, 0);
    lnode.clear();
    llevel.clear();
    for (uint32_t i = 0; i < bs; ++i) {
      uint32_t id = ids[inserted + i];
      uint32_t nl = std::min<uint32_t>(h->node_level[id], top) + 1;
      coff[i] = (uint32_t)lnode.size();
      for (uint32_t L = 0; L < nl; ++L) {
        lnode.push_back(id);
        llevel.push_back(L);
      }
    }
    coff[bs] = (uint32_t)lnode.size();
    const uint32_t T = (uint32_t)lnode.size();
    if (T > Tcap) return set_error(COZO_GPU_ECUDA, "internal: batch list overflow");
    H_CUDA(cudaMemcpyAsync(sc.coff, coff.data(), ((size_t)bs + 1) * 4, cudaMemcpyHostToDevice, st));
    H_CUDA(cudaMemcpyAsync(sc.list_node, lnode.data(), (size_t)T * 4, cudaMemcpyHostToDevice, st));
    H_CUDA(cudaMemcpyAsync(sc.list_level, llevel.data(), (size_t)T * 4, cudaMemcpyHostToDevice, st));
    H_CUDA(cudaMemsetAsync(sc.counters, 0, 64, st));
    BatchParams p{};
    p.begin = ids[inserted];
    p.count = bs;
    p.top = top;
    p.ef_c = ef_c;
    p.coff = sc.coff;
    p.list_node = sc.list_node;
    p.list_level = sc.list_level;
    p.T = T;
    p.cand_d = sc.cand_d;
    p.cand_id = sc.cand_id;
    p.cand_cnt = sc.cand_cnt;
    p.req_key = sc.req_key;
    p.req_src = sc.req_src;
    p.req_d = sc.req_d;
    p.req_count = sc.counters + 1;
    p.counter = sc.counters + 0;
    p.vis = ws->vis;
    p.nwords = nwords;
    p.vlog = ws->vlog;
    p.logcap = logcap;
    p.ns = ns;
    p.lay = lay;
    uint32_t grid1 = std::min<uint32_t>(max_grid1, (bs + wpc - 1) / wpc);
    k1<<<grid1, wpc * 32, smem1, st>>>(g, b, p);
    H_CUDA(cudaGetLastError());
    k2<<<(T + 3) / 4, 128, smem2, st>>>(g, b, p);
    H_CUDA(cudaGetLastError());
    uint32_t nreq = 0;
    H_CUDA(cudaMemcpyAsync(&nreq, sc.counters + 1, 4, cudaMemcpyDeviceToHost, st));
    H_CUDA(cudaStreamSynchronize(st));
    if (nreq > req_cap) return set_error(COZO_GPU_ECUDA, "internal: in-edge queue overflow");
    if (nreq && extend) {
      // the reference links the selected neighbours one by one, nearest first (hnsw.rs:279-357); a later shrink sees
      // the rows an earlier one left.  Requests sit in the queue in exactly that order (K2 writes a task's requests
      // consecutively), so: one launch per request, in queue order, on this stream.
      for (uint32_t r = 0; r < nreq; ++r)
        k4<<<1, 32, smem4, st>>>(g, b, sc.req_key, sc.perm, sc.req_src, sc.req_d, nreq, sc.perm + r, 1);
      H_CUDA(cudaGetLastError());
    } else if (nreq) {
      size_t tb = cub_bytes;
      cub::DeviceRadixSort::SortPairs(sc.cub_tmp, tb, sc.req_key, sc.req_key2, sc.perm, sc.perm2, (int)nreq, 0, 40, st);
      build_heads_kernel<<<(nreq + 255) / 256, 256, 0, st>>>(sc.req_key2, nreq, sc.heads, sc.counters + 2);
      H_CUDA(cudaGetLastError());
      uint32_t nheads = 0;
      H_CUDA(cudaMemcpyAsync(&nheads, sc.counters + 2, 4, cudaMemcpyDeviceToHost, st));
      H_CUDA(cudaStreamSynchronize(st));
      k4<<<(nheads + 3) / 4, 128, smem4, st>>>(g, b, sc.req_key2, sc.perm2, sc.req_src, sc.req_d, nreq, sc.heads,
                                               nheads);
      H_CUDA(cudaGetLastError());
    }
    // a node above the current top becomes the entry point (hnsw.rs:206-218);
    // the entry is the smallest id on the top layer (hnsw.rs:184-199)
    for (uint32_t i = 0; i < bs; ++i) {
      uint32_t id = ids[inserted + i];
      if (h->node_level[id] > g.top_level) {
        g.top_level = h->node_level[id];
        g.entry = id;
      } else if (min_entry && h->node_level[id] == g.top_level && id < g.entry) {
        g.entry = id;
      }
    }
    inserted += bs;
    h->n_live += bs;
  }
  H_CUDA(cudaStreamSynchronize(st));
  h->n_levels = g.top_level + 1;
  return 0;
}

// hnsw_insert_ids for the id range [begin, end)
int hnsw_insert_range(cozo_gpu_hnsw* h, uint32_t begin, uint32_t end, uint32_t max_batch) {
  std::vector<uint32_t> ids;
  for (uint32_t id = begin; id < end; ++id) ids.push_back(id);
  return hnsw_insert_ids(h, ids, max_batch, false);
}

// levels of `count` new rows, drawn in row order from the handle's seeded level law (hnsw.rs:46-52),
// level_multiplier = 1/ln(m) (relation.rs:1147)
static std::vector<uint8_t> draw_levels(uint64_t& rng_state, uint32_t m_max, uint32_t count) {
  SplitMix64 rng{rng_state};
  const double mult = 1.0 / std::log((double)m_max);
  std::vector<uint8_t> lv(count);
  for (uint32_t i = 0; i < count; ++i) {
    double u = rng.uniform();
    double r = -std::log(u) * mult;
    if (!(r < 15.0)) r = 15.0;
    lv[i] = (uint8_t)std::floor(r);
  }
  rng_state = rng.s;
  return lv;
}

// append `count` vectors as ids [n, n+count): levels from the handle's RNG, rows and capacity
static int append_nodes(cozo_gpu_hnsw* h, const float* vectors, int on_device, uint32_t count) {
  HnswDev& g = h->dev;
  const uint32_t n0 = g.n, n1 = n0 + count;
  if ((uint64_t)n0 + count >= 0x7FFFFFFFull) return set_error(COZO_GPU_EUNSUP, "too many vectors");
  const std::vector<uint8_t> lvs = draw_levels(h->rng_state, h->m_max, count);
  h->node_level.resize(n1, 0);
  h->live.resize(n1, 1);
  std::vector<uint32_t> upper_off(count, NONE);
  std::vector<uint32_t> owners;
  uint64_t up = h->up_rows;
  for (uint32_t i = 0; i < count; ++i) {
    const uint8_t lv = lvs[i];
    h->node_level[n0 + i] = lv;
    if (lv) {
      upper_off[i] = (uint32_t)up;
      up += lv;
      for (uint32_t L = 0; L < lv; ++L) owners.push_back(n0 + i);
    }
  }
  int rc = hnsw_reserve(h, n1, up);
  if (rc) return rc;
  if (vectors)  // nullptr: the (borrowed) rows are already in place
    H_CUDA(cudaMemcpy2D(h->d_vec + (size_t)n0 * g.ld, (size_t)g.ld * 4, vectors, (size_t)g.dim * 4,
                        (size_t)g.dim * 4, count, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  hnsw_codes_fill(h, n0, count);
  H_CUDA(cudaMemcpy(h->d_upper_off + n0, upper_off.data(), (size_t)count * 4, cudaMemcpyHostToDevice));
  H_CUDA(cudaMemcpy(h->d_node_level + n0, h->node_level.data() + n0, count, cudaMemcpyHostToDevice));
  if (!owners.empty())
    H_CUDA(cudaMemcpy(h->d_up_owner + h->up_rows, owners.data(), owners.size() * 4, cudaMemcpyHostToDevice));
  h->up_rows = up;
  g.n = n1;
  return 0;
}

}  // namespace cozo

using namespace cozo;

extern "C" int cozo_gpu_hnsw_build(cozo_gpu_hnsw_t** out, const CozoGpuHnswBuildDesc* d) {
  if (!out || !d) return set_error(COZO_GPU_EINVAL, "null argument");
  *out = nullptr;
  int rc = ensure_init();
  if (rc) return rc;
  if (d->dim == 0 || d->n_vectors == 0 || !d->vectors) return set_error(COZO_GPU_EINVAL, "bad build descriptor");
  if (d->metric < 0 || d->metric > 2) return set_error(COZO_GPU_EINVAL, "unknown distance %d", d->metric);
  if (d->m_neighbours < 2 || d->m_neighbours > 64)
    return set_error(COZO_GPU_EUNSUP, "m_neighbours must be in [2,64] for the device builder");
  if (d->ef_construction == 0) return set_error(COZO_GPU_EINVAL, "ef_construction must be set");  // sys.rs:603
  if (d->n_vectors >= 0x7FFFFFFFu) return set_error(COZO_GPU_EUNSUP, "too many vectors");
  const uint32_t n = d->n_vectors;
  const uint32_t m = d->m_neighbours;

  auto* h = new cozo_gpu_hnsw();
  HnswDev& g = h->dev;
  g.n = 0;
  g.dim = d->dim;
  g.ld = round_up(d->dim, 4);
  g.code_ld = code_row_bytes(g.ld);
  g.metric = d->metric;
  g.entry = NONE;
  g.top_level = 0;
  h->m_max = m;       // relation.rs:1145
  h->m_max0 = 2 * m;  // relation.rs:1146
  g.s0 = round_up(h->m_max0, 32);
  g.su = round_up(h->m_max, 32);
  h->ef_construction = d->ef_construction;
  h->keep_pruned = d->keep_pruned_connections;
  h->extend_candidates = d->extend_candidates != 0;
  h->rng_state = d->level_seed;
  h->build_state_ready = true;
  auto fail = [&](int code) {
    cozo_gpu_hnsw_free(h);
    return code;
  };
  const bool borrow = d->vectors_on_device && d->borrow_vectors && g.ld == g.dim;
  if (borrow) {  // search straight out of the caller's buffer; a later insert takes a private copy
    h->d_vec = const_cast<float*>(d->vectors);
    h->vec_owned = false;
    h->borrowed_rows = n;
  }
  rc = append_nodes(h, borrow ? nullptr : d->vectors, d->vectors_on_device, n);
  if (rc) return fail(rc);
  rc = hnsw_insert_range(h, 0, n, d->max_batch);
  if (rc) return fail(rc);
  *out = h;
  return 0;
}

// The settings and build state an insertion needs (shared by insert and insert_at).
static int prepare_insert(cozo_gpu_hnsw* h, uint32_t ef_construction, int32_t keep_pruned_connections) {
  // A handle staged from the canary row alone (n = 0) grows from empty arrays: hnsw_ensure_build_state gives it
  // capacities equal to its live rows (0), so every row the first insert creates is initialised by grow().
  if (h->m_max < 2 || h->m_max > 64) return set_error(COZO_GPU_EUNSUP, "m_neighbours must be in [2,64] for the device builder");
  if (ef_construction) h->ef_construction = ef_construction;
  if (h->ef_construction == 0) return set_error(COZO_GPU_EINVAL, "ef_construction must be set");
  if (keep_pruned_connections >= 0) h->keep_pruned = keep_pruned_connections;
  // a staged handle learns the manifest's extend_candidates through the option (a built handle keeps its own)
  if (get_option("hnsw.extend_candidates", -1) >= 0) h->extend_candidates = get_option("hnsw.extend_candidates", 0) != 0;
  return hnsw_ensure_build_state(h);
}

// The builder needs at least one warp's shared memory (for wide rows: query, one ring stage and the beam); an insertion
// checks it before any row is appended or moved.
static int check_build_smem(cozo_gpu_hnsw* h) {
  const HnswDev& g = h->dev;
  const uint32_t wb = make_layout(h->ef_construction, build_stages(g.ld, h->ef_construction), g.ld).warp_bytes;
  return wb > device_info().smem_optin ? build_smem_unsup(g, h->ef_construction, wb) : 0;
}

// hnsw_put for rows that sort after every indexed key (query/stored.rs:332 -> hnsw.rs:679-727).
extern "C" int cozo_gpu_hnsw_insert(cozo_gpu_hnsw_t* h, const float* vectors, uint32_t count, int32_t vectors_on_device,
                                    uint32_t ef_construction, int32_t keep_pruned_connections, uint32_t* first_id) {
  if (!h || (count && !vectors)) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (first_id) *first_id = h->dev.n;
  if (count == 0) return 0;
  rc = prepare_insert(h, ef_construction, keep_pruned_connections);
  if (!rc) rc = check_build_smem(h);
  if (rc) return rc;
  const uint32_t n0 = h->dev.n;
  rc = append_nodes(h, vectors, vectors_on_device, count);
  if (rc) return rc;
  return hnsw_insert_range(h, n0, n0 + count, 0);
}

// a device allocation freed at the end of the scope
template <class T>
struct DevScratch {
  T* p = nullptr;
  ~DevScratch() {
    if (p) cudaFree(p);
  }
};

template <class T, class Map>
static void launch_move_rows(const uint8_t* stage, uint8_t* base, size_t row_bytes, uint32_t lo, uint32_t rows, Map map) {
  const uint32_t e = (uint32_t)(row_bytes / sizeof(T));
  const uint64_t threads = (uint64_t)rows * (e >= 32 ? 32 : 1);
  move_rows_kernel<T, Map><<<(uint32_t)((threads + 255) / 256), 256>>>(reinterpret_cast<const T*>(stage),
                                                                         reinterpret_cast<T*>(base), e, lo, rows, map);
}

// Moves rows [first, n) of one array to rows map(j), dropping rows that map to NONE, `chunk` rows at a time through
// `stage`: from the tail when destinations are above their sources, from the head when they are below.  Either way a
// chunk only overwrites rows already read, so no second copy of the array is needed.  On the legacy default stream.
template <class Map>
static int move_rows(const RowArray& a, uint32_t first, uint32_t n, bool tail_first, uint8_t* stage, uint64_t chunk,
                     Map map) {
  uint8_t* p = static_cast<uint8_t*>(a.ptr);
  const size_t rb = a.row_bytes;
  for (uint32_t done = 0; done < n - first;) {
    const uint32_t rows = (uint32_t)std::min<uint64_t>(chunk, n - first - done);
    const uint32_t lo = tail_first ? n - done - rows : first + done;
    H_CUDA(cudaMemcpyAsync(stage, p + (size_t)lo * rb, (size_t)rows * rb, cudaMemcpyDeviceToDevice, 0));
    if (rb % 16 == 0) launch_move_rows<uint4>(stage, p, rb, lo, rows, map);
    else if (rb % 4 == 0) launch_move_rows<uint32_t>(stage, p, rb, lo, rows, map);
    else launch_move_rows<uint8_t>(stage, p, rb, lo, rows, map);
    H_CUDA(cudaGetLastError());
    done += rows;
  }
  return 0;
}

template <class Map>
static int map_ids(uint32_t* ids, size_t count, Map map, uint32_t* bad) {
  if (!count) return 0;
  map_ids_kernel<Map><<<(uint32_t)((count + 255) / 256), 256>>>(ids, count, map, bad);
  H_CUDA(cudaGetLastError());
  return 0;
}

// Applies a monotone relabelling to the handle.  Node row j >= first moves to row node_map(j) (host_map[j] on the host;
// NONE drops the row) and n1 node rows remain.  With up_map, upper row r >= up_first likewise moves to up_map[r] and up1
// upper rows remain; without it the upper rows stay where they are.  Every row array moves through one staging buffer
// in chunks of 64 MB, or of `hnsw.shift_chunk_rows` rows when that is set; then every stored id is mapped, rows freed
// at the end return to the state of unused capacity, and the host copies of levels, live flags and the entry follow.
// The caller has made room for n1 rows.  All scratch is allocated before any row moves, so that running out of memory
// leaves the index as it was.
template <class NodeMap>
static int relabel_rows(cozo_gpu_hnsw* h, NodeMap node_map, const std::vector<uint32_t>& host_map, uint32_t first,
                        uint32_t n1, const uint32_t* up_map = nullptr, uint32_t up_first = 0, uint32_t up1 = 0) {
  HnswDev& g = h->dev;
  const uint32_t n0 = g.n, up0 = (uint32_t)h->up_rows;
  if (!up_map) up_first = up1 = up0;
  const size_t kStageBytes = (size_t)64 << 20;
  const int64_t chunk_opt = get_option("hnsw.shift_chunk_rows", 0);
  auto chunk_rows = [&](const RowArray& a) {
    const uint64_t moving = a.upper ? up0 - up_first : n0 - first;
    const uint64_t c = chunk_opt > 0 ? (uint64_t)chunk_opt : std::max<uint64_t>(1, kStageBytes / a.row_bytes);
    return std::max<uint64_t>(1, std::min(c, moving));
  };
  size_t stage_bytes = 1;
  for (const RowArray& a : row_arrays(h)) stage_bytes = std::max(stage_bytes, (size_t)chunk_rows(a) * a.row_bytes);
  DevScratch<uint8_t> stage;
  DevScratch<uint32_t> bad;  // stored ids that name a dropped row
  H_CUDA(cudaMalloc(&stage.p, stage_bytes));
  H_CUDA(cudaMalloc(&bad.p, 4));
  H_CUDA(cudaMemsetAsync(bad.p, 0, 4, 0));
  int rc = own_vectors(h);
  if (rc) return rc;

  // after the private copy: the arrays' current addresses
  const auto arrays = row_arrays(h);
  for (const RowArray& a : arrays) {
    if (!a.ptr) continue;
    const uint64_t chunk = chunk_rows(a);
    rc = a.upper ? move_rows(a, up_first, up0, up1 > up0, stage.p, chunk, TableMap{up_map})
                 : move_rows(a, first, n0, n1 > n0, stage.p, chunk, node_map);
    if (rc) return rc;
  }
  rc = map_ids(h->d_adj0, (size_t)n1 * g.s0, node_map, bad.p);
  if (!rc) rc = map_ids(h->d_adj_up, (size_t)up1 * g.su, node_map, bad.p);
  if (!rc) rc = map_ids(h->d_up_owner, up1, node_map, bad.p);
  if (!rc && up_map) rc = map_ids(h->d_upper_off, n1, TableMap{up_map}, bad.p);
  if (rc) return rc;
  for (const RowArray& a : arrays) {
    const uint32_t from = a.upper ? up1 : n1, to = a.upper ? up0 : n0;
    if (a.ptr && from < to)
      H_CUDA(cudaMemsetAsync(static_cast<uint8_t*>(a.ptr) + (size_t)from * a.row_bytes, a.fill,
                             (size_t)(to - from) * a.row_bytes, 0));
  }
  // the host copies, built while the device works
  std::vector<uint8_t> level(n1), live(n1, 1);
  for (uint32_t j = 0; j < n0; ++j)
    if (host_map[j] != NONE) {
      level[host_map[j]] = h->node_level[j];
      live[host_map[j]] = h->live[j];
    }
  uint32_t nbad = 0;
  H_CUDA(cudaMemcpy(&nbad, bad.p, 4, cudaMemcpyDeviceToHost));
  if (nbad) return set_error(COZO_GPU_ECUDA, "internal: %u stored ids name removed ids", nbad);
  h->node_level.swap(level);
  h->live.swap(live);
  if (g.entry != NONE) g.entry = host_map[g.entry];
  h->up_rows = up1;
  g.n = n1;
  return 0;
}

// hnsw_put of new rows at any key position (query/stored.rs:332 -> hnsw.rs:679-727).  Existing ids move up to open a
// gap before every new row, so that dense ids stay in compound-key order; then the new ids are linked in one batched run.
extern "C" int cozo_gpu_hnsw_insert_at(cozo_gpu_hnsw_t* h, const uint32_t* positions, const float* vectors, uint32_t count,
                                       int32_t vectors_on_device, uint32_t ef_construction,
                                       int32_t keep_pruned_connections, uint32_t* out_ids) {
  if (!h || (count && (!positions || !vectors))) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (count == 0) return 0;
  HnswDev& g = h->dev;
  const uint32_t n0 = g.n;
  for (uint32_t i = 0; i < count; ++i)
    if (positions[i] > n0 || (i && positions[i] < positions[i - 1]))
      return set_error(COZO_GPU_EINVAL, "positions must be non-decreasing and at most n = %u (row %u)", n0, i);
  if ((uint64_t)n0 + count >= 0x7FFFFFFFull) return set_error(COZO_GPU_EUNSUP, "too many vectors");
  // an asynchronous search_dev may still be reading the rows about to move (and ids up to its n)
  H_CUDA(cudaDeviceSynchronize());
  if (positions[0] == n0) {  // every row after every indexed key: an append
    uint32_t first = 0;
    rc = cozo_gpu_hnsw_insert(h, vectors, count, vectors_on_device, ef_construction, keep_pruned_connections, &first);
    if (!rc && out_ids)
      for (uint32_t i = 0; i < count; ++i) out_ids[i] = first + i;
    return rc;
  }
  rc = prepare_insert(h, ef_construction, keep_pruned_connections);
  if (rc) return rc;
  rc = check_build_smem(h);  // refuse before any row moves
  if (rc) return rc;

  // scratch first, so that running out of memory leaves the index as it was
  DevScratch<uint32_t> d_pos, d_ids, d_up_off;
  DevScratch<uint8_t> d_levels;
  DevScratch<float> d_vec;
  H_CUDA(cudaMalloc(&d_pos.p, (size_t)count * 4));
  H_CUDA(cudaMalloc(&d_ids.p, (size_t)count * 4));
  H_CUDA(cudaMalloc(&d_up_off.p, (size_t)count * 4));
  H_CUDA(cudaMalloc(&d_levels.p, count));
  if (!vectors_on_device) H_CUDA(cudaMalloc(&d_vec.p, (size_t)count * g.dim * 4));

  const uint32_t n1 = n0 + count;
  uint64_t rng = h->rng_state;  // kept until the rows have moved
  const std::vector<uint8_t> lvs = draw_levels(rng, h->m_max, count);
  std::vector<uint32_t> new_ids(count), up_off(count, NONE), owners;
  uint64_t up = h->up_rows;
  for (uint32_t i = 0; i < count; ++i) {
    new_ids[i] = positions[i] + i;
    if (lvs[i]) {
      up_off[i] = (uint32_t)up;
      up += lvs[i];
      for (uint32_t L = 0; L < lvs[i]; ++L) owners.push_back(new_ids[i]);
    }
  }
  // old row j -> j + #{positions <= j}; rows below positions[0] stay
  std::vector<uint32_t> map(n0);
  for (uint32_t j = 0, i = 0; j < n0; ++j) {
    while (i < count && positions[i] <= j) ++i;
    map[j] = j + i;
  }
  const uint64_t up0 = h->up_rows;
  rc = hnsw_reserve(h, n1, up);
  if (rc) return rc;
  H_CUDA(cudaMemcpy(d_pos.p, positions, (size_t)count * 4, cudaMemcpyHostToDevice));
  H_CUDA(cudaMemcpy(d_ids.p, new_ids.data(), (size_t)count * 4, cudaMemcpyHostToDevice));
  H_CUDA(cudaMemcpy(d_up_off.p, up_off.data(), (size_t)count * 4, cudaMemcpyHostToDevice));
  H_CUDA(cudaMemcpy(d_levels.p, lvs.data(), count, cudaMemcpyHostToDevice));
  const float* d_new_vec = vectors;
  if (!vectors_on_device) {
    H_CUDA(cudaMemcpy(d_vec.p, vectors, (size_t)count * g.dim * 4, cudaMemcpyHostToDevice));
    d_new_vec = d_vec.p;
  }
  // adj_up rows stay where they are (upper_off holds row numbers)
  rc = relabel_rows(h, GapMap{d_pos.p, count}, map, positions[0], n1);
  if (rc) return rc;
  h->rng_state = rng;
  // the new rows; their upper rows are fresh rows at the end of adj_up
  place_new_rows_kernel<<<(uint32_t)(((uint64_t)count * 32 + 255) / 256), 256>>>(
      d_ids.p, count, d_new_vec, g.dim, h->d_vec, g.ld, h->d_adj0, g.s0, h->d_deg0, d_up_off.p, h->d_upper_off,
      d_levels.p, h->d_node_level, h->d_dead);
  H_CUDA(cudaGetLastError());
  hnsw_codes_fill(h, 0, count, d_ids.p);
  if (!owners.empty())
    H_CUDA(cudaMemcpyAsync(h->d_up_owner + up0, owners.data(), owners.size() * 4, cudaMemcpyHostToDevice, 0));
  H_CUDA(cudaDeviceSynchronize());  // the builder runs on a workspace stream, which the legacy stream does not order
  for (uint32_t i = 0; i < count; ++i) h->node_level[new_ids[i]] = lvs[i];
  h->up_rows = up;
  rc = hnsw_insert_ids(h, new_ids, 0, true);
  if (rc) return rc;
  if (out_ids) std::copy(new_ids.begin(), new_ids.end(), out_ids);
  return 0;
}

// Drops every removed id.  Live id j becomes j - #{removed ids < j}; the upper-layer rows of removed ids go too.  The
// map is monotone, so stored neighbour order, edge distances and the entry rule are unchanged.  Capacity is kept.
extern "C" int cozo_gpu_hnsw_compact(cozo_gpu_hnsw_t* h, uint32_t* old_to_new) {
  if (!h) return set_error(COZO_GPU_EINVAL, "null index handle");
  int rc = ensure_init();
  if (rc) return rc;
  if (h->f64) return set_error(COZO_GPU_EUNSUP, "F64 indexes are search-only on the device: re-stage after a mutation");
  HnswDev& g = h->dev;
  const uint32_t n0 = g.n;
  std::vector<uint32_t> map(n0);
  uint32_t n1 = 0, first = n0;
  for (uint32_t j = 0; j < n0; ++j) {
    const bool keep = j >= h->live.size() || h->live[j];
    map[j] = keep ? n1++ : NONE;
    if (!keep && first == n0) first = j;
  }
  if (n1 == n0) {  // nothing removed: nothing moves
    if (old_to_new) std::copy(map.begin(), map.end(), old_to_new);
    return 0;
  }
  // removed ids exist only after cozo_gpu_hnsw_remove, which made the build state (degrees, distances, owners)
  // an asynchronous search_dev may still be reading the rows about to move
  H_CUDA(cudaDeviceSynchronize());
  const uint32_t up0 = (uint32_t)h->up_rows;

  // scratch first, so that running out of memory leaves the index as it was
  DevScratch<uint32_t> d_map, keep, up_map, first_drop;
  DevScratch<uint8_t> cub_tmp;
  H_CUDA(cudaMalloc(&d_map.p, (size_t)n0 * 4));
  H_CUDA(cudaMalloc(&keep.p, ((size_t)up0 + 1) * 4));
  H_CUDA(cudaMalloc(&up_map.p, ((size_t)up0 + 1) * 4));
  H_CUDA(cudaMalloc(&first_drop.p, 4));
  size_t cub_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, keep.p, up_map.p, (int)(up0 + 1));
  H_CUDA(cudaMalloc(&cub_tmp.p, std::max<size_t>(cub_bytes, 16)));
  H_CUDA(cudaMemcpy(d_map.p, map.data(), (size_t)n0 * 4, cudaMemcpyHostToDevice));
  H_CUDA(cudaMemset(first_drop.p, 0xFF, 4));  // NONE: no upper row is dropped
  // the upper-row map: rows whose owner stays, in row order
  upper_keep_kernel<<<(up0 + 256) / 256, 256>>>(h->d_up_owner, up0, d_map.p, keep.p);
  H_CUDA(cudaGetLastError());
  cub::DeviceScan::ExclusiveSum(cub_tmp.p, cub_bytes, keep.p, up_map.p, (int)(up0 + 1));
  if (up0) upper_map_kernel<<<(up0 + 255) / 256, 256>>>(keep.p, up0, up_map.p, first_drop.p);
  H_CUDA(cudaGetLastError());
  uint32_t up1 = 0, up_first = NONE;
  H_CUDA(cudaMemcpy(&up1, up_map.p + up0, 4, cudaMemcpyDeviceToHost));
  H_CUDA(cudaMemcpy(&up_first, first_drop.p, 4, cudaMemcpyDeviceToHost));
  if (up_first == NONE) up_first = up0;

  rc = relabel_rows(h, TableMap{d_map.p}, map, first, n1, up_map.p, up_first, up1);
  if (rc) return rc;
  h->n_live = n1;
  if (old_to_new) std::copy(map.begin(), map.end(), old_to_new);
  return 0;
}

// hnsw_remove (hnsw.rs:728-868) for a batch of ids.
extern "C" int cozo_gpu_hnsw_remove(cozo_gpu_hnsw_t* h, const uint32_t* ids, uint32_t count) {
  if (!h || (count && !ids)) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (count == 0) return 0;
  HnswDev& g = h->dev;
  for (uint32_t i = 0; i < count; ++i)
    if (ids[i] >= g.n) return set_error(COZO_GPU_EINVAL, "id %u out of range", ids[i]);
  rc = hnsw_ensure_build_state(h);
  if (rc) return rc;
  uint32_t* d_ids = nullptr;
  H_CUDA(cudaMalloc(&d_ids, (size_t)count * 4));
  cudaMemcpy(d_ids, ids, (size_t)count * 4, cudaMemcpyHostToDevice);
  mark_dead_kernel<<<(count + 255) / 256, 256>>>(d_ids, count, h->d_dead);
  remove_compact_kernel<<<(g.n + 3) / 4, 128>>>(h->d_adj0, h->d_adj0_dist, h->d_deg0, g.s0, g.n, nullptr, h->d_dead);
  if (h->up_rows)
    remove_compact_kernel<<<(uint32_t)((h->up_rows + 3) / 4), 128>>>(h->d_adj_up, h->d_adj_up_dist, h->d_deg_up, g.su,
                                                                     (uint32_t)h->up_rows, h->d_up_owner, h->d_dead);
  cudaError_t e = cudaDeviceSynchronize();
  cudaFree(d_ids);
  if (e != cudaSuccess) return set_error(COZO_GPU_ECUDA, "remove failed: %s", cudaGetErrorString(e));
  for (uint32_t i = 0; i < count; ++i)
    if (h->live[ids[i]]) {
      h->live[ids[i]] = 0;
      h->n_live--;
    }
  // the entry point was removed: re-point to the first remaining row in key order (hnsw.rs:828-865)
  if (g.entry != NONE && !h->live[g.entry]) {
    uint32_t best = NONE;
    uint32_t top = 0;
    for (uint32_t i = 0; i < g.n; ++i)
      if (h->live[i] && (best == NONE || h->node_level[i] > top)) {
        best = i;
        top = h->node_level[i];
      }
    g.entry = best;
    g.top_level = best == NONE ? 0 : top;
    h->n_levels = g.top_level + 1;
  }
  return 0;
}

__global__ void clear_dead_kernel(const uint32_t* ids, uint32_t count, uint8_t* dead) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) dead[ids[i]] = 0;
}

// hnsw_put of a CHANGED vector under an existing key (hnsw.rs:175-182: the hash differs, so the old
// vector is removed and the new one inserted).  The node keeps its id and its layer (the reference
// draws a fresh level; the level law is the same either way).  Also revives removed ids.
extern "C" int cozo_gpu_hnsw_update(cozo_gpu_hnsw_t* h, const uint32_t* ids, const float* vectors, uint32_t count,
                                    uint32_t ef_construction, int32_t keep_pruned_connections) {
  if (!h || (count && (!ids || !vectors))) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (count == 0) return 0;
  HnswDev& g = h->dev;
  std::vector<uint32_t> order(count);
  for (uint32_t i = 0; i < count; ++i) {
    if (ids[i] >= g.n) return set_error(COZO_GPU_EINVAL, "id %u out of range", ids[i]);
    order[i] = i;
  }
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ids[a] < ids[b]; });
  for (uint32_t i = 1; i < count; ++i)
    if (ids[order[i]] == ids[order[i - 1]]) return set_error(COZO_GPU_EINVAL, "id %u given twice", ids[order[i]]);
  if (ef_construction) h->ef_construction = ef_construction;
  if (h->ef_construction == 0) return set_error(COZO_GPU_EINVAL, "ef_construction must be set");
  if (keep_pruned_connections >= 0) h->keep_pruned = keep_pruned_connections;
  rc = hnsw_ensure_build_state(h);
  if (!rc) rc = check_build_smem(h);
  if (rc) return rc;
  // 1. drop the old vectors' links (no-op for ids that were already removed)
  std::vector<uint32_t> live_ids;
  for (uint32_t i = 0; i < count; ++i)
    if (h->live[ids[i]]) live_ids.push_back(ids[i]);
  if (!live_ids.empty()) {
    rc = cozo_gpu_hnsw_remove(h, live_ids.data(), (uint32_t)live_ids.size());
    if (rc) return rc;
  }
  // 2. new payloads, revive
  rc = own_vectors(h);
  if (rc) return rc;
  for (uint32_t i = 0; i < count; ++i)
    H_CUDA(cudaMemcpy(h->d_vec + (size_t)ids[i] * g.ld, vectors + (size_t)i * g.dim, (size_t)g.dim * 4,
                      cudaMemcpyHostToDevice));
  uint32_t* d_ids = nullptr;
  H_CUDA(cudaMalloc(&d_ids, (size_t)count * 4));
  cudaMemcpy(d_ids, ids, (size_t)count * 4, cudaMemcpyHostToDevice);
  hnsw_codes_fill(h, 0, count, d_ids);
  clear_dead_kernel<<<(count + 255) / 256, 256>>>(d_ids, count, h->d_dead);
  cudaError_t e = cudaDeviceSynchronize();
  cudaFree(d_ids);
  if (e != cudaSuccess) return set_error(COZO_GPU_ECUDA, "update failed: %s", cudaGetErrorString(e));
  for (uint32_t i = 0; i < count; ++i) h->live[ids[i]] = 1;
  // 3. re-insert, one contiguous id run at a time (hnsw_insert_range links [begin,end) into the graph)
  for (uint32_t i = 0; i < count;) {
    uint32_t j = i + 1;
    while (j < count && ids[order[j]] == ids[order[j - 1]] + 1) ++j;
    rc = hnsw_insert_range(h, ids[order[i]], ids[order[j - 1]] + 1, 0);
    if (rc) return rc;
    i = j;
  }
  return 0;
}
