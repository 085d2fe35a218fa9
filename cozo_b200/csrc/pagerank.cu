// pagerank.cu — graph::page_rank as called from PageRank::run (fixed_rule/algos/pagerank.rs:29-56)
// on the HBM-resident CSR.  GAP-style pull iteration (graph 0.3.1, un-vendored; DESIGN.md §3.3):
//     new[u] = base + d * sum_{v in in(u)} contrib[v];  err += |new[u]-old[u]|;  contrib'[u] = new[u]/outdeg(u)
// f32 scores, Jacobi schedule, no dangling redistribution.
//
// Everything runs in "slot space": slot[v] = rank of v by out-degree, descending.  Scores,
// contributions, out-degrees and the rows of the in-CSR are slot-indexed; scores are un-permuted once
// at the end.  Two iteration engines over it:
//
//   mode 1            PROPAGATION BLOCKING with TMA-staged contribution tiles.  The random 4-byte gather
//     of the pull (one 32-byte L2 sector per in-edge) is replaced by streaming passes:
//       sources by slot:  H = the first NH slots (hub sources, ~30 % of an R-MAT's edges), their
//                         contributions live in shared memory where they are needed;
//                         M = the other sources with out-edges, in groups of GS consecutive slots.
//       K_A  pb_gather    per group: the group's GS contributions are staged in shared memory by
//                         cp.async.bulk (one 128 KB tile), the group's in-edge entries (u16 source index
//                         inside the tile, stored group-major) are streamed and the gathered values
//                         written back as a dense f32 stream `val` — 2 + 4 bytes per entry, coalesced.
//       K_B  pb_accumulate per bin (= WIN consecutive positions of the row-major in-edge order): the
//                         bin's entries are read from `val` (one contiguous piece per group) and dropped
//                         at their u16 position inside a shared-memory window; then every row of the bin
//                         is summed from the window in stored order.  4 + 2 bytes per entry.
//       K_S  pb_straddle  rows longer than a window: their per-bin partial sums added in bin order.
//       K_F  pb_final     per row: the hub part sum_{v in H} contrib[v] through a shared-memory copy of
//                         the hub contributions (u16 index per entry, 2 bytes; a lane per row of at most 64
//                         entries, the warp per longer row), + the M part, new score, error, new contribution.
//     No atomics on floating point anywhere: sums have a fixed order, results are bit-reproducible.
//   mode 0 (default)  the round-1 gather pull (one persistent launch, L2 eviction hints).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <vector>

#include "graph_host.hpp"
#include "pagerank_pb.cuh"

namespace cozo {

constexpr uint32_t HUB_T = 4096;   // mode 0: rows longer than this are cut into HUB_CHUNK pieces, one warp each
constexpr uint32_t BLK_CAP = 256;  // mode 0: in-edges of a warp's mini-block (8 gathers per lane in flight)
constexpr uint32_t BLK_ROWS = 32;  // mode 0: rows per mini-block: one lane sums one row
constexpr uint32_t HUB_CHUNK = 4096;

struct PrState {
  uint32_t n = 0;
  uint64_t m = 0;
  // ---- slot space (both engines) ----------------------------------------------------------------
  uint32_t* slot = nullptr;                          // [n] original id -> slot
  uint32_t *in_ptr = nullptr, *in_idx = nullptr;     // in-CSR in slot space ([n+1], [m]), rows sorted by source slot
  uint32_t* od = nullptr;                            // [n] out-degree by slot
  // ---- mode 0 work lists ---------------------------------------------------------------------------
  bool v6_ready = false;
  uint32_t *hubs = nullptr, *blk_start = nullptr, *med_rows = nullptr;
  uint32_t *hub_chunk_ptr = nullptr, *chunk_beg = nullptr, *chunk_end = nullptr;
  uint32_t n_hubs = 0, n_blk = 0, n_med = 0, n_chunks = 0;
  // ---- mode 1 (propagation blocking) ------------------------------------------------------------
  bool pb_ready = false;
  uint32_t NH = 0, GS = 0, WIN = 0, G = 0, NB = 0;
  uint64_t Mtot = 0, Htot = 0, Mpad = 0;
  uint32_t *hptr = nullptr, *mptr = nullptr;  // [n+1] row pointers of the hub part / the M part
  uint16_t* hub_idx = nullptr;                // [Htot] hub source slots, row-major
  uint16_t* a_src = nullptr;                  // [Mpad] group-major: source index inside the group's tile
  uint16_t* b_pos = nullptr;                  // [Mpad] group-major: position inside the bin's window
  uint32_t* ctab = nullptr;                   // [(NB+1) x G] first group-major index of cell (bin, group)
  uint32_t* rowstart = nullptr;               // [NB+1] first row whose M part starts at or after bin*WIN
  uint4* items = nullptr;                     // K_A work items {group, begin, end, 0}
  uint32_t n_items = 0;
};

void pr_state_free(PrState* p) {
  if (!p) return;
  void* ptrs[] = {p->slot, p->in_ptr, p->in_idx, p->od, p->hubs, p->blk_start, p->med_rows, p->hub_chunk_ptr,
                  p->chunk_beg, p->chunk_end, p->hptr, p->mptr, p->hub_idx, p->a_src, p->b_pos, p->ctab,
                  p->rowstart, p->items};
  for (void* q : ptrs)
    if (q) cudaFree(q);
  delete p;
}

#define P_CUDA(call)                                                                                 \
  do {                                                                                               \
    cudaError_t _e = (call);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return set_error(_e == cudaErrorMemoryAllocation ? COZO_GPU_ENOMEM : COZO_GPU_ECUDA,            \
                       "%s failed: %s (pagerank.cu:%d)", #call, cudaGetErrorString(_e), __LINE__);    \
  } while (0)

// ---- slot space ---------------------------------------------------------------------------------------
__global__ void pr_init_kernel(const uint32_t* __restrict__ od, uint32_t n, float init, float* scores, float* contrib) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  scores[r] = init;
  const uint32_t d = od[r];
  contrib[r] = d ? init / (float)d : 0.f;  // d==0: value is never read (no out edge leads anywhere)
}
__global__ void pr_slot_kernel(const uint32_t* perm, uint32_t n, uint32_t* slot) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) slot[perm[r]] = r;
}
__global__ void pr_degkey_kernel(const uint32_t* out_ptr, uint32_t n, uint32_t* key, uint32_t* val) {
  uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u < n) {
    key[u] = 0xFFFFFFFFu - (out_ptr[u + 1] - out_ptr[u]);  // ascending sort => descending out-degree
    val[u] = u;
  }
}
__global__ void pr_degrees_kernel(const uint32_t* out_ptr, const uint32_t* in_ptr, const uint32_t* slot, uint32_t n,
                                  uint32_t* od_slot, uint32_t* in_cnt_slot) {
  uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n) return;
  const uint32_t r = slot[u];
  od_slot[r] = out_ptr[u + 1] - out_ptr[u];
  in_cnt_slot[r] = in_ptr[u + 1] - in_ptr[u];
}
// one warp per original destination row: key = (slot[dst] << 32) | slot[src] for each in-edge
__global__ void pr_edge_keys_kernel(const uint32_t* __restrict__ in_ptr, const uint32_t* __restrict__ in_idx,
                                    const uint32_t* __restrict__ slot, uint32_t n, unsigned long long* keys) {
  const uint32_t w = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const unsigned long long hi = (unsigned long long)slot[w] << 32;
  for (uint32_t e = in_ptr[w] + lane; e < in_ptr[w + 1]; e += 32) keys[e] = hi | slot[in_idx[e]];
}
__global__ void pr_low_word_kernel(const unsigned long long* keys, uint64_t m, uint32_t* lo) {
  uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) lo[e] = (uint32_t)(keys[e] & 0xFFFFFFFFull);
}
__global__ void pr_unpermute_kernel(const float* __restrict__ scores_slot, const uint32_t* __restrict__ slot, uint32_t n,
                                    float* out) {
  uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u < n) out[u] = scores_slot[slot[u]];
}

static int pr_stage_slots(cozo_gpu_graph* g, PrState* st) {
  const uint32_t n = g->n;
  const uint64_t m = g->m;
  const size_t np1 = (size_t)n + 1, mm = std::max<uint64_t>(m, 1);
  DevBuf key, key2, val, perm, tmp2;
  P_CUDA(cudaMalloc(&key.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&key2.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&val.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&perm.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&st->slot, (size_t)n * 4));
  P_CUDA(cudaMalloc(&st->od, (size_t)n * 4));
  P_CUDA(cudaMalloc(&st->in_ptr, np1 * 4));
  P_CUDA(cudaMalloc(&st->in_idx, mm * 4));
  pr_degkey_kernel<<<(n + 255) / 256, 256>>>(g->out_ptr, n, key.as<uint32_t>(), val.as<uint32_t>());
  size_t sb = 0, sb2 = 0, sb3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sb, key.as<uint32_t>(), key2.as<uint32_t>(), val.as<uint32_t>(),
                                  perm.as<uint32_t>(), (int)n);
  cub::DeviceScan::ExclusiveSum(nullptr, sb2, st->in_ptr, st->in_ptr, (int)np1);
  int end_bit = 32;
  while (end_bit < 64 && (n >> (end_bit - 32)) != 0) ++end_bit;
  if (m)
    cub::DeviceRadixSort::SortKeys(nullptr, sb3, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)m, 0,
                                   end_bit);
  sb = std::max(sb, std::max(sb2, sb3));
  P_CUDA(cudaMalloc(&tmp2.p, sb));
  {
    size_t t = sb;
    cub::DeviceRadixSort::SortPairs(tmp2.p, t, key.as<uint32_t>(), key2.as<uint32_t>(), val.as<uint32_t>(),
                                    perm.as<uint32_t>(), (int)n);
  }
  pr_slot_kernel<<<(n + 255) / 256, 256>>>(perm.as<uint32_t>(), n, st->slot);
  P_CUDA(cudaMemset(st->in_ptr, 0, np1 * 4));
  pr_degrees_kernel<<<(n + 255) / 256, 256>>>(g->out_ptr, g->in_ptr, st->slot, n, st->od, st->in_ptr);
  {
    size_t t = sb;
    cub::DeviceScan::ExclusiveSum(tmp2.p, t, st->in_ptr, st->in_ptr, (int)np1);
  }
  if (m) {
    DevBuf k1, k2;
    P_CUDA(cudaMalloc(&k1.p, m * 8));
    P_CUDA(cudaMalloc(&k2.p, m * 8));
    pr_edge_keys_kernel<<<(uint32_t)(((uint64_t)n * 32 + 255) / 256), 256>>>(g->in_ptr, g->in_idx, st->slot, n,
                                                                             k1.as<unsigned long long>());
    size_t t = sb;
    cub::DeviceRadixSort::SortKeys(tmp2.p, t, k1.as<unsigned long long>(), k2.as<unsigned long long>(), (int)m, 0,
                                   end_bit);
    pr_low_word_kernel<<<(uint32_t)((m + 255) / 256), 256>>>(k2.as<unsigned long long>(), m, st->in_idx);
  }
  P_CUDA(cudaGetLastError());
  P_CUDA(cudaDeviceSynchronize());
  return 0;
}

// =========================================================================================================
// mode 0: gather pull (round 1, v6)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float ldg_f32_hint(const float* a, uint64_t pol) {
  float v;
  asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(a), "l"(pol));
  return v;
}
__device__ __forceinline__ uint32_t ldg_u32_hint(const uint32_t* a, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(a), "l"(pol));
  return v;
}

struct PrArgs {
  const uint32_t *in_ptr, *in_idx, *od;  // slot-space in-CSR and out-degrees
  const uint32_t *blk_start, *med_rows, *chunk_beg, *chunk_end;
  uint32_t n_blk, n_med, n_chunks;
  uint32_t dynamic;  // 1: warps draw work items from device counters
  float base, damping;
  const float* contrib_old;
  float *contrib_new, *scores, *partial;
  unsigned long long* err;  // err[0]; the three work counters follow at err + 1
};

// a warp sums contrib over in_idx[b, en): 8 independent gathers per lane in flight, shuffle tree
__device__ __forceinline__ float pr_warp_row_sum(const PrArgs& a, uint32_t b, uint32_t en, int lane, uint64_t keep,
                                                 uint64_t stream) {
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  uint32_t k = b + lane;
  for (; k + 224 < en; k += 256) {
    uint32_t i[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) i[j] = ldg_u32_hint(a.in_idx + k + 32 * j, stream);
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] += ldg_f32_hint(a.contrib_old + i[j], keep);
  }
  for (; k < en; k += 32) s[0] += ldg_f32_hint(a.contrib_old + ldg_u32_hint(a.in_idx + k, stream), keep);
  return warp_sum(((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7])));
}

struct PrCursor {
  uint32_t cur, end, stride;
};
__device__ __forceinline__ bool pr_next(PrCursor& c, uint32_t n_items, uint32_t* ctr, uint32_t batch, bool dynamic,
                                        int lane) {
  if (!dynamic) {
    if (c.cur >= n_items) return false;
    c.end = c.cur + 1;  // one item; the caller advances by stride
    return true;
  }
  uint32_t v = 0;
  if (lane == 0) v = atomicAdd(ctr, batch);
  v = __shfl_sync(0xffffffffu, v, 0);
  if (v >= n_items) return false;
  c.cur = v;
  c.end = min(v + batch, n_items);
  return true;
}

// ONE persistent launch per iteration: hub chunks -> medium rows -> CSR-stream mini-blocks (DESIGN.md §3.3)
template <int WARPS, int MINB>
__global__ void __launch_bounds__(WARPS * 32, MINB) pr_pull_kernel(const PrArgs a) {
  __shared__ float vals_all[WARPS][BLK_CAP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* vals = vals_all[warp];
  const uint64_t keep = l2_policy_evict_last();
  const uint64_t stream = l2_policy_evict_first();
  const uint32_t wglobal = blockIdx.x * WARPS + warp, wtotal = gridDim.x * WARPS;
  const bool dyn = a.dynamic != 0;
  uint32_t* ctr = reinterpret_cast<uint32_t*>(a.err + 1);
  unsigned long long e = 0;
  PrCursor c{wglobal, 0, wtotal};
  while (pr_next(c, a.n_chunks, ctr + 0, 1, dyn, lane)) {
    for (uint32_t i = c.cur; i < c.end; ++i) {
      const float s = pr_warp_row_sum(a, a.chunk_beg[i], a.chunk_end[i], lane, keep, stream);
      if (lane == 0) a.partial[i] = s;
    }
    c.cur += c.stride;
  }
  c = PrCursor{wglobal, 0, wtotal};
  while (pr_next(c, a.n_med, ctr + 1, 2, dyn, lane)) {
    for (uint32_t i = c.cur; i < c.end; ++i) {
      const uint32_t r = a.med_rows[i];
      const float s = pr_warp_row_sum(a, a.in_ptr[r], a.in_ptr[r + 1], lane, keep, stream);
      if (lane == 0) {
        const float nw = a.base + a.damping * s;
        e += err_fixed(nw, a.scores[r]);
        a.scores[r] = nw;
        const uint32_t od = a.od[r];
        a.contrib_new[r] = od ? nw / (float)od : 0.f;
      }
    }
    c.cur += c.stride;
  }
  c = PrCursor{wglobal, 0, wtotal};
  while (pr_next(c, a.n_blk, ctr + 2, 8, dyn, lane)) {
    for (uint32_t blk = c.cur; blk < c.end; ++blk) {
      const uint32_t r0 = a.blk_start[2 * blk], r1 = a.blk_start[2 * blk + 1];
      const uint32_t nrows = r1 - r0;
      uint32_t lo = 0, hi = 0;
      if ((uint32_t)lane < nrows) {
        lo = a.in_ptr[r0 + lane];
        hi = a.in_ptr[r0 + lane + 1];
      }
      const uint32_t e0 = __shfl_sync(0xffffffffu, lo, 0);
      const uint32_t e1 = __shfl_sync(0xffffffffu, hi, nrows - 1);
      uint32_t idx[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t k = e0 + lane + 32 * j;
        idx[j] = k < e1 ? ldg_u32_hint(a.in_idx + k, stream) : NONE;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) vals[lane + 32 * j] = idx[j] != NONE ? ldg_f32_hint(a.contrib_old + idx[j], keep) : 0.f;
      __syncwarp();
      if ((uint32_t)lane < nrows) {
        const uint32_t r = r0 + lane;
        float s = 0.f;
        for (uint32_t j = lo - e0; j < hi - e0; ++j) s += vals[j];
        const float nw = a.base + a.damping * s;
        e += err_fixed(nw, a.scores[r]);
        a.scores[r] = nw;
        const uint32_t od = a.od[r];
        a.contrib_new[r] = od ? nw / (float)od : 0.f;
      }
      __syncwarp();
    }
    c.cur += c.stride;
  }
  block_add_err(e, a.err);
}

// one thread per hub row adds its chunk partials in chunk order (deterministic)
__global__ void __launch_bounds__(256) pr_hub_final_kernel(const uint32_t* __restrict__ hubs, uint32_t n_hubs,
                                                           const uint32_t* __restrict__ hub_chunk_ptr,
                                                           const float* __restrict__ partial,
                                                           const uint32_t* __restrict__ od, float base, float damping,
                                                           float* __restrict__ contrib_new,
                                                           float* __restrict__ scores, unsigned long long* err) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long e = 0;
  if (i < n_hubs) {
    const uint32_t u = hubs[i];
    float s = 0.f;
    for (uint32_t c = hub_chunk_ptr[i]; c < hub_chunk_ptr[i + 1]; ++c) s += partial[c];
    const float nw = base + damping * s;
    e = err_fixed(nw, scores[u]);
    scores[u] = nw;
    const uint32_t d = od[u];
    contrib_new[u] = d ? nw / (float)d : 0.f;
  }
  block_add_err(e, err);
}

template <class T>
static int upload(T*& dst, const std::vector<T>& v) {
  P_CUDA(cudaMalloc(&dst, std::max<size_t>(v.size(), 2) * sizeof(T)));
  if (!v.empty()) P_CUDA(cudaMemcpy(dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

static int pr_stage_v6(PrState* st) {
  const uint32_t n = st->n;
  const size_t np1 = (size_t)n + 1;
  std::vector<uint32_t> hin(np1);
  P_CUDA(cudaMemcpy(hin.data(), st->in_ptr, np1 * 4, cudaMemcpyDeviceToHost));
  std::vector<uint32_t> blocks, hubs, med;
  uint32_t r = 0;
  while (r < n) {
    const uint32_t d0 = hin[r + 1] - hin[r];
    if (d0 > HUB_T) {
      hubs.push_back(r++);
      continue;
    }
    if (d0 > BLK_CAP) {
      med.push_back(r++);
      continue;
    }
    const uint32_t r0 = r;
    while (r < n && r - r0 < BLK_ROWS && hin[r + 1] - hin[r] <= BLK_CAP && hin[r + 1] - hin[r0] <= BLK_CAP) ++r;
    blocks.push_back(r0);
    blocks.push_back(r);
  }
  std::vector<uint32_t> cptr(1, 0), cbeg, cend;
  for (uint32_t hr : hubs) {
    for (uint32_t b = hin[hr]; b < hin[hr + 1]; b += HUB_CHUNK) {
      cbeg.push_back(b);
      cend.push_back(std::min(b + HUB_CHUNK, hin[hr + 1]));
    }
    cptr.push_back((uint32_t)cbeg.size());
  }
  st->n_med = (uint32_t)med.size();
  st->n_blk = (uint32_t)(blocks.size() / 2);
  st->n_hubs = (uint32_t)hubs.size();
  st->n_chunks = (uint32_t)cbeg.size();
  int rc = upload(st->med_rows, med);
  if (!rc) rc = upload(st->blk_start, blocks);
  if (!rc) rc = upload(st->hubs, hubs);
  if (!rc) rc = upload(st->hub_chunk_ptr, cptr);
  if (!rc) rc = upload(st->chunk_beg, cbeg);
  if (!rc) rc = upload(st->chunk_end, cend);
  if (rc) return rc;
  st->v6_ready = true;
  return 0;
}

// =========================================================================================================
// mode 1: propagation blocking
// ---- the four passes of an iteration: thin __global__ wrappers around the bodies in pagerank_pb.cuh --------------
__global__ void __launch_bounds__(1024, 1) pb_gather_kernel(const PbArgs a) {
  extern __shared__ __align__(128) uint8_t pb_smem[];
  pb_gather_body(a, pb_smem);
}
template <int THREADS>
__global__ void __launch_bounds__(THREADS) pb_accumulate_kernel(const PbArgs a) {
  extern __shared__ __align__(128) uint8_t pb_smem[];
  pb_accumulate_body<THREADS>(a, pb_smem);
}
__global__ void __launch_bounds__(KF_THREADS) pb_final_kernel(const PbArgs a) {
  extern __shared__ __align__(128) uint8_t pb_smem[];
  pb_final_body(a, pb_smem);
}

static int pr_stage_pb(PrState* st, uint32_t NH, uint32_t GS, uint32_t WIN) {
  const uint32_t n = st->n;
  const uint64_t m = st->m;
  const size_t np1 = (size_t)n + 1;
  st->NH = NH = std::min(NH, n);
  st->GS = GS;
  st->WIN = WIN;
  // a handle may be re-staged with another geometry: nothing derived from the previous one may survive an early return
  // (the all-hub case below used to leave n_items / Mpad of the old blocking behind -> K_A launched on freed tables)
  st->n_items = 0;
  st->Mpad = 0;
  st->G = st->NB = 0;
  st->Htot = st->Mtot = 0;
  P_CUDA(cudaMalloc(&st->hptr, np1 * 4));
  P_CUDA(cudaMalloc(&st->mptr, np1 * 4));
  pb_row_split_kernel<<<(uint32_t)((np1 + 255) / 256), 256>>>(st->in_ptr, st->in_idx, n, NH, st->hptr, st->mptr);
  {
    size_t sb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, sb, st->hptr, st->hptr, (int)np1);
    DevBuf tmp;
    P_CUDA(cudaMalloc(&tmp.p, std::max<size_t>(sb, 16)));
    cub::DeviceScan::ExclusiveSum(tmp.p, sb, st->hptr, st->hptr, (int)np1);
    cub::DeviceScan::ExclusiveSum(tmp.p, sb, st->mptr, st->mptr, (int)np1);
    P_CUDA(cudaDeviceSynchronize());
  }
  uint32_t ht = 0, mt = 0;
  P_CUDA(cudaMemcpy(&ht, st->hptr + n, 4, cudaMemcpyDeviceToHost));
  P_CUDA(cudaMemcpy(&mt, st->mptr + n, 4, cudaMemcpyDeviceToHost));
  st->Htot = ht;
  st->Mtot = mt;
  if ((uint64_t)ht + mt != m) return set_error(COZO_GPU_ECUDA, "internal: pagerank split lost edges");
  st->G = n > NH ? (uint32_t)(((uint64_t)(n - NH) + GS - 1) / GS) : 0;
  // groups beyond the last source with an out-edge are empty; trim them (slots are sorted by out-degree)
  {
    uint32_t lo = 0, hi = n;  // first slot with out-degree 0
    while (lo < hi) {
      uint32_t mid = lo + ((hi - lo) >> 1), d = 0;
      P_CUDA(cudaMemcpy(&d, st->od + mid, 4, cudaMemcpyDeviceToHost));
      if (d > 0) lo = mid + 1;
      else hi = mid;
    }
    const uint32_t n_src = lo;
    st->G = n_src > NH ? (uint32_t)(((uint64_t)(n_src - NH) + GS - 1) / GS) : 0;
  }
  st->NB = (uint32_t)((st->Mtot + WIN - 1) / WIN);
  P_CUDA(cudaMalloc(&st->hub_idx, std::max<uint64_t>(st->Htot, 8) * 2));
  const uint32_t G = st->G, NB = st->NB;
  if (st->Mtot == 0 || G == 0) {
    if (st->Mtot) return set_error(COZO_GPU_ECUDA, "internal: pagerank groups");
    // every source is a hub source: only K_F runs
    DevBuf key, val;
    pb_emit_kernel<<<(uint32_t)(((uint64_t)n * 32 + 255) / 256), 256>>>(st->in_ptr, st->in_idx, st->hptr, st->mptr, n, NH,
                                                                       GS, st->hub_idx, nullptr, nullptr);
    P_CUDA(cudaGetLastError());
    P_CUDA(cudaDeviceSynchronize());
    st->pb_ready = true;
    return 0;
  }
  if ((uint64_t)(NB + 1) * G > (1ull << 30))
    return set_error(COZO_GPU_EUNSUP, "pagerank tables too large (%u bins x %u groups): raise pagerank.window / pagerank.group_slots",
                     NB, G);
  const uint64_t M = st->Mtot;
  DevBuf key, key2, val, val2, tmp, gfirst_d, gbase_d, gend_d;
  P_CUDA(cudaMalloc(&key.p, M * 4));
  P_CUDA(cudaMalloc(&key2.p, M * 4));
  P_CUDA(cudaMalloc(&val.p, M * 8));
  P_CUDA(cudaMalloc(&val2.p, M * 8));
  pb_emit_kernel<<<(uint32_t)(((uint64_t)n * 32 + 255) / 256), 256>>>(st->in_ptr, st->in_idx, st->hptr, st->mptr, n, NH, GS,
                                                                     st->hub_idx, key.as<uint32_t>(),
                                                                     val.as<unsigned long long>());
  P_CUDA(cudaGetLastError());
  int gbits = 1;
  while ((1u << gbits) < G) ++gbits;
  {
    size_t sb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sb, key.as<uint32_t>(), key2.as<uint32_t>(), val.as<unsigned long long>(),
                                    val2.as<unsigned long long>(), (int)M, 0, gbits);
    P_CUDA(cudaMalloc(&tmp.p, std::max<size_t>(sb, 16)));
    cub::DeviceRadixSort::SortPairs(tmp.p, sb, key.as<uint32_t>(), key2.as<uint32_t>(), val.as<unsigned long long>(),
                                    val2.as<unsigned long long>(), (int)M, 0, gbits);  // stable: Mpos order kept per group
  }
  // group extents (host: G is small)
  P_CUDA(cudaMalloc(&gfirst_d.p, (size_t)G * 4));
  P_CUDA(cudaMemset(gfirst_d.p, 0xFF, (size_t)G * 4));
  pb_group_bounds_kernel<<<(uint32_t)((M + 255) / 256), 256>>>(key2.as<uint32_t>(), M, gfirst_d.as<uint32_t>());
  std::vector<uint32_t> gfirst(G), gcnt(G), gbase(G), gend(G);
  P_CUDA(cudaMemcpy(gfirst.data(), gfirst_d.p, (size_t)G * 4, cudaMemcpyDeviceToHost));
  {
    uint32_t next = (uint32_t)M;
    for (uint32_t g = G; g-- > 0;) {
      if (gfirst[g] == NONE) gfirst[g] = next;  // empty group
      gcnt[g] = next - gfirst[g];
      next = gfirst[g];
    }
  }
  uint64_t pad = 0;
  std::vector<uint4> items;
  const uint32_t CH = (uint32_t)std::max<int64_t>(1024, get_option("pagerank.chunk", 262144)) & ~7u;
  for (uint32_t g = 0; g < G; ++g) {
    gbase[g] = (uint32_t)pad;
    gend[g] = gbase[g] + gcnt[g];
    const uint32_t padded = (gcnt[g] + 7u) & ~7u;
    for (uint32_t c = 0; c < padded; c += CH)
      items.push_back(make_uint4(g, gbase[g] + c, gbase[g] + std::min(padded, c + CH), 0));
    pad += padded;
    if (pad >= 0xFFFFFFF0ull) return set_error(COZO_GPU_EUNSUP, "pagerank: too many edges for 32-bit positions");
  }
  st->Mpad = pad;
  st->n_items = (uint32_t)items.size();
  P_CUDA(cudaMemcpy(gfirst_d.p, gfirst.data(), (size_t)G * 4, cudaMemcpyHostToDevice));
  P_CUDA(cudaMalloc(&gbase_d.p, (size_t)G * 4));
  P_CUDA(cudaMalloc(&gend_d.p, (size_t)G * 4));
  P_CUDA(cudaMemcpy(gbase_d.p, gbase.data(), (size_t)G * 4, cudaMemcpyHostToDevice));
  P_CUDA(cudaMemcpy(gend_d.p, gend.data(), (size_t)G * 4, cudaMemcpyHostToDevice));
  P_CUDA(cudaMalloc(&st->a_src, (pad + 8) * 2));
  P_CUDA(cudaMalloc(&st->b_pos, (pad + 8) * 2));
  P_CUDA(cudaMemset(st->a_src, 0, (pad + 8) * 2));
  P_CUDA(cudaMemset(st->b_pos, 0, (pad + 8) * 2));
  P_CUDA(cudaMalloc(&st->ctab, (size_t)(NB + 1) * G * 4));
  pb_ctab_init_kernel<<<(uint32_t)(((uint64_t)(NB + 1) * G + 255) / 256), 256>>>(st->ctab, NB + 1, G, gend_d.as<uint32_t>());
  pb_place_kernel<<<(uint32_t)((M + 255) / 256), 256>>>(key2.as<uint32_t>(), val2.as<unsigned long long>(), M,
                                                        gfirst_d.as<uint32_t>(), gbase_d.as<uint32_t>(), WIN, G, st->a_src,
                                                        st->b_pos, st->ctab);
  P_CUDA(cudaMalloc(&st->rowstart, (size_t)(NB + 1) * 4));
  pb_rowstart_kernel<<<(NB + 1 + 255) / 256, 256>>>(st->mptr, n, WIN, NB + 1, st->rowstart);
  P_CUDA(cudaMalloc(&st->items, std::max<size_t>(items.size(), 1) * sizeof(uint4)));
  P_CUDA(cudaMemcpy(st->items, items.data(), items.size() * sizeof(uint4), cudaMemcpyHostToDevice));
  P_CUDA(cudaGetLastError());
  P_CUDA(cudaDeviceSynchronize());
  st->pb_ready = true;
  return 0;
}

}  // namespace cozo

using namespace cozo;

extern "C" int cozo_gpu_pagerank(cozo_gpu_graph_t* g, float damping, double tol, uint32_t max_iter,
                                 float* out_scores, uint32_t* out_iters, double* out_err, double* out_kernel_ms,
                                 const volatile int* poison) {
  if (!g || !out_scores) return set_error(COZO_GPU_EINVAL, "null argument");
  if (max_iter == 0) return set_error(COZO_GPU_EINVAL, "iterations must be positive");  // pos_integer_option
  int rc = ensure_init();
  if (rc) return rc;
  if (out_iters) *out_iters = 0;
  if (out_err) *out_err = 0;
  if (out_kernel_ms) *out_kernel_ms = 0;
  const uint32_t n = g->n;
  if (n == 0) return 0;  // pagerank.rs:43-45
  const DeviceInfo& di = device_info();
  // default = the round-1 gather pull; "pagerank.mode" = 1 selects propagation blocking (DESIGN.md §3.3)
  const int64_t mode = get_option("pagerank.mode", 0);
  uint32_t NH = (uint32_t)std::min<int64_t>(65536, std::max<int64_t>(0, get_option("pagerank.hub_slots", 16384)));
  NH &= ~3u;
  uint32_t GS = (uint32_t)std::min<int64_t>(49152, std::max<int64_t>(64, get_option("pagerank.group_slots", 32768))) & ~3u;
  uint32_t WIN = (uint32_t)std::min<int64_t>(49152, std::max<int64_t>(64, get_option("pagerank.window", 24576)));
  // ---- lazily built layouts (the staged graph is shared by concurrent callers) --------------------------
  PrState* st = nullptr;
  {
    std::lock_guard<std::mutex> lk(g->pr_mu);
    if (!g->pr) {
      auto* p = new PrState();
      p->n = n;
      p->m = g->m;
      rc = pr_stage_slots(g, p);
      if (rc) {
        pr_state_free(p);
        return rc;
      }
      g->pr = p;
    }
    st = g->pr;
    if (mode == 0 && !st->v6_ready) rc = pr_stage_v6(st);
    if (mode != 0 && (!st->pb_ready || st->NH != std::min(NH, n) || st->GS != GS || st->WIN != WIN)) {
      if (st->pb_ready) {  // options changed: rebuild the blocking
        void* ptrs[] = {st->hptr, st->mptr, st->hub_idx, st->a_src, st->b_pos, st->ctab, st->rowstart, st->items};
        for (void* q : ptrs)
          if (q) cudaFree(q);
        st->hptr = st->mptr = st->ctab = st->rowstart = nullptr;
        st->hub_idx = st->a_src = st->b_pos = nullptr;
        st->items = nullptr;
        st->pb_ready = false;
      }
      rc = pr_stage_pb(st, NH, GS, WIN);
    }
    if (rc) return rc;
  }
  cudaStream_t sm = nullptr;
  P_CUDA(cudaStreamCreateWithFlags(&sm, cudaStreamNonBlocking));
  struct StreamGuard {
    cudaStream_t s;
    ~StreamGuard() { cudaStreamDestroy(s); }
  } sguard{sm};
  const size_t slack = 65536 + 8;  // K_A's tile copies may read past n (rounded up to 16 bytes)
  DevBuf scores, c0, c1, err, partial, unperm, val, msum, pa, pz;
  P_CUDA(cudaMalloc(&scores.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&c0.p, ((size_t)n + slack) * 4));
  P_CUDA(cudaMalloc(&c1.p, ((size_t)n + slack) * 4));
  P_CUDA(cudaMemsetAsync(c0.p, 0, ((size_t)n + slack) * 4, sm));
  P_CUDA(cudaMemsetAsync(c1.p, 0, ((size_t)n + slack) * 4, sm));
  P_CUDA(cudaMalloc(&unperm.p, (size_t)n * 4));
  P_CUDA(cudaMalloc(&err.p, 32));
  const float init = 1.0f / (float)n;
  const float base = (1.0f - damping) / (float)n;
  cudaEvent_t e0, e1;
  P_CUDA(cudaEventCreate(&e0));
  P_CUDA(cudaEventCreate(&e1));
  uint32_t launches = 0;
  PrArgs a{};
  PbArgs pb{};
  uint32_t grid0 = 0, wpc = 32, gridA = 0, gridB = 0, gridF = 0, threadsB = 512;
  size_t smemA = 0, smemB = 0, smemF = 0;
  if (mode == 0) {
    P_CUDA(cudaMalloc(&partial.p, (size_t)std::max(st->n_chunks, 1u) * 4));
    a.in_ptr = st->in_ptr;
    a.in_idx = st->in_idx;
    a.od = st->od;
    a.blk_start = st->blk_start;
    a.med_rows = st->med_rows;
    a.chunk_beg = st->chunk_beg;
    a.chunk_end = st->chunk_end;
    a.n_blk = st->n_blk;
    a.n_med = st->n_med;
    a.n_chunks = st->n_chunks;
    a.scores = scores.as<float>();
    a.partial = partial.as<float>();
    a.err = err.as<unsigned long long>();
    a.base = base;
    a.damping = damping;
    const int64_t warps = get_option("pagerank.warps", 32);
    const int64_t cps = std::max<int64_t>(1, get_option("pagerank.ctas_per_sm", warps == 32 ? 2 : 8));
    a.dynamic = get_option("pagerank.dynamic", 1) ? 1u : 0u;
    const uint64_t items = (uint64_t)st->n_blk + st->n_med + st->n_chunks;
    wpc = warps == 32 ? 32u : 8u;
    grid0 = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((items + wpc - 1) / wpc, (uint64_t)di.sm_count * (uint64_t)cps));
  } else {
    pb.n = n;
    pb.NH = st->NH;
    pb.GS = st->GS;
    pb.WIN = st->WIN;
    pb.G = st->G;
    pb.NB = st->NB;
    pb.hptr = st->hptr;
    pb.mptr = st->mptr;
    pb.od = st->od;
    pb.hub_idx = st->hub_idx;
    pb.a_src = st->a_src;
    pb.b_pos = st->b_pos;
    pb.ctab = st->ctab;
    pb.rowstart = st->rowstart;
    pb.items = st->items;
    pb.n_items = st->n_items;
    pb.scores = scores.as<float>();
    pb.base = base;
    pb.damping = damping;
    pb.err = err.as<unsigned long long>();
    P_CUDA(cudaMalloc(&msum.p, (size_t)n * 4));
    P_CUDA(cudaMemsetAsync(msum.p, 0, (size_t)n * 4, sm));  // rows without an M part keep 0
    P_CUDA(cudaMalloc(&val.p, (std::max<uint64_t>(st->Mpad, 8) + 8) * 4));
    P_CUDA(cudaMalloc(&pa.p, (size_t)std::max(st->NB, 1u) * 4));
    P_CUDA(cudaMalloc(&pz.p, (size_t)std::max(st->NB, 1u) * 4));
    P_CUDA(cudaMemsetAsync(pa.p, 0, (size_t)std::max(st->NB, 1u) * 4, sm));
    P_CUDA(cudaMemsetAsync(pz.p, 0, (size_t)std::max(st->NB, 1u) * 4, sm));
    pb.val = val.as<float>();
    pb.msum = msum.as<float>();
    pb.part_a = pa.as<float>();
    pb.part_z = pz.as<float>();
    smemA = (size_t)st->GS * 4 + 16;
    smemB = (size_t)st->WIN * 4 + ((size_t)2 * st->G + 2) * 4;
    smemF = (size_t)((st->NH + 3u) & ~3u) * 4 + 16 + (size_t)(KF_THREADS / 32) * KF_STAGE * 2;
    if (smemA > di.smem_optin || smemB > di.smem_optin || smemF > di.smem_optin)
      return set_error(COZO_GPU_EUNSUP, "pagerank blocking does not fit shared memory (%zu / %zu / %zu of %zu bytes)", smemA,
                       smemB, smemF, di.smem_optin);
    // the dynamic limit is the opt-in maximum minus the kernel's static shared memory (never lowered per call)
    auto raise_smem = [&](const void* fn, size_t need) -> int {
      cudaFuncAttributes fa;
      P_CUDA(cudaFuncGetAttributes(&fa, fn));
      if (need + fa.sharedSizeBytes > di.smem_optin)
        return set_error(COZO_GPU_EUNSUP, "pagerank blocking needs %zu + %zu B of shared memory (limit %zu)", need,
                         (size_t)fa.sharedSizeBytes, di.smem_optin);
      P_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(di.smem_optin - fa.sharedSizeBytes)));
      return 0;
    };
    if ((rc = raise_smem((const void*)pb_gather_kernel, smemA)) != 0) return rc;
    // a window above half of the shared memory leaves one CTA per SM: give it 32 warps instead of 16
    const bool bigB = smemB > di.smem_optin / 2 || get_option("pagerank.accumulate_threads", 0) == 1024;
    if ((rc = raise_smem(bigB ? (const void*)pb_accumulate_kernel<1024> : (const void*)pb_accumulate_kernel<512>, smemB)) != 0)
      return rc;
    if ((rc = raise_smem((const void*)pb_final_kernel, smemF)) != 0) return rc;
    int occB = 1, occF = 1;
    if (bigB) P_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occB, pb_accumulate_kernel<1024>, 1024, smemB));
    else P_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occB, pb_accumulate_kernel<512>, 512, smemB));
    threadsB = bigB ? 1024 : 512;
    P_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occF, pb_final_kernel, KF_THREADS, smemF));
    if (occB < 1 || occF < 1) return set_error(COZO_GPU_ECUDA, "pagerank kernels do not fit on an SM");
    gridA = std::max(1u, std::min<uint32_t>(st->n_items, (uint32_t)di.sm_count));
    gridB = std::max(1u, std::min<uint32_t>(st->NB, (uint32_t)di.sm_count * (uint32_t)occB));
    gridF = std::max(1u, std::min<uint32_t>((n + 127) / 128, (uint32_t)di.sm_count * (uint32_t)occF));
  }
  P_CUDA(cudaEventRecord(e0, sm));
  pr_init_kernel<<<(n + 255) / 256, 256, 0, sm>>>(st->od, n, init, scores.as<float>(), c0.as<float>());
  ++launches;
  float* cold = c0.as<float>();
  float* cnew = c1.as<float>();
  uint32_t iter = 0;
  unsigned long long herr_fx = 0;
  double herr = 0;
  int ret = 0;
  for (;;) {
    if (poisoned(poison)) {
      ret = set_error(COZO_GPU_EKILLED, "Running query is killed before completion");
      break;
    }
    cudaMemsetAsync(err.p, 0, 32, sm);
    if (mode == 0) {
      a.contrib_old = cold;
      a.contrib_new = cnew;
      if (wpc == 32) pr_pull_kernel<32, 2><<<grid0, 1024, 0, sm>>>(a);
      else pr_pull_kernel<8, 8><<<grid0, 256, 0, sm>>>(a);
      ++launches;
      if (st->n_hubs) {
        pr_hub_final_kernel<<<(st->n_hubs + 255) / 256, 256, 0, sm>>>(st->hubs, st->n_hubs, st->hub_chunk_ptr,
                                                                       partial.as<float>(), st->od, base, damping, cnew,
                                                                       scores.as<float>(), err.as<unsigned long long>());
        ++launches;
      }
    } else {
      pb.contrib_old = cold;
      pb.contrib_new = cnew;
      if (st->n_items) {
        pb_gather_kernel<<<gridA, 1024, smemA, sm>>>(pb);
        if (threadsB == 1024) pb_accumulate_kernel<1024><<<gridB, 1024, smemB, sm>>>(pb);
        else pb_accumulate_kernel<512><<<gridB, 512, smemB, sm>>>(pb);
        pb_straddle_kernel<<<(st->NB + 255) / 256, 256, 0, sm>>>(pb);
        launches += 3;
      }
      pb_final_kernel<<<gridF, KF_THREADS, smemF, sm>>>(pb);
      ++launches;
    }
    cudaError_t ce = cudaMemcpyAsync(&herr_fx, err.p, 8, cudaMemcpyDeviceToHost, sm);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(sm);
    if (ce != cudaSuccess) {
      ret = set_error(COZO_GPU_ECUDA, "pagerank iteration failed: %s", cudaGetErrorString(ce));
      break;
    }
    herr = (double)herr_fx / ERR_SCALE;
    std::swap(cold, cnew);
    ++iter;
    if (herr < tol || iter == max_iter) break;
  }
  if (!ret) {
    pr_unpermute_kernel<<<(n + 255) / 256, 256, 0, sm>>>(scores.as<float>(), st->slot, n, unperm.as<float>());
    ++launches;
  }
  cudaEventRecord(e1, sm);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (ret) return ret;
  P_CUDA(cudaMemcpyAsync(out_scores, unperm.p, (size_t)n * 4, cudaMemcpyDeviceToHost, sm));
  P_CUDA(cudaStreamSynchronize(sm));
  if (out_iters) *out_iters = iter;
  if (out_err) *out_err = herr;
  if (out_kernel_ms) *out_kernel_ms = ms;
  cozo_gpu_set_option("pagerank.last_launches", launches);
  return 0;
}
