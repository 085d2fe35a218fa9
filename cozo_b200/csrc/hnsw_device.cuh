// hnsw_device.cuh — device-side HNSW layer search shared by the batched k-NN
// kernel and the batched index builder.
//
// Semantics follow SessionTx::hnsw_search_level (runtime/hnsw.rs:539-587) with
// one warp per query:
//   * `found_nn` (max-queue bounded by ef) and `candidates` (min-queue) are ONE
//     sorted array in shared memory: found = the array, candidates = its not yet
//     expanded entries.  An admitted neighbour that was later evicted from
//     found_nn has dist >= furthest, so the reference pops it only to `break`
//     (hnsw.rs:562); dropping it changes nothing except on exact distance ties.
//   * the neighbours of one candidate are evaluated together; admission
//     (hnsw.rs:575-581) is applied in neighbour order with the live bound, so the
//     traversal, dist_evals and nodes_expanded equal the reference's.
//   * `visited` (hnsw.rs:549) is a per-warp bitmap in HBM, set with atomicOr and
//     cleared at the end of every layer (visit_clear), through a log of the ids
//     that were set or by sweeping the whole bitmap.
#pragma once
#include "common.cuh"
#include "hnsw_codes.cuh"

namespace cozo {

struct HnswDev {
  const float* vec;  // [n x ld] row-major f32, rows zero-padded to ld (multiple of 4)
  uint32_t n, dim, ld;
  int metric;
  const uint32_t* adj0;       // layer 0: [n x s0], ids packed at the front, NONE padded
  uint32_t s0;                // multiple of 32
  const uint32_t* upper_off;  // [n] first row in adj_up of the node's layer -1 list, NONE if layer 0 only
  const uint32_t* adj_up;     // [rows x su]; node on layers 1..t owns rows upper_off .. upper_off+t-1
  uint32_t su;                // multiple of 32
  uint32_t entry;             // NONE = empty index
  uint32_t top_level;         // entry lives on layer -top_level
  const uint8_t* codes;       // [n x code_ld] uint8 code rows (hnsw_codes.cuh); nullptr = no codes, nothing is pruned
  uint32_t code_ld;           // bytes per code row
};

// Per-phase clock64 totals of the warp-per-query search, compiled only with -DCOZO_HOP_CLOCKS (tools/hop_clocks.py):
// pop + adjacency read, visited test, code-ring waits, code scoring, f32-ring waits, f32 scoring + admissions.
enum HopPhase { HC_POP, HC_VISIT, HC_CWAIT, HC_CSCORE, HC_FWAIT, HC_FSCORE, HC_N };
#ifdef COZO_HOP_CLOCKS
#define HOP_T(t) long long t = clock64()
#define HOP_SET(t) (t = clock64())
#define HOP_ADD(w, k, t) ((w).clk[k] += (unsigned long long)(clock64() - (t)))
#else
#define HOP_T(t)
#define HOP_SET(t)
#define HOP_ADD(w, k, t)
#endif

struct WarpCtx {
  float* fd;       // smem: sorted distances (ascending)
  uint32_t* fi;    // smem: ids, bit31 = expanded
  uint32_t* pend;  // smem [32]: compacted unvisited neighbour ids of the current hop
  float* ring;     // smem: NS row buffers (bulk mode)
  uint64_t* bars;  // smem: NS mbarriers (bulk mode)
  uint32_t* vis;   // HBM: this warp's visited bitmap, all zero between layers
  uint32_t nwords;
  uint32_t* vlog;  // HBM: ids whose bit was set on this layer
  uint32_t logcap;
  uint32_t ns;     // ring stages
  // registers, warp-uniform
  uint32_t len, cursor, nlog;
  uint32_t head, phase;  // ring position / per-stage parity bits
  uint32_t dist_evals, nodes_expanded, nbr_reads;
  uint32_t pruned;  // evaluations whose f32 row was never fetched (prune_chunk)
  // code-row ring of the pruned search (used only when g.codes is set)
  uint8_t* cring;
  uint64_t* cbars;
  uint32_t cns, chead, cphase;
#ifdef COZO_HOP_CLOCKS
  unsigned long long clk[HC_N];
#endif
};

constexpr uint32_t EXPANDED = 0x80000000u;
constexpr uint32_t IDMASK = 0x7FFFFFFFu;

template <int METRIC>
__device__ __forceinline__ void accum(const float4& q, const float4& v, float& a, float& b) {
  if (METRIC == COZO_GPU_L2) {
    float dx = q.x - v.x, dy = q.y - v.y, dz = q.z - v.z, dw = q.w - v.w;
    a = fmaf(dx, dx, a);
    a = fmaf(dy, dy, a);
    a = fmaf(dz, dz, a);
    a = fmaf(dw, dw, a);
  } else {
    a = fmaf(q.x, v.x, a);
    a = fmaf(q.y, v.y, a);
    a = fmaf(q.z, v.z, a);
    a = fmaf(q.w, v.w, a);
    if (METRIC == COZO_GPU_COSINE) {
      b = fmaf(v.x, v.x, b);
      b = fmaf(v.y, v.y, b);
      b = fmaf(v.z, v.z, b);
      b = fmaf(v.w, v.w, b);
    }
  }
}

// VectorCache::dist (hnsw.rs:66-109): reduce the per-lane partials and apply the
// metric's final scalar step in f64, then round to the f32 ordering key.
template <int METRIC>
__device__ __forceinline__ float finish(float a, float b, float qnorm) {
  a = warp_sum(a);
  if (METRIC == COZO_GPU_L2) return a;
  if (METRIC == COZO_GPU_IP) return (float)(1.0 - (double)a);
  b = warp_sum(b);
  return (float)(1.0 - (double)a / sqrt((double)qnorm * (double)b));
}

// The register query (float4 q[NV], lane-strided) covers rows of up to 32 * 4 * 16 = 2048 floats; wider ones spill.
// Above that the query is a WideQuery (NV = 0): a pointer to the query zero-padded to ld, which the search kernels keep
// in shared memory and the builder's selection passes read from the index's own row.  The wide helpers below visit
// idx = lane + 32 i in the same order as the register ones, so a wide distance is the same formula.  Their loops step
// over warp-uniform bases with the element test inside, as the unrolled register loops do: a lane-dependent trip count
// would put divergent control flow before the warp reductions, and ptxas keeps values across it on the stack.
constexpr uint32_t REG_QUERY_MAX_LD = 2048;
constexpr uint32_t WIDE_RING_BYTES = 32768;  // per-warp f32 ring budget of the wide kernels: 2 stages of 16 KB rows
struct WideQuery {
  const float4* v;
};
template <int NV>
struct QueryOf {
  using type = float4[NV];
};
template <>
struct QueryOf<0> {
  using type = WideQuery;
};
constexpr int WIDE_CHUNK = 8;  // float4 per lane and row in flight in the ld.global form

template <int NV, int METRIC>
__device__ __forceinline__ float dist_smem(const WideQuery& q, const float4* row, int lane, int nvec4, float qnorm) {
  float a = 0.f, b = 0.f;
#pragma unroll 4
  for (int base = 0; base < nvec4; base += 32) {
    const int idx = base + lane;
    if (idx < nvec4) accum<METRIC>(q.v[idx], row[idx], a, b);
  }
  return finish<METRIC>(a, b, qnorm);
}

template <int NV, int METRIC>
__device__ __forceinline__ void dist_ldg2(const WideQuery& q, const float4* r0, const float4* r1, int lane, int nvec4,
                                          float qnorm, float& d0, float& d1) {
  float a0 = 0.f, b0 = 0.f, a1 = 0.f, b1 = 0.f;
  for (int base = 0; base < nvec4; base += 32 * WIDE_CHUNK) {
    float4 v0[WIDE_CHUNK], v1[WIDE_CHUNK];
#pragma unroll
    for (int i = 0; i < WIDE_CHUNK; ++i) {
      int idx = base + lane + 32 * i;
      if (idx < nvec4) {
        v0[i] = ldg_nc_f4(r0 + idx);
        v1[i] = ldg_nc_f4(r1 + idx);
      }
    }
#pragma unroll
    for (int i = 0; i < WIDE_CHUNK; ++i) {
      int idx = base + lane + 32 * i;
      if (idx < nvec4) {
        const float4 qv = q.v[idx];
        accum<METRIC>(qv, v0[i], a0, b0);
        accum<METRIC>(qv, v1[i], a1, b1);
      }
    }
  }
  d0 = finish<METRIC>(a0, b0, qnorm);
  d1 = finish<METRIC>(a1, b1, qnorm);
}

template <int NV, int METRIC>
__device__ __forceinline__ float dist_ldg1(const WideQuery& q, const float4* r0, int lane, int nvec4, float qnorm) {
  float a0 = 0.f, b0 = 0.f;
  for (int base = 0; base < nvec4; base += 32 * WIDE_CHUNK) {
    float4 v0[WIDE_CHUNK];
#pragma unroll
    for (int i = 0; i < WIDE_CHUNK; ++i) {
      int idx = base + lane + 32 * i;
      if (idx < nvec4) v0[i] = ldg_nc_f4(r0 + idx);
    }
#pragma unroll
    for (int i = 0; i < WIDE_CHUNK; ++i) {
      int idx = base + lane + 32 * i;
      if (idx < nvec4) accum<METRIC>(q.v[idx], v0[i], a0, b0);
    }
  }
  return finish<METRIC>(a0, b0, qnorm);
}

// load_query for a wide query: zero padded to round_up(dim, 4) into `dst` (when `store`), the squared norm summed in
// load_query's order.  Lane l writes and later reads only the elements idx = l + 32 i, so one warp needs no barrier.
__device__ __forceinline__ void load_query_wide(const float* qp, uint32_t dim, int lane, float4* dst, bool store,
                                                WideQuery& q, float& qnorm) {
  float s = 0.f;
  const uint32_t nvec4 = (dim + 3) / 4;
  for (uint32_t base = 0; base < nvec4; base += 32) {
    const uint32_t idx = base + lane;
    if (idx >= nvec4) continue;
    const uint32_t e = idx * 4;
    float4 v;
    v.x = qp[e];
    v.y = e + 1 < dim ? qp[e + 1] : 0.f;
    v.z = e + 2 < dim ? qp[e + 2] : 0.f;
    v.w = e + 3 < dim ? qp[e + 3] : 0.f;
    if (store) dst[idx] = v;
    s = fmaf(v.x, v.x, s);
    s = fmaf(v.y, v.y, s);
    s = fmaf(v.z, v.z, s);
    s = fmaf(v.w, v.w, s);
  }
  q.v = dst;
  qnorm = warp_sum(s);
}

template <int NV, int METRIC>
__device__ __forceinline__ float dist_smem(const float4 (&q)[NV], const float4* row, int lane, int nvec4,
                                           float qnorm) {
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) accum<METRIC>(q[i], row[idx], a, b);
  }
  return finish<METRIC>(a, b, qnorm);
}

// dist_smem's L2 distance (same order, same result) with every shared-memory load issued before the first FMA, for the
// pruned search; dist_smem itself stays as the other kernels use it.
template <int NV>
__device__ __forceinline__ float dist_smem_l2(const float4 (&q)[NV], const float4* row, int lane, int nvec4) {
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) v[i] = row[idx];
  }
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) accum<COZO_GPU_L2>(q[i], v[i], a, b);
  }
  return finish<COZO_GPU_L2>(a, b, 0.f);
}

// two rows at once straight from HBM: all 2*NV 128-bit loads are issued before
// the first use so one warp keeps 2 rows in flight.
template <int NV, int METRIC>
__device__ __forceinline__ void dist_ldg2(const float4 (&q)[NV], const float4* r0, const float4* r1, int lane,
                                          int nvec4, float qnorm, float& d0, float& d1) {
  float4 v0[NV], v1[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) {
      v0[i] = ldg_nc_f4(r0 + idx);
      v1[i] = ldg_nc_f4(r1 + idx);
    }
  }
  float a0 = 0.f, b0 = 0.f, a1 = 0.f, b1 = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) {
      accum<METRIC>(q[i], v0[i], a0, b0);
      accum<METRIC>(q[i], v1[i], a1, b1);
    }
  }
  d0 = finish<METRIC>(a0, b0, qnorm);
  d1 = finish<METRIC>(a1, b1, qnorm);
}

template <int NV, int METRIC>
__device__ __forceinline__ float dist_ldg1(const float4 (&q)[NV], const float4* r0, int lane, int nvec4,
                                           float qnorm) {
  float4 v0[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) v0[i] = ldg_nc_f4(r0 + idx);
  }
  float a0 = 0.f, b0 = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) accum<METRIC>(q[i], v0[i], a0, b0);
  }
  return finish<METRIC>(a0, b0, qnorm);
}

// found_nn.push + pop-if-over-ef (hnsw.rs:577-580) on the sorted array: keys fd (w.fd in the f32 searches, f64 keys in
// the F64 one), ids w.fi.  Precondition: len < ef || d < fd[len-1].  Equal keys keep arrival order.  Keys are ordered
// as OrderedFloat orders them: NaN after every number (+inf included) and equal to NaN, so a NaN key goes behind every
// other key.
template <typename K>
__device__ __forceinline__ void sorted_insert(WarpCtx& w, K* fd, uint32_t ef, K d, uint32_t id, int lane) {
  uint32_t pos = 0;
  for (uint32_t base = 0; base < w.len; base += 32) {
    uint32_t i = base + lane;
    bool le = (i < w.len) && (fd[i] <= d || d != d);
    uint32_t bal = __ballot_sync(0xffffffffu, le);
    pos += __popc(bal);
    if (bal != 0xffffffffu) break;
  }
  uint32_t newlen = w.len < ef ? w.len + 1 : ef;
  for (int top = (int)newlen - 1; top > (int)pos; top -= 32) {
    int i = top - 1 - lane;
    bool act = i >= (int)pos;
    K td = 0;
    uint32_t ti = 0;
    if (act) {
      td = fd[i];
      ti = w.fi[i];
    }
    __syncwarp();
    if (act) {
      fd[i + 1] = td;
      w.fi[i + 1] = ti;
    }
    __syncwarp();
  }
  __syncwarp();  // every lane has finished reading fd[len-1] / the shifted slots (vote ops do not order memory)
  if (lane == 0) {
    fd[pos] = d;
    w.fi[pos] = id;
  }
  __syncwarp();
  w.len = newlen;
  if (pos < w.cursor) w.cursor = pos;
}

// the admission of one evaluated neighbour (hnsw.rs:575-581).  d by reference: compared as a value the key is an
// argument, which the compiler's canonical form orders after the load of fd[len-1], flipping the test in the callers.
template <typename K>
__device__ __forceinline__ void admit(WarpCtx& w, K* fd, uint32_t ef, const K& d, uint32_t id, int lane) {
  if (w.len < ef || d < fd[w.len - 1]) sorted_insert(w, fd, ef, d, id, lane);
}

// visited.insert for the ids in `id` (one per lane, NONE = idle); returns whether
// this lane's id was newly inserted.  Newly set ids are logged for the clear.
__device__ __forceinline__ bool visit_mark(WarpCtx& w, uint32_t id, int lane, uint32_t& newmask) {
  bool isnew = false;
  if (id != NONE) {
    uint32_t bit = 1u << (id & 31);
    uint32_t old = atomicOr(&w.vis[id >> 5], bit);
    isnew = !(old & bit);
  }
  newmask = __ballot_sync(0xffffffffu, isnew);
  if (isnew) {
    uint32_t p = w.nlog + __popc(newmask & ((1u << lane) - 1));
    if (p < w.logcap) w.vlog[p] = id;
  }
  w.nlog += __popc(newmask);
  return isnew;
}

// visited <- keys(found); candidates <- found (hnsw.rs:554-557)
__device__ __forceinline__ void seed_visited(WarpCtx& w, int lane) {
  for (uint32_t base = 0; base < w.len; base += 32) {
    uint32_t i = base + lane;
    uint32_t id = NONE;
    if (i < w.len) {
      id = w.fi[i] & IDMASK;
      w.fi[i] = id;
    }
    uint32_t nm;
    visit_mark(w, id, lane, nm);
  }
  __syncwarp();
  w.cursor = 0;
}

// candidates.pop() (hnsw.rs:559): the nearest not-yet-expanded entry into `cand`, marked expanded.  false when there is
// none, which is the reference's `candidate_dist > furthest_dist` break (hnsw.rs:562).  (A flag rather than a NONE id:
// the compiler cannot tell that a popped id is never NONE, and would keep that test in every search loop.)
__device__ __forceinline__ bool pop_candidate(const HnswDev& g, WarpCtx& w, uint32_t level, int lane, uint32_t& cand) {
  uint32_t ci = NONE;
  for (uint32_t base = w.cursor & ~31u; base < w.len; base += 32) {
    uint32_t i = base + lane;
    bool un = (i < w.len) && (i >= w.cursor) && !(w.fi[i] & EXPANDED);
    uint32_t bal = __ballot_sync(0xffffffffu, un);
    if (bal) {
      ci = base + __ffs(bal) - 1;
      break;
    }
  }
  if (ci == NONE) return false;
  cand = w.fi[ci];
  __syncwarp();
  if (lane == 0) w.fi[ci] = cand | EXPANDED;
  w.cursor = ci + 1;
  w.nodes_expanded++;
  if (level == 0 && ci + 1 + lane < w.len && lane < 2) {
    // the next pop is most likely one of the following entries: pull their adjacency rows into L2
    uint32_t nxt = w.fi[ci + 1 + lane];
    if (!(nxt & EXPANDED)) prefetch_l2(g.adj0 + (size_t)nxt * g.s0);
  }
  return true;
}

// hnsw_get_neighbours (hnsw.rs:588-629): the padded adjacency row of `cand` on `level`
__device__ __forceinline__ const uint32_t* neighbour_row(const HnswDev& g, uint32_t cand, uint32_t level) {
  return level == 0 ? g.adj0 + (size_t)cand * g.s0 : g.adj_up + (size_t)(g.upper_off[cand] + level - 1) * g.su;
}

// the unvisited ids of one adjacency chunk (hnsw.rs:569-571,582): marks them visited, compacts them into pend in
// neighbour order, counts them as evaluations and returns how many there are
__device__ __forceinline__ uint32_t take_unvisited(WarpCtx& w, uint32_t id, int lane, uint32_t* pend) {
  uint32_t newmask;
  const bool isnew = visit_mark(w, id, lane, newmask);
  const uint32_t cnt = __popc(newmask);
  if (isnew) pend[__popc(newmask & ((1u << lane) - 1))] = id;
  w.dist_evals += cnt;
  return cnt;
}

// hnsw_knn's tail (hnsw.rs:943-956, 997-1006) for the query of this warp: walk the beam (keys fd) nearest first, drop
// `dist > radius` and rows the filter rejects, keep the first k, pad the rest with (NONE, +inf).  Without a filter the
// beam is cut to k before the radius test, and without either the kept entries are a prefix of the sorted array.  A
// radius does not keep a prefix: NaN keys sort last and pass it (`NaN > r` is false).  p supplies k, has_radius, radius
// and filter_mask (SearchParams, Search64Params); store(i, id, dist) writes result i.  Returns the number of results.
template <typename K, typename P, typename Store>
__device__ __forceinline__ uint32_t emit_results(const P& p, const WarpCtx& w, const K* fd, int lane, bool searched,
                                                 const Store& store) {
  uint32_t found = 0;
  if (searched && !p.filter_mask && !p.has_radius) {
    found = w.len < p.k ? w.len : p.k;
    for (uint32_t i = lane; i < found; i += 32) store(i, w.fi[i] & IDMASK, fd[i]);
  } else if (searched) {
    const uint32_t lim = p.filter_mask || w.len < p.k ? w.len : p.k;
    for (uint32_t base_i = 0; base_i < lim && found < p.k; base_i += 32) {
      const uint32_t i = base_i + lane;
      bool ok = i < lim;
      uint32_t id = 0;
      K d = 0;
      if (ok) {
        id = w.fi[i] & IDMASK;
        d = fd[i];
        ok = (!p.filter_mask || ((p.filter_mask[id >> 5] >> (id & 31)) & 1u)) && !(p.has_radius && (double)d > p.radius);
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, ok);
      const uint32_t pos = found + __popc(bal & ((1u << lane) - 1));
      if (ok && pos < p.k) store(pos, id, d);
      found += __popc(bal);
    }
    if (found > p.k) found = p.k;
  }
  for (uint32_t i = found + lane; i < p.k; i += 32) store(i, NONE, (K)INFINITY);
  return found;
}

// Clearing by the log costs one random atomic per logged id; by the sweep, one coalesced 16-byte store per 4 words.  A
// random atomic on a bitmap that has left L2 costs about as much as half a 784-byte row gather (tools/gather_ceiling.py
// --visited), far more than the 128 bytes of sweep that replace it, so the log is used only for layers that set fewer
// than one id per VISIT_SWEEP_WORDS words (the upper layers; at 1 M rows, fewer than ~980 ids).
constexpr uint32_t VISIT_SWEEP_WORDS = 32;

__device__ __forceinline__ void visit_clear(WarpCtx& w, int lane) {
  __syncwarp();
  if (w.nlog <= w.logcap && w.nlog * VISIT_SWEEP_WORDS <= w.nwords) {
    for (uint32_t i = lane; i < w.nlog; i += 32) atomicAnd(&w.vis[w.vlog[i] >> 5], 0u);
  } else {
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4* p = reinterpret_cast<uint4*>(w.vis);
    for (uint32_t i = lane; i < w.nwords / 4; i += 32) p[i] = z;
    __threadfence();
  }
  w.nlog = 0;
  __syncwarp();
}

// The query in the fixed point of the integer bound (hnsw_codes.cuh, CodeQuery), in the layout of the code words: the
// lane that reads code word idx = lane + 32 i (elements 4 idx .. 4 idx + 3) owns a[32 i + lane] = {the int16 pair of
// elements 4 idx, 4 idx + 1; that of 4 idx + 2, 4 idx + 3} (low half = lower element).  a lives in the warp's shared
// memory (ceil(ld / 128) * 256 bytes; in registers the pruned kernel spills), and each lane reads only what it wrote.
struct alignas(8) QueryPair {
  uint32_t lo, hi;
};
struct QueryCodes {
  QueryPair* a;
  CodeQuery c;
};
// Cosine and IP: the query's CodeDotQuery (code_dot_query) sits in shared memory right before a[], read where it is used
// (in registers the pruned kernel spills)
__device__ __forceinline__ CodeDotQuery* dot_query_of(const QueryCodes& qc) {
  return reinterpret_cast<CodeDotQuery*>(qc.a) - 1;
}

// code_query_prepare of hnsw_codes.cuh, across the warp: the same per-element functions, the sums in lane order
template <int NV>
__device__ __forceinline__ void load_query_codes(const float4 (&q)[NV], uint32_t ld, int lane, QueryCodes& qc) {
  float m = 0.f;
  bool finite = true;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float v[4] = {q[i].x, q[i].y, q[i].z, q[i].w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      finite = finite && code_finite(v[k]);
      m = fmaxf(m, fabsf(v[k]));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  finite = __ballot_sync(0xffffffffu, !finite) == 0u;
  const int32_t A = code_query_amax(ld);
  const double sq = code_query_scale(finite ? m : 0.f, A);
  int32_t suma = 0;
  double suma2 = 0.0, ss = 0.0;
#pragma unroll
  for (int i = 0; i < NV; ++i) {  // elements past ld are zero (load_query): a = 0, no residual
    const float v[4] = {q[i].x, q[i].y, q[i].z, q[i].w};
    int32_t a[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      a[k] = code_query_level(v[k], sq, A);
      suma += a[k];
      suma2 += (double)a[k] * (double)a[k];
      ss += code_query_resid2(v[k], sq, a[k]);
    }
    if (32 * i < (int)ld / 4)
      qc.a[32 * i + lane] = QueryPair{((uint32_t)a[0] & 0xFFFFu) | ((uint32_t)a[1] << 16),
                                      ((uint32_t)a[2] & 0xFFFFu) | ((uint32_t)a[3] << 16)};
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    suma += __shfl_xor_sync(0xffffffffu, suma, o);
    suma2 += __shfl_xor_sync(0xffffffffu, suma2, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  qc.c = code_query_finish(sq, suma, suma2, ss, finite);
}

// acc + the exact integer dot product of the four int16 query levels in (alo, ahi) with the four uint8 codes of c
__device__ __forceinline__ int32_t code_idot4(uint32_t alo, uint32_t ahi, uint32_t c, int32_t acc) {
#if defined(__CUDA_ARCH__)
  // dp2a: two 16x8-bit products per instruction, int16 pairs against the low (.lo) or high (.hi) two code bytes
  asm("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(acc) : "r"(alo), "r"(c));
  asm("dp2a.hi.s32.u32 %0, %1, %2, %0;" : "+r"(acc) : "r"(ahi), "r"(c));
#else
  acc += (int32_t)(int16_t)(alo & 0xFFFFu) * (int32_t)(c & 0xFFu) + (int32_t)(int16_t)(alo >> 16) * (int32_t)((c >> 8) & 0xFFu) +
         (int32_t)(int16_t)(ahi & 0xFFFFu) * (int32_t)((c >> 16) & 0xFFu) + (int32_t)(int16_t)(ahi >> 16) * (int32_t)(c >> 24);
#endif
  return acc;
}

// S = sum_j a_j c_j (CodeQuery) for two code rows in shared memory, exact in int32 (so any summation order gives the same
// S).  Each row's words alternate between two dp2a chains, and the warp sum is one redux.sync per row: the scoring is
// bound by this chain's latency, not by issue.
template <int NV>
__device__ __forceinline__ void code_idot2(const QueryCodes& qc, const uint8_t* r0, const uint8_t* r1, int lane,
                                           int nvec4, int32_t& s0, int32_t& s1) {
  const uint32_t* c0 = reinterpret_cast<const uint32_t*>(r0 + CODE_HDR);
  const uint32_t* c1 = reinterpret_cast<const uint32_t*>(r1 + CODE_HDR);
  // every shared-memory load first, so their latencies overlap (above NV = 8 that needs more registers than the
  // kernel has: loaded where used)
  constexpr bool HOIST = NV <= 8;
  uint32_t w0[NV], w1[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (HOIST) {
      w0[i] = idx < nvec4 ? c0[idx] : 0u;
      w1[i] = idx < nvec4 ? c1[idx] : 0u;
    }
  }
  int32_t a0[2] = {0, 0}, a1[2] = {0, 0};
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec4) {
      const QueryPair qa = qc.a[idx];
      a0[i & 1] = code_idot4(qa.lo, qa.hi, HOIST ? w0[i] : c0[idx], a0[i & 1]);
      a1[i & 1] = code_idot4(qa.lo, qa.hi, HOIST ? w1[i] : c1[idx], a1[i & 1]);
    }
  }
#if defined(__CUDA_ARCH__)
  s0 = __reduce_add_sync(0xffffffffu, a0[0] + a0[1]);
  s1 = __reduce_add_sync(0xffffffffu, a1[0] + a1[1]);
#else
  int32_t t0 = a0[0] + a0[1], t1 = a1[0] + a1[1];
  for (int o = 16; o > 0; o >>= 1) {
    t0 += __shfl_xor_sync(0xffffffffu, t0, o);
    t1 += __shfl_xor_sync(0xffffffffu, t1, o);
  }
  s0 = t0;
  s1 = t1;
#endif
}

// One 32-id adjacency chunk of a pruned hop (codes present, beam full), as one stream per warp.  `id` is this lane's
// neighbour id (NONE = idle), `validmask` the lanes that hold one.
//   * The code rows of the first w.cns valid ids are issued before the visited test, so their fetch overlaps the
//     atomicOr round trip.  Those that turn out to be visited are waited for and discarded (not scored, not counted);
//     later ids are fetched only if they are unvisited.  Stream position p holds w.pend[p], bit 31 set = discard.
//   * Each code row's distance is bounded from below (hnsw_codes.cuh, code_int_prunes for L2, code_dot_prunes for Cosine
//     and IP: from the exact integer product of the code row with the fixed-point query qc) against the beam's worst
//     distance AT THAT MOMENT.  With a
//     full beam fd[len-1] only decreases, and a neighbour's admission test `d < fd[len-1]` comes after every earlier
//     survivor's admission, so the value tested here is at least the one its admission would face: a dropped
//     neighbour could not have been admitted.
//   * A survivor's f32 row is issued as soon as an f32 slot is free and consumed, in survivor (= neighbour) order,
//     as soon as it has landed (polled, never waited for while code rows remain); the rest are drained at the end.
//     Admissions therefore happen in neighbour order with the live bound, exactly as without pruning: ids, distances
//     and the traversal counters are unchanged; only the number of f32 rows fetched can go down.
template <int NV, int METRIC>
__device__ __forceinline__ void prune_chunk(const HnswDev& g, WarpCtx& w, const float4 (&q)[NV], float qnorm,
                                            const QueryCodes& qc, uint32_t ef, uint32_t id, uint32_t validmask, int lane) {
  const int nvec4 = g.ld >> 2;
  const uint32_t crow = g.code_ld, row_bytes = g.ld * 4;
  const uint32_t lt = (1u << lane) - 1;
  const uint32_t rank = __popc(validmask & lt);
  const uint32_t spec = min((uint32_t)__popc(validmask), w.cns);  // speculative code rows: valid ids of rank < spec
  const bool early = id != NONE && rank < spec;
  HOP_T(t0);
  if (early) {
    uint32_t s = w.chead + rank;
    if (s >= w.cns) s -= w.cns;
    fence_proxy_async_smem();
    mbar_expect_tx(&w.cbars[s], crow);
    bulk_g2s(w.cring + (size_t)s * crow, g.codes + (size_t)id * crow, crow, &w.cbars[s]);
  }
  uint32_t newmask;
  const bool isnew = visit_mark(w, id, lane, newmask);  // hnsw.rs:569-571,582
  const uint32_t earlymask = __ballot_sync(0xffffffffu, early);
  w.dist_evals += __popc(newmask);
  if (early) w.pend[rank] = isnew ? id : id | EXPANDED;
  else if (isnew) w.pend[spec + __popc(newmask & ~earlymask & lt)] = id;
  const uint32_t len = spec + __popc(newmask & ~earlymask);
  __syncwarp();
  HOP_ADD(w, HC_VISIT, t0);

  uint32_t fq = 0, fin = 0;  // bits by stream position: survivors whose f32 row is queued / in flight (in order)
  // the per-row test and what it compares with, recomputed whenever the beam's worst distance changes
  auto radius = [&](float worst) {
    if constexpr (METRIC == COZO_GPU_L2) return code_int_radius(qc.c, worst);
    else return code_dot_radius(*dot_query_of(qc), worst);
  };
  auto prunes = [&](int32_t S, const float* hdr, double WE) {
    if constexpr (METRIC == COZO_GPU_L2) return code_int_prunes(qc.c, S, hdr, WE);
    else return code_dot_prunes<METRIC>(*dot_query_of(qc), S, hdr, WE);
  };
  double WE = radius(w.fd[ef - 1]);
  // f32 ring: slot w.head holds the oldest row in flight, popc(fin) rows are in flight
  auto f32_issue = [&]() {
    while (fq && __popc(fin) < w.ns) {
      const uint32_t c = __ffs(fq) - 1;
      if (lane == 0) {
        uint32_t s = w.head + __popc(fin);
        if (s >= w.ns) s -= w.ns;
        fence_proxy_async_smem();
        mbar_expect_tx(&w.bars[s], row_bytes);
        bulk_g2s(w.ring + (size_t)s * g.ld, g.vec + (size_t)w.pend[c] * g.ld, row_bytes, &w.bars[s]);
      }
      fq &= fq - 1;
      fin |= 1u << c;
    }
  };
  auto f32_consume = [&]() {
    HOP_T(t1);
    mbar_wait(&w.bars[w.head], (w.phase >> w.head) & 1u);
    w.phase ^= (1u << w.head);
    HOP_ADD(w, HC_FWAIT, t1);
    HOP_T(t2);
    const float4* row = reinterpret_cast<const float4*>(w.ring + (size_t)w.head * g.ld);
    // above NV = 6 the loads-first form needs more registers than the kernel has (it spills)
    float d;
    if constexpr (METRIC == COZO_GPU_L2)
      d = NV > 6 ? dist_smem<NV, COZO_GPU_L2>(q, row, lane, nvec4, 0.f) : dist_smem_l2<NV>(q, row, lane, nvec4);
    else
      d = dist_smem<NV, METRIC>(q, row, lane, nvec4, qnorm);
    if (++w.head == w.ns) w.head = 0;
    const uint32_t nid = w.pend[__ffs(fin) - 1];
    fin &= fin - 1;
    __syncwarp();
    if (d < w.fd[ef - 1]) {  // hnsw.rs:575-581 (the beam stays full)
      sorted_insert(w, w.fd, ef, d, nid, lane);
      WE = radius(w.fd[ef - 1]);
    }
    HOP_ADD(w, HC_FSCORE, t2);
  };

  // code rows two at a time (code_idot2); position `issued` is the next one to fetch, into slot chead + issued - c
  uint32_t issued = spec;
  for (uint32_t c = 0; c < len;) {
    const uint32_t upto = min(len, c + w.cns);
    if (lane == 0 && issued < upto) {
      fence_proxy_async_smem();
      for (uint32_t p = issued; p < upto; ++p) {
        uint32_t s = w.chead + (p - c);
        if (s >= w.cns) s -= w.cns;
        mbar_expect_tx(&w.cbars[s], crow);
        bulk_g2s(w.cring + (size_t)s * crow, g.codes + (size_t)w.pend[p] * crow, crow, &w.cbars[s]);
      }
    }
    issued = max(issued, upto);
    const bool two = c + 1 < len;
    uint32_t s1 = w.chead + 1;
    if (s1 == w.cns) s1 = 0;
    HOP_T(t3);
    mbar_wait(&w.cbars[w.chead], (w.cphase >> w.chead) & 1u);
    w.cphase ^= (1u << w.chead);
    if (two) {
      mbar_wait(&w.cbars[s1], (w.cphase >> s1) & 1u);
      w.cphase ^= (1u << s1);
    }
    HOP_ADD(w, HC_CWAIT, t3);
    HOP_T(t4);
    const uint8_t* r0 = w.cring + (size_t)w.chead * crow;
    const uint8_t* r1 = two ? w.cring + (size_t)s1 * crow : r0;
    int32_t S0, S1;
    code_idot2<NV>(qc, r0, r1, lane, nvec4, S0, S1);
    const float4 h0 = *reinterpret_cast<const float4*>(r0), h1 = *reinterpret_cast<const float4*>(r1);
    const uint32_t p0 = w.pend[c], p1 = two ? w.pend[c + 1] : EXPANDED;
    __syncwarp();  // every lane is done with the two slots before lane 0 refills them
    if (!(p0 & EXPANDED)) {
      if (prunes(S0, &h0.x, WE)) w.pruned++;
      else fq |= 1u << c;
    }
    if (!(p1 & EXPANDED)) {
      if (prunes(S1, &h1.x, WE)) w.pruned++;
      else fq |= 1u << (c + 1);
    }
    const uint32_t step = two ? 2 : 1;
    w.chead += step;
    if (w.chead >= w.cns) w.chead -= w.cns;
    c += step;
    HOP_ADD(w, HC_CSCORE, t4);
    f32_issue();
    // admit the rows that have landed; a row in flight is not waited for while code rows remain
    while (fin && __shfl_sync(0xffffffffu, lane == 0 ? (uint32_t)mbar_try_wait(&w.bars[w.head], (w.phase >> w.head) & 1u) : 0u, 0)) {
      f32_consume();
      f32_issue();
    }
  }
  while (fin) {
    f32_consume();
    f32_issue();
  }
}

// hnsw_search_level (hnsw.rs:539-587) for one query held in registers.
// `level` 0 is the bottom layer.  On entry the sorted array holds found_nn.
// PRUNE (the bulk ring, register query): when g.codes is set, the chunks of a hop that find the beam full run prune_chunk, which
// fetches f32 rows only for the neighbours whose code row cannot rule out admission.
// qc: the query's fixed-point form (load_query_codes), read only by prune_chunk.
// NV = 0: the query is a WideQuery (no pruning).
template <int NV, int METRIC, bool BULK, bool PRUNE = false>
__device__ __forceinline__ void search_level(const HnswDev& g, WarpCtx& w, const typename QueryOf<NV>::type& q, float qnorm,
                                             uint32_t ef, uint32_t level, int lane,
                                             const QueryCodes* qc = nullptr) {
  const int nvec4 = g.ld >> 2;
  const uint32_t row_bytes = g.ld * 4;
  seed_visited(w, lane);
  const uint32_t stride = level == 0 ? g.s0 : g.su;

  for (;;) {
    HOP_T(tp);
    uint32_t cand;
    if (!pop_candidate(g, w, level, lane, cand)) break;
    const uint32_t* row = neighbour_row(g, cand, level);
    for (uint32_t nb = 0; nb < stride; nb += 32) {
      if (nb) HOP_SET(tp);
      uint32_t id = __ldg(row + nb + lane);
      uint32_t validmask = __ballot_sync(0xffffffffu, id != NONE);
      HOP_ADD(w, HC_POP, tp);
      if (!validmask) break;
      w.nbr_reads += __popc(validmask);
      if constexpr (PRUNE) {
        if (g.codes && w.len == ef) {
          prune_chunk<NV, METRIC>(g, w, q, qnorm, *qc, ef, id, validmask, lane);
          __syncwarp();
          continue;
        }
      }
      HOP_T(tv);
      const uint32_t cnt = take_unvisited(w, id, lane, w.pend);
      __syncwarp();
      HOP_ADD(w, HC_VISIT, tv);
      if (BULK) {
        // ring indices advance by compare-and-wrap (a runtime `% ns` costs ~20 instructions)
        uint32_t issued = 0, si = w.head, sc = w.head;
        for (uint32_t c = 0; c < cnt; ++c) {
          if (lane == 0) {
            fence_proxy_async_smem();
            while (issued < cnt && issued - c < w.ns) {
              mbar_expect_tx(&w.bars[si], row_bytes);
              bulk_g2s(w.ring + (size_t)si * g.ld, g.vec + (size_t)w.pend[issued] * g.ld, row_bytes, &w.bars[si]);
              ++issued;
              if (++si == w.ns) si = 0;
            }
          }
          HOP_T(tw);
          mbar_wait(&w.bars[sc], (w.phase >> sc) & 1u);
          w.phase ^= (1u << sc);
          HOP_ADD(w, HC_FWAIT, tw);
          HOP_T(ts);
          float d = dist_smem<NV, METRIC>(q, reinterpret_cast<const float4*>(w.ring + (size_t)sc * g.ld), lane, nvec4,
                                          qnorm);
          if (++sc == w.ns) sc = 0;
          uint32_t nid = w.pend[c];
          __syncwarp();
          admit(w, w.fd, ef, d, nid, lane);
          HOP_ADD(w, HC_FSCORE, ts);
        }
        w.head = sc;
      } else {
        for (uint32_t c = 0; c < cnt; c += 2) {
          uint32_t id0 = w.pend[c];
          bool two = c + 1 < cnt;
          uint32_t id1 = two ? w.pend[c + 1] : id0;
          float d0, d1;
          if (two) {
            dist_ldg2<NV, METRIC>(q, reinterpret_cast<const float4*>(g.vec + (size_t)id0 * g.ld),
                                  reinterpret_cast<const float4*>(g.vec + (size_t)id1 * g.ld), lane, nvec4, qnorm, d0,
                                  d1);
          } else {
            d0 = dist_ldg1<NV, METRIC>(q, reinterpret_cast<const float4*>(g.vec + (size_t)id0 * g.ld), lane, nvec4,
                                       qnorm);
            d1 = 0.f;
          }
          admit(w, w.fd, ef, d0, id0, lane);
          if (two) admit(w, w.fd, ef, d1, id1, lane);
        }
      }
      __syncwarp();
    }
  }
  visit_clear(w, lane);
}

// ---------------------------------------------------------------------------------------------
// Cooperative form: ONE CTA (4 warps) per query.  Warp 0 owns the sorted found/candidate array, the
// visited bitmap and the admission order — exactly the routine above — but the rows of a hop are
// dealt round-robin to all warps, each with its own bulk-copy ring, and their distances meet in
// shared memory before warp 0 applies the admissions IN NEIGHBOUR ORDER.  Same traversal, same
// counters, same results; a query advances ~4x faster, which is what small batches (and the tail of
// a large one) need: there are not enough queries to fill the SMs with one warp each.
struct CoopShared {
  uint32_t* pend;    // [32] unvisited neighbour ids of the current round
  float* pdist;      // [32] their distances
  uint32_t* ctrl;    // [0] = number of rows of this round, COOP_DONE = layer finished
};
constexpr uint32_t COOP_DONE = 0xFFFFFFFFu;
constexpr uint32_t COOP_WARPS = 4;

template <int NV, int METRIC>
__device__ __forceinline__ void coop_search_level(const HnswDev& g, WarpCtx& w, const CoopShared& cs,
                                                  const typename QueryOf<NV>::type& q, float qnorm, uint32_t ef, uint32_t level,
                                                  int lane, int warp) {
  const int nvec4 = g.ld >> 2;
  const uint32_t row_bytes = g.ld * 4;
  const uint32_t stride = level == 0 ? g.s0 : g.su;
  // warp-0 state of the current expansion
  const uint32_t* row = nullptr;
  uint32_t nb = stride;  // chunk offset inside the candidate's adjacency row; stride = need a new candidate
  if (warp == 0) seed_visited(w, lane);
  for (;;) {
    if (warp == 0) {
      uint32_t cnt = 0;
      while (cnt == 0) {
        if (nb >= stride) {
          uint32_t cand;
          if (!pop_candidate(g, w, level, lane, cand)) {
            cnt = COOP_DONE;
            break;
          }
          row = neighbour_row(g, cand, level);
          nb = 0;
        }
        uint32_t id = __ldg(row + nb + lane);
        uint32_t validmask = __ballot_sync(0xffffffffu, id != NONE);
        nb = validmask ? nb + 32 : stride;  // rows are packed: an empty chunk ends the row
        if (!validmask) continue;
        w.nbr_reads += __popc(validmask);
        cnt = take_unvisited(w, id, lane, cs.pend);
      }
      if (lane == 0) cs.ctrl[0] = cnt;
    }
    __syncthreads();  // the round's ids are published
    const uint32_t cnt = cs.ctrl[0];
    if (cnt == COOP_DONE) break;
    {  // every warp: rows warp, warp+4, ... through its own ring
      uint32_t issued = warp, si = w.head, sc = w.head;
      for (uint32_t c = warp; c < cnt; c += COOP_WARPS) {
        if (lane == 0) {
          fence_proxy_async_smem();
          while (issued < cnt && (issued - c) / COOP_WARPS < w.ns) {
            mbar_expect_tx(&w.bars[si], row_bytes);
            bulk_g2s(w.ring + (size_t)si * g.ld, g.vec + (size_t)cs.pend[issued] * g.ld, row_bytes, &w.bars[si]);
            issued += COOP_WARPS;
            if (++si == w.ns) si = 0;
          }
        }
        mbar_wait(&w.bars[sc], (w.phase >> sc) & 1u);
        w.phase ^= (1u << sc);
        float d = dist_smem<NV, METRIC>(q, reinterpret_cast<const float4*>(w.ring + (size_t)sc * g.ld), lane, nvec4,
                                        qnorm);
        if (++sc == w.ns) sc = 0;
        if (lane == 0) cs.pdist[c] = d;
        __syncwarp();
      }
      w.head = sc;
    }
    __syncthreads();  // all distances of the round are in shared memory
    if (warp == 0) {
      for (uint32_t c = 0; c < cnt; ++c) {  // hnsw.rs:575-581, in neighbour order with the live bound
        const float d = cs.pdist[c];
        const uint32_t nid = cs.pend[c];
        __syncwarp();
        admit(w, w.fd, ef, d, nid, lane);
      }
    }
  }
  if (warp == 0) visit_clear(w, lane);
  __syncthreads();
}

// load one query into registers (zero padded), optionally its squared norm
template <int NV>
__device__ __forceinline__ void load_query(const float* qp, uint32_t dim, int lane, float4 (&q)[NV], float& qnorm) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    uint32_t e = (uint32_t)(lane + 32 * i) * 4;
    float4 v;
    v.x = e + 0 < dim ? qp[e + 0] : 0.f;
    v.y = e + 1 < dim ? qp[e + 1] : 0.f;
    v.z = e + 2 < dim ? qp[e + 2] : 0.f;
    v.w = e + 3 < dim ? qp[e + 3] : 0.f;
    q[i] = v;
    s = fmaf(v.x, v.x, s);
    s = fmaf(v.y, v.y, s);
    s = fmaf(v.z, v.z, s);
    s = fmaf(v.w, v.w, s);
  }
  qnorm = warp_sum(s);
}

}  // namespace cozo
