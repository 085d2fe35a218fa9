// graph_kernels.cuh — device code of the FixedRule graph algorithms (graph.cu): the SSSP family in its three frontier
// forms, closeness, betweenness, clustering and the read-out kernels.  A header so that the same source is compiled by
// nvcc into libcozo_gpu.so and by tests/emu (a CPU SIMT emulator, test infrastructure) into a host program.
#pragma once
#include "common.cuh"

namespace cozo {

// ---- SSSP ---------------------------------------------------------------------
// One CTA per source.  Label-correcting relaxation to the fixed point
// dist[v] = min_u fl32(dist[u] + w(u,v)); with non-negative weights this is the
// value Dijkstra's `cost + path_weight` recursion produces
// (shortest_path_dijkstra.rs:304-309), bit for bit.  State per (source, node)
// is one u64 = (f32 bits of dist << 32) | predecessor, updated by CAS only on a
// strictly smaller distance (strict `<`, shortest_path_dijkstra.rs:305), so the
// predecessors always form a tree.
constexpr unsigned long long SSSP_INF = 0x7F800000FFFFFFFFull;  // (+inf, NONE)

// ForbiddenNode / ForbiddenEdge sets (shortest_path_dijkstra.rs:188-218) of source `si` are the
// slices [fn_ptr[si], fn_ptr[si+1]) of fn_nodes and [fe_ptr[si], fe_ptr[si+1]) of (fe_src, fe_dst);
// they are a handful of entries (KShortestPathYen: one root path + at most k edges).
struct ForbiddenSets {
  const uint32_t *fn_ptr, *fn_nodes, *fe_ptr, *fe_src, *fe_dst;
};

// The goals a search may stop at (cozo_gpu_sssp_goals): distinct node ids, shared by every source.
// `red` = 64 floats of shared memory for the per-warp lower bounds and largest goal distances of a round.
struct GoalSet {
  const uint32_t* goals;
  uint32_t n;
  float* red;
};

// SMEM = the per-source state (8 B/node) and the two frontier flag arrays (1 B/node each) live in
// shared memory (graphs up to ~22 k nodes); the final state is copied out for the read-out kernels.
// A warp takes one frontier node at a time and its lanes stride the node's out-edges.  A round scans the
// flag arrays (O(n) per round): the default form, verified on the GPU since round 1.
//
// GOALS = stop once every goal is settled.  L = the smallest distance written by a successful CAS in the round is a
// lower bound on every node of the next frontier, and every later update is >= L (weights are non-negative and
// fl32(a + w) >= a).  So when every goal is finite and L > G = max goal distance, no node at distance <= G can change
// again: the goals' costs, their predecessor paths and every tied predecessor of a node at distance <= G are those of
// the full run.  The test is strict: with L == G a zero-weight edge could still bring a new tied predecessor at G.
template <bool FORB, bool SMEM, bool GOALS = false>
__device__ __forceinline__ void sssp_body(const uint32_t* __restrict__ out_ptr, const uint32_t* __restrict__ out_idx,
                                          const float* __restrict__ out_w, uint32_t n,
                                          const uint32_t* __restrict__ sources, uint32_t n_src,
                                          unsigned long long* state, uint8_t* flags, size_t flags_stride,
                                          ForbiddenSets fs, uint8_t* sssp_smem, GoalSet gs = GoalSet{}) {
  const uint32_t si = blockIdx.x;
  if (si >= n_src) return;
  uint32_t fnb = 0, fne = 0, feb = 0, fee = 0;
  if (FORB) {
    fnb = fs.fn_ptr[si];
    fne = fs.fn_ptr[si + 1];
    feb = fs.fe_ptr[si];
    fee = fs.fe_ptr[si + 1];
  }
  unsigned long long* gst = state + (size_t)si * n;
  unsigned long long* st = SMEM ? reinterpret_cast<unsigned long long*>(sssp_smem) : gst;
  uint8_t* cur = SMEM ? sssp_smem + (size_t)n * 8 : flags + (size_t)si * flags_stride;
  uint8_t* nxt = cur + n;
  __shared__ int s_any;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) {
    st[v] = SSSP_INF;
    cur[v] = 0;
    nxt[v] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = sources[si];
    st[s] = 0x00000000FFFFFFFFull;  // dist 0, no predecessor
    cur[s] = 1;
  }
  __syncthreads();
  for (;;) {
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    bool any_local = false;
    float lb = __int_as_float(0x7f800000);  // GOALS: smallest distance this thread wrote in the round
    for (uint32_t u = warp; u < n; u += nwarps) {
      if (!cur[u]) continue;  // warp-uniform
      __syncwarp();
      if (lane == 0) cur[u] = 0;
      const float du = __uint_as_float((uint32_t)(st[u] >> 32));
      const uint32_t kb = out_ptr[u], ke = out_ptr[u + 1];
      for (uint32_t k = kb + lane; k < ke; k += 32) {
        const uint32_t v = out_idx[k];
        if (FORB) {  // shortest_path_dijkstra.rs:298-303
          bool skip = false;
          for (uint32_t f = fnb; f < fne; ++f) skip |= fs.fn_nodes[f] == v;
          for (uint32_t f = feb; f < fee; ++f) skip |= (fs.fe_src[f] == u) & (fs.fe_dst[f] == v);
          if (skip) continue;
        }
        const float nd = du + (out_w ? out_w[k] : 1.0f);
        unsigned long long old = st[v];
        while (nd < __uint_as_float((uint32_t)(old >> 32))) {
          unsigned long long want = ((unsigned long long)__float_as_uint(nd) << 32) | u;
          unsigned long long got = atomicCAS(&st[v], old, want);
          if (got == old) {
            nxt[v] = 1;
            any_local = true;
            if constexpr (GOALS) lb = fminf(lb, nd);
            break;
          }
          old = got;
        }
      }
    }
    if constexpr (GOALS) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) lb = fminf(lb, __shfl_xor_sync(0xffffffffu, lb, o));
      if (lane == 0) gs.red[warp] = lb;
    }
    if (any_local) s_any = 1;
    __syncthreads();
    const int any = s_any;
    if constexpr (GOALS) {  // this round's writes are complete: the largest goal distance, +inf while a goal is unreached
      float gmax = 0.0f;
      for (uint32_t i = threadIdx.x; i < gs.n; i += blockDim.x)
        gmax = fmaxf(gmax, __uint_as_float((uint32_t)(st[gs.goals[i]] >> 32)));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
      if (lane == 0) gs.red[32 + warp] = gmax;
    }
    __syncthreads();
    if (!any) break;
    if constexpr (GOALS) {
      float L = gs.red[0], G = gs.red[32];
      for (uint32_t w = 1; w < nwarps; ++w) {
        L = fminf(L, gs.red[w]);
        G = fmaxf(G, gs.red[32 + w]);
      }
      if (G < L) break;  // G finite: L is +inf only when no update can follow
    }
    uint8_t* t = cur;
    cur = nxt;
    nxt = t;
  }
  if (SMEM)
    for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) gst[v] = st[v];
}

// COMPACTED frontier (option "sssp.frontier" = 1; not yet run on a GPU, see DESIGN.md §0): state in HBM, two node
// queues per source plus an "already queued" byte per node, so a round costs O(frontier + its edges), not O(n).
// Layout of `flags` per source: [queue A: n u32][queue B: n u32][queued: n u8 (padded)].  Rounds are capped at n + 2
// (a label-correcting search settles a shortest path of h hops within h rounds), so the kernel always terminates.
template <bool FORB>
__global__ void __launch_bounds__(256) sssp_queue_kernel(const uint32_t* __restrict__ out_ptr,
                                                         const uint32_t* __restrict__ out_idx,
                                                         const float* __restrict__ out_w, uint32_t n,
                                                         const uint32_t* __restrict__ sources, uint32_t n_src,
                                                         unsigned long long* state, uint8_t* flags, size_t flags_stride,
                                                         ForbiddenSets fs) {
  const uint32_t si = blockIdx.x;
  if (si >= n_src) return;
  uint32_t fnb = 0, fne = 0, feb = 0, fee = 0;
  if (FORB) {
    fnb = fs.fn_ptr[si];
    fne = fs.fn_ptr[si + 1];
    feb = fs.fe_ptr[si];
    fee = fs.fe_ptr[si + 1];
  }
  unsigned long long* st = state + (size_t)si * n;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ uint32_t s_tail;
  uint8_t* fb = flags + (size_t)si * flags_stride;
  uint32_t* qa = reinterpret_cast<uint32_t*>(fb);
  uint32_t* qb = qa + n;
  uint8_t* queued = reinterpret_cast<uint8_t*>(qb + n);
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) {
    st[v] = SSSP_INF;
    queued[v] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = sources[si];
    st[s] = 0x00000000FFFFFFFFull;
    qa[0] = s;
    s_tail = 0;
  }
  uint32_t count = 1;
  __syncthreads();
  for (uint32_t round = 0; count && round < n + 2; ++round) {
    for (uint32_t i = warp; i < count; i += nwarps) {
      const uint32_t u = qa[i];
      __syncwarp();
      if (lane == 0) {  // u may be queued again by a later improvement ...
        atomicAnd(reinterpret_cast<uint32_t*>(queued + (u & ~3u)), ~(0xFFu << (8 * (u & 3u))));
        __threadfence_block();
      }
      // ... but only one that lands AFTER the clear: every lane reads u's distance after it (an improvement that still
      // saw the bit set is then part of the value read here).  Found by the CPU SIMT emulator (tests/emu/graph_emu.cpp).
      __syncwarp();
      const float du = __uint_as_float((uint32_t)(*reinterpret_cast<volatile unsigned long long*>(st + u) >> 32));
      const uint32_t kb = out_ptr[u], ke = out_ptr[u + 1];
      for (uint32_t k = kb + lane; k < ke; k += 32) {
        const uint32_t v = out_idx[k];
        if (FORB) {
          bool skip = false;
          for (uint32_t f = fnb; f < fne; ++f) skip |= fs.fn_nodes[f] == v;
          for (uint32_t f = feb; f < fee; ++f) skip |= (fs.fe_src[f] == u) & (fs.fe_dst[f] == v);
          if (skip) continue;
        }
        const float nd = du + (out_w ? out_w[k] : 1.0f);
        unsigned long long old = st[v];
        while (nd < __uint_as_float((uint32_t)(old >> 32))) {
          unsigned long long want = ((unsigned long long)__float_as_uint(nd) << 32) | u;
          unsigned long long got = atomicCAS(&st[v], old, want);
          if (got == old) {
            // one byte per node: test-and-set through a 32-bit atomicOr on the aligned word
            uint32_t* wp = reinterpret_cast<uint32_t*>(queued + (v & ~3u));
            const uint32_t bit = 1u << (8 * (v & 3u));
            if (!(atomicOr(wp, bit) & bit)) {
              const uint32_t at = atomicAdd(&s_tail, 1u);
              if (at < n) qb[at] = v;
            }
            break;
          }
          old = got;
        }
      }
    }
    __syncthreads();
    count = s_tail < n ? s_tail : n;
    __syncthreads();
    if (threadIdx.x == 0) s_tail = 0;
    uint32_t* t = qa;
    qa = qb;
    qb = t;
    __syncthreads();
  }
}

// ---- "wide" form: few sources on a large graph --------------------------------------------------------------
// One CTA per source leaves the device idle when a rule asks for one or a handful of start nodes on a big graph
// (the common ShortestPathDijkstra call).  Here a ROUND is one launch of grid (ctas, n_src): all CTAs of a column
// share the source's frontier queue (same layout as above), queue tails are device counters, the host reads the
// n_src tail counts between rounds.  State is read with ld.global.cg (L2): the relaxing CTAs sit on different SMs.
__global__ void sssp_wide_init_kernel(uint32_t n, const uint32_t* __restrict__ sources, uint32_t n_src,
                                      unsigned long long* state, uint8_t* flags, size_t flags_stride, uint32_t* counts) {
  const uint32_t si = blockIdx.y;
  unsigned long long* st = state + (size_t)si * n;
  uint8_t* fb = flags + (size_t)si * flags_stride;
  uint32_t* qa = reinterpret_cast<uint32_t*>(fb);
  uint8_t* queued = reinterpret_cast<uint8_t*>(qa + 2 * (size_t)n);
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    st[v] = v == sources[si] ? 0x00000000FFFFFFFFull : SSSP_INF;
    queued[v] = 0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    qa[0] = sources[si];
    counts[si] = 1;           // current frontier
    counts[n_src + si] = 0;   // next frontier
  }
}

template <bool FORB>
__global__ void __launch_bounds__(256) sssp_wide_round_kernel(const uint32_t* __restrict__ out_ptr,
                                                              const uint32_t* __restrict__ out_idx,
                                                              const float* __restrict__ out_w, uint32_t n, uint32_t n_src,
                                                              unsigned long long* state, uint8_t* flags,
                                                              size_t flags_stride, uint32_t* counts, uint32_t parity,
                                                              ForbiddenSets fs) {
  const uint32_t si = blockIdx.y;
  const uint32_t count = min(counts[parity * n_src + si], n);
  if (count == 0) return;
  uint32_t* tail = counts + (parity ^ 1u) * n_src + si;
  unsigned long long* st = state + (size_t)si * n;
  uint8_t* fb = flags + (size_t)si * flags_stride;
  uint32_t* q0 = reinterpret_cast<uint32_t*>(fb);
  uint32_t* qa = q0 + (size_t)parity * n;
  uint32_t* qb = q0 + (size_t)(parity ^ 1u) * n;
  uint8_t* queued = reinterpret_cast<uint8_t*>(q0 + 2 * (size_t)n);
  uint32_t fnb = 0, fne = 0, feb = 0, fee = 0;
  if (FORB) {
    fnb = fs.fn_ptr[si];
    fne = fs.fn_ptr[si + 1];
    feb = fs.fe_ptr[si];
    fee = fs.fe_ptr[si + 1];
  }
  const int lane = threadIdx.x & 31;
  const uint32_t wpb = blockDim.x >> 5;
  for (uint32_t i = blockIdx.x * wpb + (threadIdx.x >> 5); i < count; i += gridDim.x * wpb) {
    const uint32_t u = qa[i];
    if (lane == 0) {
      atomicAnd(reinterpret_cast<uint32_t*>(queued + (u & ~3u)), ~(0xFFu << (8 * (u & 3u))));
      __threadfence();  // the clear is ordered before the read of u's distance below
    }
    __syncwarp();
    const float du = __uint_as_float((uint32_t)(__ldcg(st + u) >> 32));
    const uint32_t kb = out_ptr[u], ke = out_ptr[u + 1];
    for (uint32_t k = kb + lane; k < ke; k += 32) {
      const uint32_t v = out_idx[k];
      if (FORB) {
        bool skip = false;
        for (uint32_t f = fnb; f < fne; ++f) skip |= fs.fn_nodes[f] == v;
        for (uint32_t f = feb; f < fee; ++f) skip |= (fs.fe_src[f] == u) & (fs.fe_dst[f] == v);
        if (skip) continue;
      }
      const float nd = du + (out_w ? out_w[k] : 1.0f);
      unsigned long long old = __ldcg(st + v);
      while (nd < __uint_as_float((uint32_t)(old >> 32))) {
        const unsigned long long want = ((unsigned long long)__float_as_uint(nd) << 32) | u;
        const unsigned long long got = atomicCAS(&st[v], old, want);
        if (got == old) {
          __threadfence();  // the new distance is visible before the node can be seen as queued
          uint32_t* wp = reinterpret_cast<uint32_t*>(queued + (v & ~3u));
          const uint32_t bit = 1u << (8 * (v & 3u));
          if (!(atomicOr(wp, bit) & bit)) {
            const uint32_t at = atomicAdd(tail, 1u);
            if (at < n) qb[at] = v;
          }
          break;
        }
        old = got;
      }
    }
  }
}
__global__ void sssp_wide_reset_kernel(uint32_t* counts, uint32_t n_src, uint32_t parity) {
  const uint32_t si = blockIdx.x * blockDim.x + threadIdx.x;
  if (si < n_src) counts[parity * n_src + si] = 0;
}

// goal-directed read-out (shortest_path_dijkstra.rs:318-336): walk the predecessors from the goal
__global__ void sssp_path_kernel(const unsigned long long* state, uint32_t n, const uint32_t* sources,
                                 const uint32_t* goals, uint32_t n_src, uint32_t max_len, float* cost, uint32_t* len,
                                 uint32_t* paths) {
  const uint32_t si = blockIdx.x * blockDim.x + threadIdx.x;
  if (si >= n_src) return;
  const unsigned long long* st = state + (size_t)si * n;
  const uint32_t s = sources[si], t = goals[si];
  const float c = __uint_as_float((uint32_t)(st[t] >> 32));
  cost[si] = c;
  if (!isfinite(c)) {  // (target, inf, [])
    len[si] = 0;
    return;
  }
  uint32_t cnt = 1, cur = t;
  while (cur != s && cnt <= n) {
    cur = (uint32_t)(st[cur] & 0xFFFFFFFFull);
    ++cnt;
  }
  len[si] = cnt;
  if (cnt > max_len) return;  // caller sees len > max_len and retries with a larger buffer
  uint32_t* p = paths + (size_t)si * max_len;
  cur = t;
  for (uint32_t i = cnt; i-- > 0;) {
    p[i] = cur;
    cur = (uint32_t)(st[cur] & 0xFFFFFFFFull);
  }
}

// ---- cozo_gpu_sssp_goals read-out: pair i = si * n_goals + gi of a chunk ----
// cost of every pair and, when `len` is given, its path length in nodes (0 when unreachable); len[c * n_goals] = 0 so
// that an exclusive scan over c * n_goals + 1 entries leaves the chunk's total in the last one
__global__ void sssp_goal_len_kernel(const unsigned long long* state, uint32_t n, const uint32_t* sources,
                                     const uint32_t* goals, uint32_t n_goals, uint32_t c, float* cost, uint64_t* len) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t pairs = (uint64_t)c * n_goals;
  if (len && i == pairs) len[i] = 0;
  if (i >= pairs) return;
  const uint32_t si = (uint32_t)(i / n_goals);
  const unsigned long long* st = state + (size_t)si * n;
  const uint32_t s = sources[si], t = goals[i % n_goals];
  const float d = __uint_as_float((uint32_t)(st[t] >> 32));
  cost[i] = d;
  if (!len) return;
  uint64_t cnt = 0;
  if (isfinite(d)) {
    uint32_t cur = t;
    for (cnt = 1; cur != s && cnt <= n; ++cnt) cur = (uint32_t)(st[cur] & 0xFFFFFFFFull);
  }
  len[i] = cnt;
}

// path of pair i at paths[off[i] .. off[i+1]), start..goal
__global__ void sssp_goal_path_kernel(const unsigned long long* state, uint32_t n, const uint32_t* goals,
                                      uint32_t n_goals, uint32_t c, const uint64_t* off, uint32_t* paths) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint64_t)c * n_goals) return;
  const unsigned long long* st = state + (size_t)(i / n_goals) * n;
  uint32_t cur = goals[i % n_goals];
  for (uint64_t k = off[i + 1]; k-- > off[i];) {
    paths[k] = cur;
    cur = (uint32_t)(st[cur] & 0xFFFFFFFFull);
  }
}

// keep_ties: the tied-predecessor edges that lead back from the goals of one source (one CTA per source).
// C = the goals with a finite cost other than s, closed under "p has a tight edge (p -> v) with v in C, v != s";
// E = those tight edges, one per CSR edge.  Marking is idempotent, so the closure ends on zero-weight tied cycles too.
// The out-CSR is scanned in rounds (the staged in-CSR carries no weights), as betweenness_kernel walks its tie DAG.
__device__ __forceinline__ bool tie_edge(const unsigned long long* st, const uint8_t* mark, uint32_t s, float du,
                                         uint32_t v, float w) {
  return v != s && mark[v] && du + w == __uint_as_float((uint32_t)(st[v] >> 32));
}

__global__ void __launch_bounds__(256) sssp_tie_mark_kernel(const uint32_t* __restrict__ out_ptr,
                                                            const uint32_t* __restrict__ out_idx,
                                                            const float* __restrict__ out_w, uint32_t n,
                                                            const uint32_t* __restrict__ sources, GoalSet gs, uint32_t c,
                                                            const unsigned long long* state, uint8_t* mark_buf,
                                                            uint64_t* count) {
  const uint32_t si = blockIdx.x;
  if (si >= c) return;
  const unsigned long long* st = state + (size_t)si * n;
  uint8_t* mark = mark_buf + (size_t)si * n;
  const uint32_t s = sources[si];
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ int s_any;
  __shared__ unsigned long long s_cnt[32];
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) mark[v] = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < gs.n; i += blockDim.x) {
    const uint32_t t = gs.goals[i];
    if (t != s && isfinite(__uint_as_float((uint32_t)(st[t] >> 32)))) mark[t] = 1;
  }
  for (;;) {
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    bool any_local = false;
    for (uint32_t u = warp; u < n; u += nwarps) {
      if (mark[u]) continue;  // warp-uniform: read before any lane of this warp can set it
      const float du = __uint_as_float((uint32_t)(st[u] >> 32));
      if (!isfinite(du)) continue;
      bool hit = false;
      for (uint32_t k = out_ptr[u] + lane; k < out_ptr[u + 1] && !hit; k += 32)
        hit = tie_edge(st, mark, s, du, out_idx[k], out_w ? out_w[k] : 1.0f);
      if (__ballot_sync(0xffffffffu, hit)) {
        if (lane == 0) mark[u] = 1;
        any_local = true;
      }
      __syncwarp();
    }
    if (any_local) s_any = 1;
    __syncthreads();
    const int any = s_any;
    __syncthreads();
    if (!any) break;
  }
  unsigned long long cnt = 0;
  for (uint32_t u = warp; u < n; u += nwarps) {
    const float du = __uint_as_float((uint32_t)(st[u] >> 32));
    if (!mark[u] || !isfinite(du)) continue;  // a tight edge into C starts in C
    for (uint32_t k = out_ptr[u] + lane; k < out_ptr[u + 1]; k += 32)
      cnt += tie_edge(st, mark, s, du, out_idx[k], out_w ? out_w[k] : 1.0f) ? 1ull : 0ull;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) s_cnt[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (uint32_t w = 0; w < nwarps; ++w) t += s_cnt[w];
    count[si] = t;
    if (si == c - 1) count[c] = 0;  // scanned over c + 1 entries: the chunk's total lands in the last
  }
}

// the edges counted above as (v, p) pairs at edges[2 * off[si] ...], in no particular order within a source
__global__ void __launch_bounds__(256) sssp_tie_write_kernel(const uint32_t* __restrict__ out_ptr,
                                                             const uint32_t* __restrict__ out_idx,
                                                             const float* __restrict__ out_w, uint32_t n,
                                                             const uint32_t* __restrict__ sources, uint32_t c,
                                                             const unsigned long long* state, const uint8_t* mark_buf,
                                                             const uint64_t* off, uint32_t* edges) {
  const uint32_t si = blockIdx.x;
  if (si >= c) return;
  const unsigned long long* st = state + (size_t)si * n;
  const uint8_t* mark = mark_buf + (size_t)si * n;
  const uint32_t s = sources[si];
  const int lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  __shared__ unsigned long long s_at;
  if (threadIdx.x == 0) s_at = off[si];
  __syncthreads();
  for (uint32_t u = warp; u < n; u += nwarps) {
    const float du = __uint_as_float((uint32_t)(st[u] >> 32));
    if (!mark[u] || !isfinite(du)) continue;
    for (uint32_t k = out_ptr[u] + lane; k < out_ptr[u + 1]; k += 32) {
      const uint32_t v = out_idx[k];
      if (!tie_edge(st, mark, s, du, v, out_w ? out_w[k] : 1.0f)) continue;
      const unsigned long long at = atomicAdd(&s_at, 1ull);
      edges[2 * at] = v;
      edges[2 * at + 1] = u;
    }
  }
}

__global__ void sssp_unpack_kernel(const unsigned long long* state, uint64_t total, float* dist, uint32_t* pred) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  unsigned long long s = state[i];
  if (dist) dist[i] = __uint_as_float((uint32_t)(s >> 32));
  if (pred) pred[i] = (uint32_t)(s & 0xFFFFFFFFull);
}

// closeness of one source: nc^2 / total / (n-1), nc counting the source itself
// (all_pairs_shortest_path.rs:118-120)
__global__ void __launch_bounds__(256) closeness_kernel(const unsigned long long* state, uint32_t n, uint32_t n_src,
                                                        uint32_t src_base, float* out) {
  const uint32_t si = blockIdx.x;
  if (si >= n_src) return;
  const unsigned long long* st = state + (size_t)si * n;
  double tot = 0.0;
  uint32_t cnt = 0;
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) {
    float d = __uint_as_float((uint32_t)(st[v] >> 32));
    if (isfinite(d)) {
      tot += (double)d;
      cnt++;
    }
  }
  __shared__ double sh_t[8];
  __shared__ uint32_t sh_c[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    tot += __shfl_xor_sync(0xffffffffu, tot, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) {
    sh_t[warp] = tot;
    sh_c[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    uint32_t c = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
      t += sh_t[i];
      c += sh_c[i];
    }
    float nc = (float)c;
    float total = (float)t;
    out[src_base + si] = nc * nc / total / (float)(n - 1);
  }
}

// Betweenness of one source (Brandes form of all_pairs_shortest_path.rs:54-68:
// every tied shortest path adds 1/l to each interior node, i.e. node v receives
// sigma_st(v)/sigma_st per target t).  sigma and delta are iterated to their
// fixed points over the shortest-path DAG { (u,v) : fl32(dist[u]+w) == dist[v] }.
__global__ void __launch_bounds__(256) betweenness_kernel(const uint32_t* __restrict__ out_ptr,
                                                          const uint32_t* __restrict__ out_idx,
                                                          const float* __restrict__ out_w, uint32_t n,
                                                          const uint32_t* __restrict__ sources, uint32_t n_src,
                                                          const unsigned long long* state, double* sigma_buf,
                                                          double* delta_buf, int* cyclic) {
  const uint32_t si = blockIdx.x;
  if (si >= n_src) return;
  const unsigned long long* st = state + (size_t)si * n;
  double* sigma = sigma_buf + (size_t)si * 2 * n;
  double* sigma2 = sigma + n;
  double* delta = delta_buf + (size_t)si * 2 * n;
  double* delta2 = delta + n;
  const uint32_t s = sources[si];
  __shared__ int s_any, s_cyc;
  if (threadIdx.x == 0) s_cyc = 0;
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) {
    sigma[v] = v == s ? 1.0 : 0.0;
    sigma2[v] = 0.0;
    delta[v] = 0.0;
    delta2[v] = 0.0;
  }
  __syncthreads();
  // sigma: push along DAG edges until nothing changes (<= DAG depth rounds)
  for (uint32_t round = 0; round < n + 1; ++round) {
    if (threadIdx.x == 0) s_any = 0;
    for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) sigma2[v] = v == s ? 1.0 : 0.0;
    __syncthreads();
    for (uint32_t u = threadIdx.x; u < n; u += blockDim.x) {
      const float du = __uint_as_float((uint32_t)(st[u] >> 32));
      if (!isfinite(du) || sigma[u] == 0.0) continue;
      for (uint32_t k = out_ptr[u]; k < out_ptr[u + 1]; ++k) {
        const uint32_t v = out_idx[k];
        if (v == s) continue;
        const float dv = __uint_as_float((uint32_t)(st[v] >> 32));
        if (du + (out_w ? out_w[k] : 1.0f) == dv) atomicAdd(&sigma2[v], sigma[u]);
      }
    }
    __syncthreads();
    for (uint32_t v = threadIdx.x; v < n; v += blockDim.x)
      if (sigma2[v] != sigma[v]) s_any = 1;
    __syncthreads();
    const int any = s_any;
    double* t = sigma;
    sigma = sigma2;
    sigma2 = t;
    __syncthreads();
    if (!any) break;
    // an acyclic tie graph settles within n rounds; still changing => a zero-weight cycle of tied paths
    // (the reference's path enumeration, all_pairs_shortest_path.rs:54-68, does not terminate on it either)
    if (round == n && threadIdx.x == 0) {
      atomicExch(cyclic, 1);
      s_cyc = 1;
    }
  }
  __syncthreads();
  if (s_cyc) return;
  // delta: pull from DAG successors until nothing changes
  for (uint32_t round = 0; round < n + 1; ++round) {
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    for (uint32_t u = threadIdx.x; u < n; u += blockDim.x) {
      const float du = __uint_as_float((uint32_t)(st[u] >> 32));
      double acc = 0.0;
      if (isfinite(du) && sigma[u] != 0.0) {
        for (uint32_t k = out_ptr[u]; k < out_ptr[u + 1]; ++k) {
          const uint32_t v = out_idx[k];
          if (v == s) continue;
          const float dv = __uint_as_float((uint32_t)(st[v] >> 32));
          if (du + (out_w ? out_w[k] : 1.0f) == dv) acc += sigma[u] / sigma[v] * (1.0 + delta[v]);
        }
      }
      delta2[u] = acc;
      if (acc != delta[u]) s_any = 1;
    }
    __syncthreads();
    const int any = s_any;
    double* t = delta;
    delta = delta2;
    delta2 = t;
    __syncthreads();
    if (!any) break;
  }
  // leave this source's dependencies in the first half of its delta block for the ordered reduction
  double* out = delta_buf + (size_t)si * 2 * n;
  for (uint32_t v = threadIdx.x; v < n; v += blockDim.x) {
    const double d = v != s ? delta[v] : 0.0;
    if (out != delta) out[v] = d;
    else if (v == s) out[v] = 0.0;
  }
}

// "sums merged serially in source order" (all_pairs_shortest_path.rs:72-77): one thread per node adds the
// per-source dependencies in source order — no atomics, run-to-run identical
__global__ void __launch_bounds__(256) betweenness_reduce_kernel(const double* __restrict__ delta_buf, uint32_t n,
                                                                 uint32_t n_src, double* __restrict__ bc) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  double acc = bc[v];
  for (uint32_t si = 0; si < n_src; ++si) acc += delta_buf[(size_t)si * 2 * n + v];
  bc[v] = acc;
}

// ClusteringCoefficients (fixed_rule/algos/triangles.rs:59-98): one warp per node u.  For every
// position i of u's (sorted, duplicate-keeping) out-neighbour list the lanes sweep the positions j
// whose value is smaller and test membership of that value in adj(edges[i]) by binary search.
// Integer work: counts are exact, cc is the same f64 expression as the reference.
__global__ void __launch_bounds__(256) clustering_kernel(const uint32_t* __restrict__ out_ptr,
                                                         const uint32_t* __restrict__ out_idx, uint32_t n,
                                                         double* __restrict__ cc,
                                                         unsigned long long* __restrict__ n_tri,
                                                         unsigned long long* __restrict__ degree) {
  const int lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (u >= n) return;
  const uint32_t b = out_ptr[u], e = out_ptr[u + 1];
  const uint32_t deg = e - b;
  unsigned long long t = 0;
  if (deg >= 2) {
    uint32_t lo_end = b;  // first position whose value is >= a (the list is sorted, a is non-decreasing in i)
    for (uint32_t i = b; i < e; ++i) {
      const uint32_t a = out_idx[i];
      while (lo_end < e && out_idx[lo_end] < a) ++lo_end;
      const uint32_t ab = out_ptr[a], ae = out_ptr[a + 1];
      for (uint32_t j = b + lane; j < lo_end; j += 32) {
        const uint32_t v = out_idx[j];
        uint32_t lo = ab, hi = ae;
        while (lo < hi) {
          uint32_t mid = (lo + hi) >> 1;
          if (out_idx[mid] < v) lo = mid + 1;
          else hi = mid;
        }
        t += (lo < ae && out_idx[lo] == v) ? 1ull : 0ull;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  if (lane == 0) {
    degree[u] = deg;
    n_tri[u] = t;
    cc[u] = deg < 2 ? 0.0 : 2. * (double)t / ((double)deg * ((double)deg - 1.));
  }
}

__global__ void f64_to_f32_kernel(const double* in, uint32_t n, float* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}

}  // namespace cozo
