// pagerank_pb.cuh — device code of the propagation-blocking PageRank engine (pagerank.cu, mode 1): the staging
// kernels and the bodies of the four per-iteration passes.  Kept in a header so that the SAME source is compiled by
// nvcc into libcozo_gpu.so and, by tests/emu (a CPU SIMT emulator, test infrastructure), into a host program that runs
// the passes thread for thread.
#pragma once
#include "common.cuh"

namespace cozo {

constexpr double ERR_SCALE = 4611686018427387904.0;  // 2^62: |delta| accumulated as exact u64 fixed point

// exact, order-independent error accumulation: |delta| as u64 fixed point (2^-62 units)
__device__ __forceinline__ void block_add_err(unsigned long long e, unsigned long long* out) {
  __shared__ unsigned long long sh[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if (lane == 0) sh[warp] = e;
  __syncthreads();
  if (warp == 0) {
    int nw = (blockDim.x + 31) >> 5;
    unsigned long long v = lane < nw ? sh[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0 && v) atomicAdd(out, v);
  }
}
__device__ __forceinline__ unsigned long long err_fixed(float nw, float old) {
  return __double2ull_rn((double)fabsf(nw - old) * ERR_SCALE);
}


struct PbArgs {
  uint32_t n, NH, GS, WIN, G, NB;
  const uint32_t *hptr, *mptr, *od;
  const uint16_t *hub_idx, *a_src, *b_pos;
  const uint32_t *ctab, *rowstart;
  const uint4* items;
  uint32_t n_items;
  const float* contrib_old;
  float *contrib_new, *scores, *val, *msum, *part_a, *part_z;
  float base, damping;
  unsigned long long* err;  // err[0] = fixed-point error, err[1] = row-group counter of K_F
};

// ---- staging kernels --------------------------------------------------------------------------------------
// per row: how many of its (slot-sorted) in-neighbours are hub sources (slot < NH)
__global__ void pb_row_split_kernel(const uint32_t* __restrict__ in_ptr, const uint32_t* __restrict__ in_idx, uint32_t n,
                                    uint32_t NH, uint32_t* hcnt, uint32_t* mcnt) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n) return;
  if (r == n) {
    hcnt[n] = 0;
    mcnt[n] = 0;
    return;
  }
  uint32_t lo = in_ptr[r], hi = in_ptr[r + 1];
  const uint32_t b = lo, e = hi;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (in_idx[mid] < NH) lo = mid + 1;
    else hi = mid;
  }
  hcnt[r] = lo - b;
  mcnt[r] = e - lo;
}
// one warp per row: hub entries -> hub_idx (row-major), M entries -> (group key, packed (Mpos, src in tile))
__global__ void pb_emit_kernel(const uint32_t* __restrict__ in_ptr, const uint32_t* __restrict__ in_idx,
                               const uint32_t* __restrict__ hptr, const uint32_t* __restrict__ mptr, uint32_t n,
                               uint32_t NH, uint32_t GS, uint16_t* hub_idx, uint32_t* key, unsigned long long* val) {
  const uint32_t r = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const uint32_t b = in_ptr[r], e = in_ptr[r + 1];
  const uint32_t h0 = hptr[r], hc = hptr[r + 1] - h0, m0 = mptr[r];
  for (uint32_t k = b + lane; k < e; k += 32) {
    const uint32_t o = k - b, src = in_idx[k];
    if (o < hc) {
      hub_idx[h0 + o] = (uint16_t)src;
    } else {
      const uint32_t mpos = m0 + (o - hc), s2 = src - NH;
      key[mpos] = s2 / GS;
      val[mpos] = ((unsigned long long)mpos << 16) | (s2 % GS);
    }
  }
}
__global__ void pb_group_bounds_kernel(const uint32_t* __restrict__ skey, uint64_t M, uint32_t* gfirst) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  if (i == 0 || skey[i] != skey[i - 1]) gfirst[skey[i]] = (uint32_t)i;
}
__global__ void pb_ctab_init_kernel(uint32_t* ctab, uint32_t NBp1, uint32_t G, const uint32_t* __restrict__ gend_pad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint64_t)NBp1 * G) return;
  ctab[i] = gend_pad[i % G];  // "no entry of this group at or after this bin"
}
// sorted (group-major) entries -> padded group-major arrays + the cell table
__global__ void pb_place_kernel(const uint32_t* __restrict__ skey, const unsigned long long* __restrict__ sval, uint64_t M,
                                const uint32_t* __restrict__ gfirst, const uint32_t* __restrict__ gbase, uint32_t WIN,
                                uint32_t G, uint16_t* a_src, uint16_t* b_pos, uint32_t* ctab) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const uint32_t g = skey[i];
  const unsigned long long v = sval[i];
  const uint32_t mpos = (uint32_t)(v >> 16);
  const uint32_t ip = gbase[g] + (uint32_t)(i - gfirst[g]);
  a_src[ip] = (uint16_t)(v & 0xFFFFull);
  b_pos[ip] = (uint16_t)(mpos % WIN);
  const uint32_t bin = mpos / WIN;
  const bool first = i == gfirst[g];
  const uint32_t prev = first ? 0u : (uint32_t)(sval[i - 1] >> 16) / WIN;
  if (first) {
    for (uint32_t b = 0; b <= bin; ++b) ctab[(size_t)b * G + g] = ip;
  } else if (prev != bin) {
    for (uint32_t b = prev + 1; b <= bin; ++b) ctab[(size_t)b * G + g] = ip;
  }
}
__global__ void pb_rowstart_kernel(const uint32_t* __restrict__ mptr, uint32_t n, uint32_t WIN, uint32_t NBp1,
                                   uint32_t* rowstart) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= NBp1) return;
  const unsigned long long target = (unsigned long long)b * WIN;
  uint32_t lo = 0, hi = n;  // first row r in [0,n] with mptr[r] >= target (mptr[n] = Mtot)
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if ((unsigned long long)mptr[mid] < target) lo = mid + 1;
    else hi = mid;
  }
  rowstart[b] = lo;
}

// ---- K_A: contribution tile in shared memory (cp.async.bulk), group-major entry stream -> dense value stream
__device__ __forceinline__ void pb_gather_body(const PbArgs& a, uint8_t* pb_smem) {
  float* win = reinterpret_cast<float*>(pb_smem);
  uint64_t* bar = reinterpret_cast<uint64_t*>(pb_smem + (size_t)a.GS * 4);
  const uint32_t per = (a.n_items + gridDim.x - 1) / gridDim.x;
  const uint32_t i0 = blockIdx.x * per, i1 = min(a.n_items, i0 + per);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  uint32_t cur_g = NONE, phase = 0;
  for (uint32_t it = i0; it < i1; ++it) {
    const uint4 item = a.items[it];
    if (item.x != cur_g) {
      __syncthreads();  // every thread is done with the previous tile
      if (threadIdx.x == 0) {
        const uint32_t first = a.NH + item.x * a.GS;
        const uint32_t cnt = min(a.GS, a.n - first);
        const uint32_t bytes = ((cnt + 3u) & ~3u) * 4u;  // the contribution arrays carry slack behind n
        fence_proxy_async_smem();
        mbar_expect_tx(bar, bytes);
        for (uint32_t off = 0; off < bytes; off += 32768u)
          bulk_g2s(reinterpret_cast<uint8_t*>(win) + off, reinterpret_cast<const uint8_t*>(a.contrib_old + first) + off,
                   min(32768u, bytes - off), bar);
      }
      mbar_wait(bar, phase);
      phase ^= 1u;
      cur_g = item.x;
    }
    // 16 entries per thread and trip: two 128-bit index loads in flight before the first gather
    for (uint32_t i = item.y + threadIdx.x * 8; i < item.z; i += 1024 * 16) {
      const uint32_t i2 = i + 1024 * 8;
      const bool two = i2 < item.z;
      const uint4 s = *reinterpret_cast<const uint4*>(a.a_src + i);  // 8 x u16
      const uint4 t = two ? *reinterpret_cast<const uint4*>(a.a_src + i2) : make_uint4(0, 0, 0, 0);
      float4 v0, v1;
      v0.x = win[s.x & 0xFFFFu];
      v0.y = win[s.x >> 16];
      v0.z = win[s.y & 0xFFFFu];
      v0.w = win[s.y >> 16];
      v1.x = win[s.z & 0xFFFFu];
      v1.y = win[s.z >> 16];
      v1.z = win[s.w & 0xFFFFu];
      v1.w = win[s.w >> 16];
      *reinterpret_cast<float4*>(a.val + i) = v0;
      *reinterpret_cast<float4*>(a.val + i + 4) = v1;
      if (two) {
        v0.x = win[t.x & 0xFFFFu];
        v0.y = win[t.x >> 16];
        v0.z = win[t.y & 0xFFFFu];
        v0.w = win[t.y >> 16];
        v1.x = win[t.z & 0xFFFFu];
        v1.y = win[t.z >> 16];
        v1.z = win[t.w & 0xFFFFu];
        v1.w = win[t.w >> 16];
        *reinterpret_cast<float4*>(a.val + i2) = v0;
        *reinterpret_cast<float4*>(a.val + i2 + 4) = v1;
      }
    }
  }
}

// ---- K_B: per bin, scatter the value stream into the window, then sum the rows of the bin -----------------
template <int THREADS>
__device__ __forceinline__ void pb_accumulate_body(const PbArgs& a, uint8_t* pb_smem) {
  float* window = reinterpret_cast<float*>(pb_smem);
  uint32_t* pre = reinterpret_cast<uint32_t*>(pb_smem + (size_t)a.WIN * 4);  // [G+1] bin-relative start of every cell
  uint32_t* cstart = pre + a.G + 1;                                          // [G]   group-major start of every cell
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = THREADS / 32;
  const uint32_t G = a.G;
  for (uint32_t b = blockIdx.x; b < a.NB; b += gridDim.x) {
    // cell table of this bin -> smem, exclusive scan of the cell sizes
    for (uint32_t g = threadIdx.x; g < G; g += THREADS) {
      const uint32_t c0 = a.ctab[(size_t)b * G + g], c1 = a.ctab[(size_t)(b + 1) * G + g];
      cstart[g] = c0;
      pre[g + 1] = c1 - c0;
    }
    __syncthreads();
    if (warp == 0) {
      uint32_t run = 0;
      for (uint32_t g0 = 0; g0 < G; g0 += 32) {
        const uint32_t g = g0 + lane;
        const uint32_t c = g < G ? pre[g + 1] : 0;
        uint32_t x = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
          if (lane >= o) x += y;
        }
        if (g < G) pre[g + 1] = run + x;
        run += __shfl_sync(0xffffffffu, x, 31);
      }
      if (lane == 0) pre[0] = 0;
    }
    __syncthreads();
    const uint32_t total = pre[G];
    // phase 1: flat index j over the bin's entries -> (group, group-major index) -> window[pos] = val
    for (uint32_t j0 = warp * 128; j0 < total; j0 += NW * 128) {  // a warp takes 128 consecutive entries
      uint32_t lo = 0, hi = G;  // largest g with pre[g] <= j0 (warp-uniform)
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pre[mid] <= j0) lo = mid;
        else hi = mid;
      }
      uint32_t g = lo, idx[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t j = j0 + 32 * u + lane;
        idx[u] = NONE;
        if (j < total) {
          while (pre[g + 1] <= j) ++g;
          idx[u] = cstart[g] + (j - pre[g]);
        }
      }
      float v[4];
      uint32_t p[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        p[u] = idx[u] != NONE ? a.b_pos[idx[u]] : 0u;
        v[u] = idx[u] != NONE ? a.val[idx[u]] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (idx[u] != NONE) window[p[u]] = v[u];
    }
    __syncthreads();
    // phase 2: rows.  Owned rows start inside this bin; a row started earlier contributes a carry-in piece.
    const unsigned long long base = (unsigned long long)b * a.WIN;
    const uint32_t r0 = a.rowstart[b], r1 = a.rowstart[b + 1];
    if (warp == 0) {
      const unsigned long long first = r0 <= a.n ? (unsigned long long)a.mptr[r0] : base;
      uint32_t cend = (uint32_t)(min(first, base + total) - base);  // [0, cend) belongs to row r0-1
      if (first <= base) cend = 0;
      if (cend) {
        float s = 0.f;
        for (uint32_t j = lane; j < cend; j += 32) s += window[j];
        s = warp_sum(s);
        if (lane == 0) a.part_a[b] = s;
      }
    }
    for (uint32_t rg = r0 + warp * 32; rg < r1; rg += NW * 32) {
      const uint32_t r = rg + lane;
      uint32_t s = 0, e = 0;
      bool partial = false;
      if (r < r1) {
        const unsigned long long ms = a.mptr[r], me = a.mptr[r + 1];
        s = (uint32_t)(ms - base);
        partial = me > base + a.WIN;
        e = (uint32_t)(min(me, base + a.WIN) - base);
      }
      const uint32_t len = e - s;
      float sum = 0.f;
      const uint32_t longmask = __ballot_sync(0xffffffffu, len > 64);
      if (len <= 64)
        for (uint32_t j = s; j < e; ++j) sum += window[j];
      uint32_t lm = longmask;
      while (lm) {  // long rows: the whole warp sums one row, lanes strided, shuffle tree
        const int l = __ffs(lm) - 1;
        lm &= lm - 1;
        const uint32_t ls = __shfl_sync(0xffffffffu, s, l), le = __shfl_sync(0xffffffffu, e, l);
        float p = 0.f;
        for (uint32_t j = ls + lane; j < le; j += 32) p += window[j];
        p = warp_sum(p);
        if (lane == l) sum = p;
      }
      if (r < r1) {
        if (partial) a.part_z[b] = sum;
        else a.msum[r] = sum;
      }
    }
    __syncthreads();  // the window is reused by the next bin
  }
}

// ---- K_S: rows longer than one window ------------------------------------------------------------------
__global__ void pb_straddle_kernel(const PbArgs a) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.NB) return;
  const uint32_t r0 = a.rowstart[b], r1 = a.rowstart[b + 1];
  if (r1 <= r0) return;
  const uint32_t r = r1 - 1;  // the last row that starts in this bin
  const unsigned long long me = a.mptr[r + 1], lim = (unsigned long long)(b + 1) * a.WIN;
  if (me <= lim) return;
  float s = a.part_z[b];
  const uint32_t bl = (uint32_t)((me - 1) / a.WIN);
  for (uint32_t bb = b + 1; bb <= bl; ++bb) s += a.part_a[bb];
  a.msum[r] = s;
}

// ---- K_F: hub part through the shared-memory hub table, + M part, new score / contribution / error ------------
constexpr uint32_t KF_THREADS = 256;
constexpr uint32_t KF_STAGE = 2048;  // u16 hub indices staged per warp
__device__ __forceinline__ void pb_final_body(const PbArgs& a, uint8_t* pb_smem) {
  float* hub = reinterpret_cast<float*>(pb_smem);
  const uint32_t nh4 = (a.NH + 3u) & ~3u;
  uint64_t* bar = reinterpret_cast<uint64_t*>(pb_smem + (size_t)nh4 * 4);
  uint16_t* stage_all = reinterpret_cast<uint16_t*>(pb_smem + (size_t)nh4 * 4 + 16);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint16_t* stage = stage_all + (size_t)warp * KF_STAGE;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (a.NH) {
    if (threadIdx.x == 0) {
      const uint32_t bytes = nh4 * 4u;
      fence_proxy_async_smem();
      mbar_expect_tx(bar, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u)
        bulk_g2s(reinterpret_cast<uint8_t*>(hub) + off, reinterpret_cast<const uint8_t*>(a.contrib_old) + off,
                 min(32768u, bytes - off), bar);
    }
    mbar_wait(bar, 0);
  }
  uint32_t* ctr = reinterpret_cast<uint32_t*>(a.err + 1);
  const uint32_t n_groups = (a.n + 31) / 32;
  unsigned long long e = 0;
  for (;;) {
    uint32_t rg = 0;
    if (lane == 0) rg = atomicAdd(ctr, 4u);
    rg = __shfl_sync(0xffffffffu, rg, 0);
    if (rg >= n_groups) break;
    const uint32_t rg_end = min(rg + 4u, n_groups);
    for (; rg < rg_end; ++rg) {
      const uint32_t r = rg * 32 + lane;
      const bool valid = r < a.n;
      const uint32_t h0 = valid ? a.hptr[r] : 0, h1 = valid ? a.hptr[r + 1] : 0;
      const uint32_t nvalid = min(32u, a.n - rg * 32);
      const uint32_t gb = __shfl_sync(0xffffffffu, h0, 0), ge = __shfl_sync(0xffffffffu, h1, nvalid - 1);
      const uint32_t T = ge - gb;
      float s = 0.f;
      if (T <= KF_STAGE) {
        for (uint32_t i = lane; i < T; i += 32) stage[i] = a.hub_idx[gb + i];
        __syncwarp();
        // as in K_B: a lane sums a row of at most 64 entries, longer rows are summed by the whole warp (lanes strided,
        // shuffle tree), so that no f32 chain is longer than 64 additions (a serial chain of 2048 equal terms drifts by
        // about 2e-5 relative)
        const uint32_t len = h1 - h0;
        if (len <= 64)
          for (uint32_t j = h0 - gb; j < h1 - gb; ++j) s += hub[stage[j]];
        uint32_t lm = __ballot_sync(0xffffffffu, len > 64);
        while (lm) {
          const int l = __ffs(lm) - 1;
          lm &= lm - 1;
          const uint32_t ls = __shfl_sync(0xffffffffu, h0, l) - gb, le = __shfl_sync(0xffffffffu, h1, l) - gb;
          float p = 0.f;
          for (uint32_t j = ls + lane; j < le; j += 32) p += hub[stage[j]];
          p = warp_sum(p);
          if (lane == l) s = p;
        }
        __syncwarp();
      } else {
        for (uint32_t l = 0; l < nvalid; ++l) {  // long hub lists: the warp sums one row at a time
          const uint32_t rb = __shfl_sync(0xffffffffu, h0, l), re = __shfl_sync(0xffffffffu, h1, l);
          float p = 0.f;
          for (uint32_t i = rb + lane; i < re; i += 32) p += hub[a.hub_idx[i]];
          p = warp_sum(p);
          if ((uint32_t)lane == l) s = p;
        }
      }
      if (valid) {
        const float tot = s + a.msum[r];
        const float nw = a.base + a.damping * tot;
        e += err_fixed(nw, a.scores[r]);
        a.scores[r] = nw;
        const uint32_t d = a.od[r];
        a.contrib_new[r] = d ? nw / (float)d : 0.f;
      }
    }
  }
  block_add_err(e, a.err);
}

}  // namespace cozo
