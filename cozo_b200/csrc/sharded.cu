// sharded.cu — the row-sharded corpus behind the C ABI (SURVEY.md §8b "Multi-GPU", §8e), and the source-sharded
// graph calls at the end of this file (replicated graph, sources split over the ranks, one exchange at the end).
// The HNSW corpus:
// one process per GPU, every rank holds one shard (its own vectors + its own HNSW graph).
//   cozo_gpu_hnsw_search_sharded = query broadcast -> per-shard hnsw_knn -> exchange of the
//   per-shard top-k lists -> k-way merge to global ids, all inside libcozo_gpu.so.
// The reference answers one query at a time from one index relation (query/ra.rs:1102-1119,
// runtime/hnsw.rs:869-1012); the sharded result is the k-NN over the union of the shards as
// searched shard by shard.
//
// Two exchanges:
//   NCCL   ONE ncclAllGather per list (ids, distances), grouped, on the search stream;
//   FUSED  the search kernel's epilogue stores every query's top-k straight into all peers'
//          gather buffers (cudaMalloc memory opened on the peers through CUDA IPC handles, plain
//          st.global over NVLink), then one flag barrier kernel — no collective kernel at all.
// NCCL is resolved with dlopen at first use (the host process may already carry its own copy,
// e.g. the one bundled with PyTorch): there is no link-time dependency.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <type_traits>
#include <vector>

#include "graph_host.hpp"
#include "hnsw_host.hpp"

namespace cozo {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
};

static NcclApi g_nccl;
static std::mutex g_nccl_mu;

static int nccl_load() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.lib) return 0;
  void* lib = nullptr;
  const char* env = getenv("COZO_GPU_NCCL_LIB");
  if (env && *env) lib = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  // a copy the process already mapped (PyTorch's bundled libnccl.so.2) wins over the system one
  if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) return set_error(COZO_GPU_ENODEV, "libnccl.so.2 not found (%s); set COZO_GPU_NCCL_LIB", dlerror());
  NcclApi a;
  a.lib = lib;
#define SYM(field, name)                                                                      \
  a.field = reinterpret_cast<decltype(a.field)>(dlsym(lib, name));                            \
  if (!a.field) return set_error(COZO_GPU_ENODEV, "libnccl lacks %s", name)
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllGather, "ncclAllGather");
  SYM(Broadcast, "ncclBroadcast");
  SYM(GroupStart, "ncclGroupStart");
  SYM(GroupEnd, "ncclGroupEnd");
  SYM(GetErrorString, "ncclGetErrorString");
  SYM(GetVersion, "ncclGetVersion");
#undef SYM
  g_nccl = a;
  return 0;
}

#define COZO_NCCL(call)                                                                                  \
  do {                                                                                                   \
    ncclResult_t _r = (call);                                                                            \
    if (_r != ncclSuccess)                                                                               \
      return ::cozo::set_error(COZO_GPU_ECUDA, "%s failed: %s (%s:%d)", #call, g_nccl.GetErrorString(_r), \
                               __FILE__, __LINE__);                                                      \
  } while (0)

}  // namespace cozo

struct cozo_gpu_shards {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  cozo_gpu_hnsw* shard = nullptr;
  std::vector<uint64_t> offsets;  // global id of every shard's row 0 (row-contiguous partition)
  uint64_t total_rows = 0;
  int dtype = 0;  // every shard's VecElementType, agreed at attach: 0 = F32, 1 = F64, -1 = the shards mix them
  uint64_t* d_offsets = nullptr;
  cudaStream_t stream = nullptr;
  int exchange = 0;  // 0 = NCCL all-gather, 1 = fused peer stores
  std::string fused_why_not;
  // capacity of the exchange buffers: `tile` queries of `k` results, distances of `dsz_cap` bytes (4 or 8)
  uint32_t tile_cap = 0, k_cap = 0, dsz_cap = 0;
  // one IPC-shareable block per rank: [flags 256 B][set 0: ids S*tile*k u32, dist S*tile*k][set 1: ...]
  uint8_t* block = nullptr;
  size_t block_bytes = 0;
  uint8_t* peer_block[COZO_GPU_MAX_PEERS] = {};  // this rank's view of every rank's block (self = block)
  uint32_t* local_ids[2] = {nullptr, nullptr};   // NCCL form: the all-gather's send buffers
  void* local_dist[2] = {nullptr, nullptr};
  uint32_t epoch = 0;
  // running tile counter: consecutive tiles — of one call or of consecutive calls — alternate between the two
  // buffer sets.  A rank may only overwrite a peer's set once that peer has merged what the set held; passing the
  // barrier of tile i proves every peer has finished merging tile i-1 (stream order on the peer), i.e. the OTHER set.
  uint32_t tile_seq = 0;
  int* d_timeout = nullptr;
  // staging of the host-pointer calls (f32 or f64 queries; distances sized for f64)
  void* d_q = nullptr;
  size_t q_bytes = 0;
  uint64_t* d_out_ids = nullptr;
  void* d_out_dist = nullptr;
  uint32_t* d_qstats = nullptr;
  size_t out_rows = 0, out_k = 0;
  uint32_t* d_mask = nullptr;  // row filter verdicts of the host-pointer call, uploaded once per call
  size_t mask_words = 0;
  // the replicated graph of the sharded graph calls (cozo_gpu_graph_attach_sharded); not owned
  cozo_gpu_graph* graph = nullptr;
  uint64_t graph_sum = 0;  // its checksum, agreed at attach
  // the status records of the sharded graph calls: [world + 1] records of 128 bytes, allocated with the group so
  // that no call has to allocate before its status all-gather; the last one is scratch
  uint8_t* d_status = nullptr;
  std::mutex mu;  // one sharded call at a time per communicator (collectives must not interleave)
};

namespace cozo {

struct PeerFlagPtrs {
  uint32_t* p[COZO_GPU_MAX_PEERS];
};

// Cross-rank barrier over IPC-mapped flag words: thread t tells rank t "my stores of `epoch` have
// landed" and waits for rank t's word in its own block.  Release/acquire at system scope order the
// search kernel's peer stores (earlier on this stream) before the flag.
__global__ void shard_barrier_kernel(uint32_t* my_flags, PeerFlagPtrs peers, int rank, int world, uint32_t epoch,
                                     int* timeout) {
  const int t = threadIdx.x;
  if (t >= world) return;
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peers.p[t] + rank), "r"(epoch) : "memory");
  const long long t0 = clock64();
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_flags + t) : "memory");
    if ((int32_t)(v - epoch) >= 0) break;
    if (clock64() - t0 > 40000000000ll) {  // ~20 s: a peer died; never hang the GPU
      *timeout = 1;
      break;
    }
    __nanosleep(200);
  }
}

static size_t ids_bytes(const cozo_gpu_shards* s, uint32_t tile, uint32_t k) {
  // the id list of one set, padded so that the distances after it stay aligned for f64
  return ((size_t)s->world * tile * k * 4 + 255) & ~(size_t)255;
}
static size_t set_bytes(const cozo_gpu_shards* s, uint32_t tile, uint32_t k, uint32_t dsz) {
  return ids_bytes(s, tile, k) * (1 + dsz / 4);  // ids, then distances of dsz bytes
}
static uint32_t* set_ids(uint8_t* blk, const cozo_gpu_shards* s, int b) {
  return reinterpret_cast<uint32_t*>(blk + 256 + (size_t)b * set_bytes(s, s->tile_cap, s->k_cap, s->dsz_cap));
}
template <typename D>
static D* set_dist(uint8_t* blk, const cozo_gpu_shards* s, int b) {
  return reinterpret_cast<D*>(reinterpret_cast<uint8_t*>(set_ids(blk, s, b)) + ids_bytes(s, s->tile_cap, s->k_cap));
}

static void close_peers(cozo_gpu_shards* s) {
  for (int r = 0; r < s->world && r < COZO_GPU_MAX_PEERS; ++r) {
    if (s->peer_block[r] && r != s->rank) cudaIpcCloseMemHandle(s->peer_block[r]);
    s->peer_block[r] = nullptr;
  }
}

// (Re)allocate the exchange buffers for `tile` x `k` distances of `dsz` bytes and, for the fused form, open every peer's
// block.  Collective: all ranks call it with the same arguments.
static int ensure_exchange(cozo_gpu_shards* s, uint32_t tile, uint32_t k, uint32_t dsz) {
  if (tile <= s->tile_cap && k <= s->k_cap && dsz <= s->dsz_cap && s->block) return 0;
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  tile = std::max(tile, s->tile_cap);
  k = std::max(k, s->k_cap);
  dsz = std::max(dsz, s->dsz_cap);
  close_peers(s);
  if (s->block && s->world > 1) {
    // every rank has closed its mappings of the old blocks before any rank frees one (freeing exported memory
    // that an importer still has open is undefined): one tiny all-gather as the rendezvous
    uint32_t* d_tok = nullptr;
    COZO_CUDA(cudaMalloc(&d_tok, 4 * (size_t)(s->world + 1)));
    COZO_NCCL(g_nccl.AllGather(d_tok + s->world, d_tok, 1, ncclUint32, s->comm, s->stream));
    COZO_CUDA(cudaStreamSynchronize(s->stream));
    cudaFree(d_tok);
  }
  if (s->block) cudaFree(s->block);
  s->block = nullptr;
  for (int b = 0; b < 2; ++b) {
    if (s->local_ids[b]) cudaFree(s->local_ids[b]);
    if (s->local_dist[b]) cudaFree(s->local_dist[b]);
    s->local_ids[b] = nullptr;
    s->local_dist[b] = nullptr;
  }
  s->tile_cap = tile;
  s->k_cap = k;
  s->dsz_cap = dsz;
  s->block_bytes = 256 + 2 * set_bytes(s, tile, k, dsz);
  COZO_CUDA(cudaMalloc(&s->block, s->block_bytes));
  COZO_CUDA(cudaMemsetAsync(s->block, 0, 256, s->stream));  // ordered before the handle exchange below
  s->epoch = 0;
  s->tile_seq = 0;
  for (int b = 0; b < 2; ++b) {
    COZO_CUDA(cudaMalloc(&s->local_ids[b], (size_t)tile * k * 4));
    COZO_CUDA(cudaMalloc(&s->local_dist[b], (size_t)tile * k * dsz));
  }
  s->peer_block[s->rank] = s->block;
  if (s->world == 1) {
    s->exchange = get_option("shard.exchange", 1) ? 1 : 0;
    return 0;
  }
  // exchange the IPC handles with one all-gather, open the peers, agree on the outcome
  int want_fused = get_option("shard.exchange", 1) ? 1 : 0;
  if (s->world > COZO_GPU_MAX_PEERS) want_fused = 0;
  cudaIpcMemHandle_t mine;
  memset(&mine, 0, sizeof(mine));
  int ok = want_fused;
  if (ok && cudaIpcGetMemHandle(&mine, s->block) != cudaSuccess) {
    s->fused_why_not = cudaGetErrorString(cudaGetLastError());
    ok = 0;
  }
  const size_t hb = sizeof(cudaIpcMemHandle_t);
  struct Rec {
    cudaIpcMemHandle_t h;
    int ok;
    int pad[15];
  };
  static_assert(sizeof(Rec) == 128, "record is one 128-byte line");
  (void)hb;
  Rec rec{};
  rec.h = mine;
  rec.ok = ok;
  Rec* d_rec = nullptr;
  COZO_CUDA(cudaMalloc(&d_rec, sizeof(Rec) * (size_t)(s->world + 1)));
  COZO_CUDA(cudaMemcpyAsync(d_rec + s->world, &rec, sizeof(Rec), cudaMemcpyHostToDevice, s->stream));
  COZO_NCCL(g_nccl.AllGather(d_rec + s->world, d_rec, sizeof(Rec), ncclUint8, s->comm, s->stream));
  std::vector<Rec> all(s->world);
  COZO_CUDA(cudaMemcpyAsync(all.data(), d_rec, sizeof(Rec) * (size_t)s->world, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  for (int r = 0; r < s->world; ++r) ok &= all[r].ok;
  if (ok) {
    for (int r = 0; r < s->world; ++r) {
      if (r == s->rank) continue;
      void* p = nullptr;
      if (cudaIpcOpenMemHandle(&p, all[r].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        s->fused_why_not = std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(cudaGetLastError());
        ok = 0;
        break;
      }
      s->peer_block[r] = static_cast<uint8_t*>(p);
    }
  }
  // second round: did every rank manage to open every peer?
  rec.ok = ok;
  COZO_CUDA(cudaMemcpyAsync(d_rec + s->world, &rec, sizeof(Rec), cudaMemcpyHostToDevice, s->stream));
  COZO_NCCL(g_nccl.AllGather(d_rec + s->world, d_rec, sizeof(Rec), ncclUint8, s->comm, s->stream));
  COZO_CUDA(cudaMemcpyAsync(all.data(), d_rec, sizeof(Rec) * (size_t)s->world, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  cudaFree(d_rec);
  for (int r = 0; r < s->world; ++r) ok &= all[r].ok;
  if (!ok) {
    close_peers(s);
    s->peer_block[s->rank] = s->block;
    if (want_fused && s->fused_why_not.empty()) s->fused_why_not = "a peer could not map the exchange buffers";
  }
  s->exchange = ok ? 1 : 0;
  return 0;
}

// the device form: everything already in HBM, asynchronous on the communicator's stream.  T is the distance (and
// query) type of the group; d_mask = this rank's filter verdicts (nullptr = no filter).  F64 groups search with `ws64`,
// a workspace of the shard the caller holds until the stream has drained.
template <typename T>
static int sharded_search_dev(cozo_gpu_shards* s, const T* d_q, uint32_t B, uint32_t k, uint32_t ef, double radius,
                              const uint32_t* d_mask, uint64_t* d_out_ids, T* d_out_dist, uint32_t* d_qstats,
                              HnswWorkspace* ws64 = nullptr) {
  constexpr bool f64 = std::is_same<T, double>::value;
  cozo_gpu_hnsw* h = s->shard;
  const uint32_t dim = h->dev.dim;
  uint32_t tile = (uint32_t)std::max<int64_t>(1, get_option("shard.tile", 65536));
  tile = std::min(tile, std::max(B, 1u));
  int rc = ensure_exchange(s, tile, k, sizeof(T));
  if (rc) return rc;
  cudaStream_t st = s->stream;
  for (uint32_t q0 = 0; q0 < B; q0 += tile) {
    const uint32_t nq = std::min(tile, B - q0);
    const int b = (int)(s->tile_seq++ & 1u);  // NOT the tile index of this call: back-to-back single-tile calls must alternate too
    const T* q = d_q + (size_t)q0 * dim;
    uint32_t* qs = d_qstats ? d_qstats + (size_t)q0 * 4 : nullptr;
    T* local_dist = static_cast<T*>(s->local_dist[b]);
    // fused: the gather layout of this tile, [world][nq][k] at the start of set b of every rank
    ScatterDestT<T> sc{};
    const ScatterDestT<T>* scatter = nullptr;
    if (s->exchange == 1) {
      sc.n_dest = (uint32_t)s->world;
      sc.slot = (uint32_t)s->rank;
      for (int r = 0; r < s->world; ++r) {
        sc.ids[r] = set_ids(s->peer_block[r], s, b);
        sc.dist[r] = set_dist<T>(s->peer_block[r], s, b);
      }
      scatter = &sc;
    }
    if constexpr (f64)  // the kernel also writes the local lists: the NCCL form sends them
      rc = hnsw_launch_search_f64(h, ws64, q, nq, k, ef, radius, s->local_ids[b], local_dist, nullptr, qs, st, scatter,
                                  d_mask);
    else if (scatter)
      rc = hnsw_search_dev(h, q, nq, k, ef, radius, nullptr, nullptr, nullptr, qs, st, scatter, d_mask);
    else
      rc = hnsw_search_dev(h, q, nq, k, ef, radius, s->local_ids[b], local_dist, nullptr, qs, st, nullptr, d_mask);
    if (rc) return rc;
    if (s->exchange == 1) {
      if (s->world > 1) {
        PeerFlagPtrs pf{};
        for (int r = 0; r < s->world; ++r) pf.p[r] = reinterpret_cast<uint32_t*>(s->peer_block[r]);
        ++s->epoch;
        shard_barrier_kernel<<<1, 32, 0, st>>>(reinterpret_cast<uint32_t*>(s->block), pf, s->rank, s->world, s->epoch,
                                               s->d_timeout);
        COZO_CUDA(cudaGetLastError());
      }
    } else if (s->world > 1) {
      COZO_NCCL(g_nccl.GroupStart());
      COZO_NCCL(g_nccl.AllGather(s->local_ids[b], set_ids(s->block, s, b), (size_t)nq * k, ncclUint32, s->comm, st));
      COZO_NCCL(g_nccl.AllGather(local_dist, set_dist<T>(s->block, s, b), (size_t)nq * k, f64 ? ncclFloat64 : ncclFloat32,
                                 s->comm, st));
      COZO_NCCL(g_nccl.GroupEnd());
    } else {
      COZO_CUDA(cudaMemcpyAsync(set_ids(s->block, s, b), s->local_ids[b], (size_t)nq * k * 4, cudaMemcpyDeviceToDevice, st));
      COZO_CUDA(cudaMemcpyAsync(set_dist<T>(s->block, s, b), local_dist, (size_t)nq * k * sizeof(T),
                                cudaMemcpyDeviceToDevice, st));
    }
    if constexpr (f64)
      rc = topk_merge_f64_dev(set_dist<T>(s->block, s, b), set_ids(s->block, s, b), (uint32_t)s->world, nq, k,
                              s->d_offsets, d_out_ids + (size_t)q0 * k, d_out_dist + (size_t)q0 * k, st);
    else
      rc = cozo_gpu_topk_merge_dev(set_dist<T>(s->block, s, b), set_ids(s->block, s, b), (uint32_t)s->world, nq, k,
                                   s->d_offsets, d_out_ids + (size_t)q0 * k, d_out_dist + (size_t)q0 * k, st);
    if (rc) return rc;
  }
  return 0;
}

// Argument checks every rank answers alike before any collective: the group's dtype was agreed at attach.
static int check_group(cozo_gpu_shards* s, uint32_t k, uint32_t ef, int want_dtype) {
  if (!s || !s->shard) return set_error(COZO_GPU_EINVAL, "no shard attached (cozo_gpu_hnsw_stage_sharded)");
  if (s->dtype < 0) return set_error(COZO_GPU_EINVAL, "the shards of the group mix F32 and F64 indexes");
  if (s->dtype != want_dtype)
    return set_error(COZO_GPU_EINVAL, want_dtype ? "not an F64 group: use cozo_gpu_hnsw_search_sharded"
                                                 : "F64 group: use cozo_gpu_hnsw_search_sharded_f64");
  if (k == 0) return set_error(COZO_GPU_EINVAL, "k must be positive");
  if (ef == 0) return set_error(COZO_GPU_EINVAL, "ef must be positive");
  return 0;
}

static int check_timeout(cozo_gpu_shards* s) {
  int t = 0;
  COZO_CUDA(cudaMemcpy(&t, s->d_timeout, 4, cudaMemcpyDeviceToHost));
  if (t) return set_error(COZO_GPU_ECUDA, "sharded search: a peer rank did not reach the exchange barrier");
  return 0;
}

}  // namespace cozo

using namespace cozo;

extern "C" int cozo_gpu_shards_unique_id(uint8_t* id) {
  if (!id) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = nccl_load();
  if (rc) return rc;
  ncclUniqueId u;
  COZO_NCCL(g_nccl.GetUniqueId(&u));
  static_assert(sizeof(u) == COZO_GPU_UID_BYTES, "unique id size");
  memcpy(id, &u, sizeof(u));
  return 0;
}

extern "C" int cozo_gpu_shards_init(cozo_gpu_shards_t** out, const uint8_t* id, int rank, int world) {
  if (!out || !id) return set_error(COZO_GPU_EINVAL, "null argument");
  *out = nullptr;
  if (world < 1 || rank < 0 || rank >= world) return set_error(COZO_GPU_EINVAL, "rank %d of %d", rank, world);
  if (world > COZO_GPU_MAX_PEERS) return set_error(COZO_GPU_EUNSUP, "more than %d shards (one NVSwitch domain)", COZO_GPU_MAX_PEERS);
  int rc = ensure_init();
  if (rc) return rc;
  rc = nccl_load();
  if (rc) return rc;
  auto* s = new cozo_gpu_shards();
  s->rank = rank;
  s->world = world;
  auto fail = [&](int code) {
    cozo_gpu_shards_free(s);
    return code;
  };
  if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMalloc(&s->d_timeout, 4) != cudaSuccess || cudaMemset(s->d_timeout, 0, 4) != cudaSuccess ||
      cudaMalloc(&s->d_offsets, (size_t)world * 8) != cudaSuccess ||
      cudaMalloc(&s->d_status, 128 * ((size_t)world + 1)) != cudaSuccess)
    return fail(set_error(COZO_GPU_ECUDA, "shard group creation failed: %s", cudaGetErrorString(cudaGetLastError())));
  ncclUniqueId u;
  memcpy(&u, id, sizeof(u));
  ncclResult_t r = g_nccl.CommInitRank(&s->comm, world, u, rank);
  if (r != ncclSuccess) return fail(set_error(COZO_GPU_ECUDA, "ncclCommInitRank failed: %s", g_nccl.GetErrorString(r)));
  *out = s;
  return 0;
}

extern "C" void cozo_gpu_shards_free(cozo_gpu_shards_t* s) {
  if (!s) return;
  if (s->stream) cudaStreamSynchronize(s->stream);
  close_peers(s);
  void* ptrs[] = {s->block,    s->local_ids[0], s->local_ids[1], s->local_dist[0], s->local_dist[1], s->d_offsets,
                  s->d_timeout, s->d_q,         s->d_out_ids,    s->d_out_dist,    s->d_qstats,      s->d_mask,
                  s->d_status};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  if (s->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(s->comm);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
}

// Collective.  Attaches this rank's shard (staged or built here) and all-gathers the shard sizes:
// shard r owns the global ids [offset_r, offset_r + rows_r) of the row-contiguous partition.
extern "C" int cozo_gpu_hnsw_stage_sharded(cozo_gpu_shards_t* s, cozo_gpu_hnsw_t* local_shard,
                                           uint64_t* out_global_offset, uint64_t* out_total_rows) {
  if (!s || !local_shard) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(s->mu);
  // every rank's (rows, dtype): [world][2] after the all-gather, this rank's pair at the end
  const uint64_t mine[2] = {local_shard->dev.n, local_shard->f64 ? 1ull : 0ull};
  uint64_t* d_tmp = nullptr;
  COZO_CUDA(cudaMalloc(&d_tmp, 16 * ((size_t)s->world + 1)));
  COZO_CUDA(cudaMemcpyAsync(d_tmp + 2 * s->world, mine, 16, cudaMemcpyHostToDevice, s->stream));
  if (s->world > 1)
    COZO_NCCL(g_nccl.AllGather(d_tmp + 2 * s->world, d_tmp, 2, ncclUint64, s->comm, s->stream));
  else
    COZO_CUDA(cudaMemcpyAsync(d_tmp, d_tmp + 2, 16, cudaMemcpyDeviceToDevice, s->stream));
  std::vector<uint64_t> all(2 * (size_t)s->world);
  COZO_CUDA(cudaMemcpyAsync(all.data(), d_tmp, (size_t)s->world * 16, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  cudaFree(d_tmp);
  s->offsets.assign(s->world, 0);
  uint64_t acc = 0;
  s->dtype = (int)all[1];
  for (int r = 0; r < s->world; ++r) {
    s->offsets[r] = acc;
    acc += all[2 * r];
    if ((int)all[2 * r + 1] != s->dtype) s->dtype = -1;
  }
  s->total_rows = acc;
  COZO_CUDA(cudaMemcpy(s->d_offsets, s->offsets.data(), (size_t)s->world * 8, cudaMemcpyHostToDevice));
  s->shard = local_shard;
  if (out_global_offset) *out_global_offset = s->offsets[s->rank];
  if (out_total_rows) *out_total_rows = acc;
  return 0;
}

extern "C" int cozo_gpu_shards_info(cozo_gpu_shards_t* s, int* rank, int* world, int* exchange, uint64_t* total_rows) {
  if (!s) return set_error(COZO_GPU_EINVAL, "null argument");
  if (rank) *rank = s->rank;
  if (world) *world = s->world;
  if (exchange) *exchange = s->exchange;
  if (total_rows) *total_rows = s->total_rows;
  return 0;
}

static int sharded_dev_entry(cozo_gpu_shards_t* s, const float* queries_dev, uint32_t B, uint32_t k, uint32_t ef,
                             double radius, bool filtered, const uint32_t* row_mask_dev, uint64_t* out_ids_dev,
                             float* out_dist_dev, uint32_t* per_query_stats_dev, void* stream) {
  int rc = check_group(s, k, ef, 0);
  if (rc) return rc;
  if (filtered && s->shard->dev.n && !row_mask_dev) return set_error(COZO_GPU_EINVAL, "null row mask");
  if (B && (!queries_dev || !out_ids_dev || !out_dist_dev)) return set_error(COZO_GPU_EINVAL, "null buffer");
  rc = ensure_init();
  if (rc) return rc;
  if (B == 0) return 0;
  std::lock_guard<std::mutex> lk(s->mu);
  // order the communicator's stream after the caller's stream and back
  cudaEvent_t e;
  COZO_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  COZO_CUDA(cudaEventRecord(e, (cudaStream_t)stream));
  COZO_CUDA(cudaStreamWaitEvent(s->stream, e, 0));
  rc = sharded_search_dev<float>(s, queries_dev, B, k, ef, radius, filtered ? row_mask_dev : nullptr, out_ids_dev,
                                 out_dist_dev, per_query_stats_dev);
  if (!rc) {
    COZO_CUDA(cudaEventRecord(e, s->stream));
    COZO_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, e, 0));
  }
  cudaEventDestroy(e);
  return rc;
}

// The host-pointer forms: T = float (F32 group) or double (F64 group); row_mask = this rank's filter verdicts, host
// memory, nullptr = no filter.
template <typename T>
static int sharded_host_entry(cozo_gpu_shards_t* s, const T* queries, uint32_t B, uint32_t k, uint32_t ef,
                              double radius, int root, bool filtered, const uint32_t* row_mask, uint64_t* out_ids,
                              T* out_dist, uint32_t* out_count, CozoGpuSearchStats* stats) {
  constexpr bool f64 = std::is_same<T, double>::value;
  int rc = check_group(s, k, ef, f64 ? 1 : 0);
  if (rc) return rc;
  if (root >= s->world) return set_error(COZO_GPU_EINVAL, "root %d out of range", root);
  if (filtered && s->shard->dev.n && !row_mask) return set_error(COZO_GPU_EINVAL, "null row mask");
  const bool have_q = root < 0 || root == s->rank;
  if (B && have_q && !queries) return set_error(COZO_GPU_EINVAL, "null query buffer");
  if (B && ((out_ids == nullptr) != (out_dist == nullptr))) return set_error(COZO_GPU_EINVAL, "ids/dist must come together");
  rc = ensure_init();
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return 0;
  std::lock_guard<std::mutex> lk(s->mu);
  cozo_gpu_hnsw* h = s->shard;
  const size_t qf = (size_t)B * h->dev.dim;
  if (s->q_bytes < qf * sizeof(T)) {
    if (s->d_q) cudaFree(s->d_q);
    s->d_q = nullptr;
    s->q_bytes = 0;
    COZO_CUDA(cudaMalloc(&s->d_q, qf * sizeof(T)));
    s->q_bytes = qf * sizeof(T);
  }
  if (s->out_rows < B || s->out_k < k) {
    for (void* p : {(void*)s->d_out_ids, s->d_out_dist, (void*)s->d_qstats})
      if (p) cudaFree(p);
    s->d_out_ids = nullptr;
    s->d_out_dist = nullptr;
    s->d_qstats = nullptr;
    const size_t rows = std::max<size_t>(B, s->out_rows), kk = std::max<size_t>(k, s->out_k);
    s->out_rows = s->out_k = 0;
    COZO_CUDA(cudaMalloc(&s->d_out_ids, rows * kk * 8));
    COZO_CUDA(cudaMalloc(&s->d_out_dist, rows * kk * 8));
    COZO_CUDA(cudaMalloc(&s->d_qstats, rows * 16));
    s->out_rows = rows;
    s->out_k = kk;
  }
  cudaStream_t st = s->stream;
  const uint32_t* d_mask = nullptr;
  if (row_mask) {
    const size_t words = ((size_t)h->dev.n + 31) / 32;
    if (s->mask_words < words || !s->d_mask) {
      if (s->d_mask) cudaFree(s->d_mask);
      s->d_mask = nullptr;
      s->mask_words = 0;
      COZO_CUDA(cudaMalloc(&s->d_mask, std::max<size_t>(words, 1) * 4));
      s->mask_words = words;
    }
    COZO_CUDA(cudaMemcpyAsync(s->d_mask, row_mask, words * 4, cudaMemcpyHostToDevice, st));
    d_mask = s->d_mask;
  }
  // an F64 shard is searched with a workspace held for the whole call
  struct Ws {
    cozo_gpu_hnsw* h;
    HnswWorkspace* ws;
    cudaStream_t st;
    ~Ws() {
      if (ws) {
        cudaStreamSynchronize(st);
        hnsw_release_ws(h, ws);
      }
    }
  } ws64{h, nullptr, st};
  if (f64) {
    ws64.ws = hnsw_acquire_ws(h);
    if (!ws64.ws) return COZO_GPU_ECUDA;
  }
  cudaEvent_t e0, e1;
  COZO_CUDA(cudaEventCreate(&e0));
  COZO_CUDA(cudaEventCreate(&e1));
  T* d_q = static_cast<T*>(s->d_q);
  T* d_out_dist = static_cast<T*>(s->d_out_dist);
  if (have_q) COZO_CUDA(cudaMemcpyAsync(d_q, queries, qf * sizeof(T), cudaMemcpyHostToDevice, st));
  if (root >= 0 && s->world > 1)
    COZO_NCCL(g_nccl.Broadcast(d_q, d_q, qf, f64 ? ncclFloat64 : ncclFloat32, root, s->comm, st));
  COZO_CUDA(cudaEventRecord(e0, st));
  rc = sharded_search_dev<T>(s, d_q, B, k, ef, radius, d_mask, s->d_out_ids, d_out_dist, s->d_qstats, ws64.ws);
  if (rc) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return rc;
  }
  COZO_CUDA(cudaEventRecord(e1, st));
  if (out_ids) {
    COZO_CUDA(cudaMemcpyAsync(out_ids, s->d_out_ids, (size_t)B * k * 8, cudaMemcpyDeviceToHost, st));
    COZO_CUDA(cudaMemcpyAsync(out_dist, d_out_dist, (size_t)B * k * sizeof(T), cudaMemcpyDeviceToHost, st));
  }
  std::vector<uint32_t> qs;
  if (stats) {
    qs.resize((size_t)B * 4);
    COZO_CUDA(cudaMemcpyAsync(qs.data(), s->d_qstats, (size_t)B * 16, cudaMemcpyDeviceToHost, st));
  }
  COZO_CUDA(cudaStreamSynchronize(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  rc = check_timeout(s);
  if (rc) return rc;
  if (out_count && out_ids)
    for (uint32_t i = 0; i < B; ++i) {
      uint32_t c = 0;
      while (c < k && out_ids[(size_t)i * k + c] != ~0ull) ++c;
      out_count[i] = c;
    }
  if (stats) {
    stats->n_queries = B;
    stats->kernel_ms = ms;
    for (uint32_t i = 0; i < B; ++i) {
      stats->dist_evals += qs[(size_t)i * 4 + 0];
      stats->nodes_expanded += qs[(size_t)i * 4 + 1];
      stats->nbr_reads += qs[(size_t)i * 4 + 2];
    }
  }
  return 0;
}

extern "C" int cozo_gpu_hnsw_search_sharded_dev(cozo_gpu_shards_t* s, const float* queries_dev, uint32_t B, uint32_t k,
                                                uint32_t ef, double radius, uint64_t* out_ids_dev, float* out_dist_dev,
                                                uint32_t* per_query_stats_dev, void* stream) {
  return sharded_dev_entry(s, queries_dev, B, k, ef, radius, false, nullptr, out_ids_dev, out_dist_dev,
                           per_query_stats_dev, stream);
}

extern "C" int cozo_gpu_hnsw_search_sharded_filtered_dev(cozo_gpu_shards_t* s, const float* queries_dev, uint32_t B,
                                                         uint32_t k, uint32_t ef, double radius,
                                                         const uint32_t* row_mask_dev, uint64_t* out_ids_dev,
                                                         float* out_dist_dev, uint32_t* per_query_stats_dev,
                                                         void* stream) {
  return sharded_dev_entry(s, queries_dev, B, k, ef, radius, true, row_mask_dev, out_ids_dev, out_dist_dev,
                           per_query_stats_dev, stream);
}

extern "C" int cozo_gpu_hnsw_search_sharded(cozo_gpu_shards_t* s, const float* queries, uint32_t B, uint32_t k,
                                            uint32_t ef, double radius, int root, uint64_t* out_ids, float* out_dist,
                                            uint32_t* out_count, CozoGpuSearchStats* stats) {
  return sharded_host_entry<float>(s, queries, B, k, ef, radius, root, false, nullptr, out_ids, out_dist, out_count,
                                   stats);
}

extern "C" int cozo_gpu_hnsw_search_sharded_filtered(cozo_gpu_shards_t* s, const float* queries, uint32_t B,
                                                     uint32_t k, uint32_t ef, double radius, int root,
                                                     const uint32_t* row_mask, uint64_t* out_ids, float* out_dist,
                                                     uint32_t* out_count, CozoGpuSearchStats* stats) {
  return sharded_host_entry<float>(s, queries, B, k, ef, radius, root, true, row_mask, out_ids, out_dist, out_count,
                                   stats);
}

extern "C" int cozo_gpu_hnsw_search_sharded_f64(cozo_gpu_shards_t* s, const double* queries, uint32_t B, uint32_t k,
                                                uint32_t ef, double radius, int root, const uint32_t* row_mask,
                                                uint64_t* out_ids, double* out_dist, uint32_t* out_count,
                                                CozoGpuSearchStats* stats) {
  return sharded_host_entry<double>(s, queries, B, k, ef, radius, root, false, row_mask, out_ids, out_dist, out_count,
                                    stats);
}

// ---- source-sharded graph calls: the graph is replicated, the sources are split ---------------------------------
// SURVEY.md §8e "replicate graph, partition sources; no exchange until the end".  Every rank stages the same graph and
// attaches it; the sources of a call are split into `world` contiguous slices in source order, rank r searches slice r
// with the single-GPU code (graph.cu: closeness_run, betweenness_run, sssp_goals_run) and the slices are exchanged
// once at the end, so every rank returns the whole answer.
// Every call, attach included, starts its collectives with one all-gather of a fixed-size status record: this rank's
// outcome (argument checks, poison, out of memory, ...) and the call's signature (which call, which graph, and every
// argument that sizes a later collective).  All ranks then take the same branch: when the signatures differ — the
// ranks made different calls, e.g. two rules run concurrently in different orders — every rank returns EINVAL, and
// when a rank failed every rank returns that rank's code, so no rank meets a peer in a collective of another size or
// waits for one that never comes.  Buffers a call needs are allocated before its status all-gather; the one whose size
// is known only after it (the rows of sssp_goals) reports its allocation in the next all-gather.
namespace cozo {

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {  // the splitmix64 finaliser
  x ^= x >> 30;
  x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27;
  x *= 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// order-free checksum of one array of 32-bit words: the sum of mix64(position, salt, word) (wrapping), so the same
// bits give the same value whatever the launch geometry or the order of the atomics
__global__ void graph_checksum_kernel(const uint32_t* a, uint64_t count, uint64_t salt, unsigned long long* out) {
  unsigned long long acc = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
    acc += mix64(mix64(i * 4 + salt) ^ a[i]);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// betweenness: the ranks' f64 partial sums [world][n] added in rank order, rounded to f32 once
__global__ void bc_rank_sum_kernel(const double* parts, uint32_t n, uint32_t world, float* out) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  double acc = parts[v];
  for (uint32_t r = 1; r < world; ++r) acc += parts[(size_t)r * n + v];
  out[v] = (float)acc;
}

// slice r of `total` sources: [total * r / world, total * (r + 1) / world); no slice is longer than ceil(total / world)
static void source_slice(uint32_t total, int world, int r, uint32_t& lo, uint32_t& hi) {
  lo = (uint32_t)((uint64_t)total * (uint64_t)r / (uint64_t)world);
  hi = (uint32_t)((uint64_t)total * (uint64_t)(r + 1) / (uint64_t)world);
}

// all-gather of `count` elements per rank on the group's stream; in place when send == recv + rank * count
static int group_all_gather(cozo_gpu_shards* s, const void* send, void* recv, size_t count, ncclDataType_t t,
                            size_t elem) {
  if (s->world > 1)
    COZO_NCCL(g_nccl.AllGather(send, recv, count, t, s->comm, s->stream));
  else if (send != recv)
    COZO_CUDA(cudaMemcpyAsync(recv, send, count * elem, cudaMemcpyDeviceToDevice, s->stream));
  return 0;
}

enum GraphCall : uint64_t { CALL_ATTACH = 1, CALL_CLOSENESS, CALL_BETWEENNESS, CALL_SSSP_GOALS };
constexpr int kSigWords = 12;
static const char* const kCallNames[] = {"no call", "attach", "closeness", "betweenness", "sssp_goals"};
static const char* const kSigNames[kSigWords] = {"the call",        "n",           "m",         "weighted",
                                                 "graph checksum",  "n_src",       "n_goals",   "keep_ties",
                                                 "row capacity",    "the sources and goals", "", ""};

// one rank's status record: its outcome, then the call's signature
struct CallRecord {
  int64_t rc = 0, cyclic = 0, rows = 0, pad = 0;  // return code, zero-weight-cycle flag, rows of its slice
  // call kind, n, m, weighted, graph checksum, n_src, n_goals, keep_ties, cap, hash of sources and goals, 0, 0
  uint64_t sig[kSigWords] = {};
};
static_assert(sizeof(CallRecord) == 128, "one 128-byte record per rank (cozo_gpu_shards::d_status)");

// the signature of a call on the attached graph (all zero but the kind when none is attached)
static CallRecord graph_record(const cozo_gpu_shards* s, uint64_t kind) {
  CallRecord r;
  r.sig[0] = kind;
  if (s->graph) {
    r.sig[1] = s->graph->n;
    r.sig[2] = s->graph->m;
    r.sig[3] = s->graph->weighted ? 1 : 0;
    r.sig[4] = s->graph_sum;
  }
  return r;
}

static uint64_t fnv1a(uint64_t h, const void* p, size_t bytes) {
  const uint8_t* b = static_cast<const uint8_t*>(p);
  for (size_t i = 0; i < bytes; ++i) h = (h ^ b[i]) * 0x100000001B3ull;
  return h;
}

// The one status all-gather of a sharded graph call.  Returns 0 when every rank succeeded with the same signature;
// otherwise, on every rank, EINVAL when the signatures differ, else the code of the first failing rank in rank order.
static int exchange_status(cozo_gpu_shards* s, const CallRecord& mine, std::vector<CallRecord>& all) {
  CallRecord* d = reinterpret_cast<CallRecord*>(s->d_status);
  COZO_CUDA(cudaMemcpyAsync(d + s->rank, &mine, sizeof(CallRecord), cudaMemcpyHostToDevice, s->stream));
  int rc = group_all_gather(s, d + s->rank, d, sizeof(CallRecord), ncclUint8, 1);
  if (rc) return rc;
  all.resize(s->world);
  COZO_CUDA(cudaMemcpyAsync(all.data(), d, sizeof(CallRecord) * (size_t)s->world, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  for (int r = 1; r < s->world; ++r)
    for (int k = 0; k < kSigWords; ++k)
      if (all[r].sig[k] != all[0].sig[k])
        return set_error(COZO_GPU_EINVAL,
                         "the ranks of the shard group made different calls (rank 0: %s, rank %d: %s; they differ in %s): "
                         "every rank must make the same call with the same arguments on the same graph",
                         kCallNames[std::min<uint64_t>(all[0].sig[0], 4)], r,
                         kCallNames[std::min<uint64_t>(all[r].sig[0], 4)], kSigNames[k]);
  for (int r = 0; r < s->world; ++r) {
    if (!all[r].rc) continue;
    if (r != s->rank)  // the failing rank keeps its own message
      set_error((int)all[r].rc, "rank %d of the shard group failed (code %d); the sharded call stops on every rank", r,
                (int)all[r].rc);
    return (int)all[r].rc;
  }
  return 0;
}

static int check_graph_group(const cozo_gpu_shards* s) {
  if (!s->graph) return set_error(COZO_GPU_EINVAL, "no graph attached to the shard group (cozo_gpu_graph_attach_sharded)");
  return 0;
}

// a rank with an empty slice runs no source chunk; it still answers its poison flag
static int poll_poison(const volatile int* poison) {
  return poisoned(poison) ? set_error(COZO_GPU_EKILLED, "Running query is killed before completion") : 0;
}

}  // namespace cozo

extern "C" int cozo_gpu_graph_attach_sharded(cozo_gpu_shards_t* s, cozo_gpu_graph_t* g) {
  if (!s) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(s->mu);
  s->graph = nullptr;
  s->graph_sum = 0;
  CallRecord rec;
  rec.sig[0] = CALL_ATTACH;
  auto local = [&]() -> int {
    if (!g) return set_error(COZO_GPU_EINVAL, "null graph handle");
    cudaStream_t st = s->stream;
    // checksum of out_ptr, out_idx and the bits of out_w, accumulated in the scratch record
    auto* sum = reinterpret_cast<unsigned long long*>(s->d_status + 128 * (size_t)s->world);
    COZO_CUDA(cudaMemsetAsync(sum, 0, 8, st));
    const struct {
      const uint32_t* a;
      uint64_t count;
    } parts[3] = {{g->out_ptr, (uint64_t)g->n + 1},
                  {g->out_idx, g->m},
                  {reinterpret_cast<const uint32_t*>(g->out_w), g->weighted ? g->m : 0}};
    for (int i = 0; i < 3; ++i) {
      if (!parts[i].a || !parts[i].count) continue;
      const uint32_t blocks = (uint32_t)std::min<uint64_t>((parts[i].count + 255) / 256, 1024);
      graph_checksum_kernel<<<blocks, 256, 0, st>>>(parts[i].a, parts[i].count, (uint64_t)i << 62, sum);
    }
    COZO_CUDA(cudaGetLastError());
    unsigned long long h = 0;
    COZO_CUDA(cudaMemcpyAsync(&h, sum, 8, cudaMemcpyDeviceToHost, st));
    COZO_CUDA(cudaStreamSynchronize(st));
    rec.sig[1] = g->n;
    rec.sig[2] = g->m;
    rec.sig[3] = g->weighted ? 1 : 0;
    rec.sig[4] = h;
    return 0;
  };
  rec.rc = local();
  std::vector<CallRecord> all;
  rc = exchange_status(s, rec, all);  // graphs that differ: EINVAL on every rank, and the group keeps no graph
  if (rc) return rc;
  s->graph = g;
  s->graph_sum = rec.sig[4];
  return 0;
}

extern "C" int cozo_gpu_closeness_sharded(cozo_gpu_shards_t* s, float* out, double* out_kernel_ms,
                                          const volatile int* poison) {
  if (!s) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  std::lock_guard<std::mutex> lk(s->mu);
  CallRecord rec = graph_record(s, CALL_CLOSENESS);
  cozo_gpu_graph* g = s->graph;
  const uint32_t n = g ? g->n : 0;
  const uint32_t W = (uint32_t)s->world, cmax = (n + W - 1) / W;
  uint32_t lo, hi;
  source_slice(n, s->world, s->rank, lo, hi);
  CallStream cs;
  DevBuf dall;  // [world][cmax]: slice r at row r
  auto local = [&]() -> int {
    if (!out) return set_error(COZO_GPU_EINVAL, "null argument");
    int e = check_graph_group(s);
    if (e || n == 0) return e;  // n == 0: all_pairs_shortest_path.rs:111-113
    COZO_CUDA(cudaMalloc(&dall.p, (size_t)W * cmax * 4));
    e = cs.init();
    if (e) return e;
    if (hi == lo) return poll_poison(poison);
    return closeness_run(g, cs, lo, hi, dall.as<float>() + (size_t)s->rank * cmax, poison);
  };
  rec.rc = local();
  const double ms = cs.e1 ? cs.stop() : 0.0;
  if (out_kernel_ms) *out_kernel_ms = ms;
  std::vector<CallRecord> all;
  rc = exchange_status(s, rec, all);
  if (rc || n == 0) return rc;
  rc = group_all_gather(s, dall.as<float>() + (size_t)s->rank * cmax, dall.p, cmax, ncclFloat32, 4);
  if (rc) return rc;
  std::vector<float> h((size_t)W * cmax);
  COZO_CUDA(cudaMemcpyAsync(h.data(), dall.p, h.size() * 4, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  for (int r = 0; r < s->world; ++r) {
    uint32_t a, b;
    source_slice(n, s->world, r, a, b);
    std::copy(h.begin() + (size_t)r * cmax, h.begin() + (size_t)r * cmax + (b - a), out + a);
  }
  return 0;
}

extern "C" int cozo_gpu_betweenness_sharded(cozo_gpu_shards_t* s, float* out, double* out_kernel_ms,
                                            const volatile int* poison) {
  if (!s) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  std::lock_guard<std::mutex> lk(s->mu);
  CallRecord rec = graph_record(s, CALL_BETWEENNESS);
  cozo_gpu_graph* g = s->graph;
  const uint32_t n = g ? g->n : 0;
  uint32_t lo, hi;
  source_slice(n, s->world, s->rank, lo, hi);
  CallStream cs;
  DevBuf dall, dcyc, dout;  // dall: [world][n] f64 partial sums, this rank's at row `rank`
  double* mine = nullptr;
  int hcyc = 0;
  auto local = [&]() -> int {
    if (!out) return set_error(COZO_GPU_EINVAL, "null argument");
    int e = check_graph_group(s);
    if (e || n == 0) return e;  // n == 0: all_pairs_shortest_path.rs:43-46
    COZO_CUDA(cudaMalloc(&dall.p, (size_t)s->world * n * 8));
    COZO_CUDA(cudaMalloc(&dcyc.p, 4));
    COZO_CUDA(cudaMalloc(&dout.p, (size_t)n * 4));
    e = cs.init();
    if (e) return e;
    mine = dall.as<double>() + (size_t)s->rank * n;
    COZO_CUDA(cudaMemsetAsync(mine, 0, (size_t)n * 8, cs.s));
    COZO_CUDA(cudaMemsetAsync(dcyc.p, 0, 4, cs.s));
    e = hi > lo ? betweenness_run(g, cs, lo, hi, mine, dcyc.as<int>(), poison) : poll_poison(poison);
    if (e) return e;
    COZO_CUDA(cudaMemcpyAsync(&hcyc, dcyc.p, 4, cudaMemcpyDeviceToHost, cs.s));
    COZO_CUDA(cudaStreamSynchronize(cs.s));
    return 0;
  };
  rec.rc = local();
  rec.cyclic = hcyc;
  const double ms = cs.e1 ? cs.stop() : 0.0;
  if (out_kernel_ms) *out_kernel_ms = ms;
  std::vector<CallRecord> all;
  rc = exchange_status(s, rec, all);
  if (rc || n == 0) return rc;
  for (const CallRecord& x : all)
    if (x.cyclic)
      return set_error(COZO_GPU_EUNSUP, "betweenness: a zero-weight cycle makes the set of tied shortest paths unbounded "
                                        "(the reference does not terminate on this input)");
  rc = group_all_gather(s, mine, dall.p, n, ncclFloat64, 8);
  if (rc) return rc;
  bc_rank_sum_kernel<<<(n + 255) / 256, 256, 0, s->stream>>>(dall.as<double>(), n, (uint32_t)s->world, dout.as<float>());
  COZO_CUDA(cudaGetLastError());
  COZO_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  return 0;
}

extern "C" int cozo_gpu_sssp_goals_sharded(cozo_gpu_shards_t* s, const uint32_t* sources, uint32_t n_src,
                                           const uint32_t* goals, uint32_t n_goals, int32_t keep_ties, float* out_cost,
                                           uint64_t* out_path_off, uint32_t* out_paths, uint64_t paths_cap,
                                           uint64_t* out_tie_off, uint32_t* out_tie_edges, uint64_t ties_cap,
                                           double* out_kernel_ms, const volatile int* poison) {
  const uint64_t pairs = (uint64_t)n_src * n_goals;
  uint64_t* off_out = keep_ties ? out_tie_off : out_path_off;
  uint32_t* rows_out = keep_ties ? out_tie_edges : out_paths;
  const uint64_t cap = keep_ties ? ties_cap : paths_cap;
  if (!s) return set_error(COZO_GPU_EINVAL, "null argument");
  int rc = ensure_init();
  if (rc) return rc;
  if (out_kernel_ms) *out_kernel_ms = 0;
  std::lock_guard<std::mutex> lk(s->mu);
  cozo_gpu_graph* g = s->graph;
  CallRecord rec = graph_record(s, CALL_SSSP_GOALS);
  rec.sig[5] = n_src;
  rec.sig[6] = n_goals;
  rec.sig[7] = keep_ties ? 1 : 0;
  rec.sig[8] = cap;
  rec.sig[9] = 0xCBF29CE484222325ull;
  if (sources) rec.sig[9] = fnv1a(rec.sig[9], sources, (size_t)n_src * 4);
  if (goals) rec.sig[9] = fnv1a(rec.sig[9], goals, (size_t)n_goals * 4);
  const uint32_t W = (uint32_t)s->world, cmax = (n_src + W - 1) / W;
  uint32_t lo, hi;
  source_slice(n_src, s->world, s->rank, lo, hi);
  const uint64_t per_row = keep_ties ? 2 : 1;          // u32 per row
  const uint64_t per_src = keep_ties ? 1 : n_goals;    // offsets per source
  // one slot per rank: costs [cmax * n_goals]; offsets [cmax * per_src + 1], then one word = "my row buffer is ready"
  const uint64_t slot_off = (uint64_t)cmax * per_src + 2, slot_cost = (uint64_t)cmax * n_goals;
  std::vector<float> lcost(slot_cost);
  std::vector<uint64_t> loff(slot_off, 0);
  DevBuf dlocal, dcost, doff;  // this rank's rows; every slot's costs and offsets
  uint64_t local_cap = 0;      // rows dlocal holds
  CallStream cs;
  auto local = [&]() -> int {
    if ((n_src && !sources) || (n_goals && !goals) || (pairs && !out_cost) || !off_out || (cap && !rows_out))
      return set_error(COZO_GPU_EINVAL, "null argument");
    int e = check_graph_group(s);
    if (!e) e = sssp_goals_check(g, sources, n_src, goals, n_goals);
    if (e || pairs == 0) return e;
    COZO_CUDA(cudaMalloc(&dcost.p, W * slot_cost * 4));
    COZO_CUDA(cudaMalloc(&doff.p, W * slot_off * 8));
    e = cs.init();
    if (e) return e;
    if (hi == lo) return poll_poison(poison);
    return sssp_goals_run(
        g, cs, sources + lo, hi - lo, goals, n_goals, keep_ties != 0, lcost.data(), loff.data(), cap, poison,
        [&](const uint32_t* drows, uint64_t base, uint64_t total) -> int {
          if (local_cap < base + total) {
            DevBuf grown;
            const uint64_t want = std::max(base + total, 2 * local_cap);
            COZO_CUDA(cudaMalloc(&grown.p, want * per_row * 4));
            if (base) COZO_CUDA(cudaMemcpyAsync(grown.p, dlocal.p, base * per_row * 4, cudaMemcpyDeviceToDevice, cs.s));
            COZO_CUDA(cudaStreamSynchronize(cs.s));
            std::swap(grown.p, dlocal.p);
            local_cap = want;
          }
          COZO_CUDA(cudaMemcpyAsync(dlocal.as<uint32_t>() + base * per_row, drows, total * per_row * 4,
                                    cudaMemcpyDeviceToDevice, cs.s));
          return 0;
        });
  };
  rec.rc = local();
  rec.rows = (int64_t)(hi > lo ? loff[(uint64_t)(hi - lo) * per_src] : 0);
  const double ms = cs.e1 ? cs.stop() : 0.0;
  if (out_kernel_ms) *out_kernel_ms = ms;
  std::vector<CallRecord> all;
  rc = exchange_status(s, rec, all);
  if (rc) return rc;
  const uint64_t n_off = keep_ties ? (uint64_t)n_src + 1 : pairs + 1;
  std::fill(off_out, off_out + n_off, 0);
  if (pairs == 0) return 0;
  std::vector<uint64_t> base(W + 1, 0);  // first row of every rank's slice; base[W] = the total
  for (uint32_t r = 0; r < W; ++r) base[r + 1] = base[r] + (uint64_t)all[r].rows;
  const uint64_t total = base[W];
  const bool move_rows = total && total <= cap;  // as on one GPU: otherwise the caller retries with room for `total`
  // the row buffer is sized by the total; whether every rank could allocate it travels with the offsets
  DevBuf drows;
  loff[slot_off - 1] = 1;
  if (move_rows && cudaMalloc(&drows.p, total * per_row * 4) != cudaSuccess) {
    cudaGetLastError();
    loff[slot_off - 1] = 0;
  }
  // costs and offsets of every slice
  float* my_cost = dcost.as<float>() + s->rank * slot_cost;
  uint64_t* my_off = doff.as<uint64_t>() + s->rank * slot_off;
  COZO_CUDA(cudaMemcpyAsync(my_cost, lcost.data(), slot_cost * 4, cudaMemcpyHostToDevice, s->stream));
  COZO_CUDA(cudaMemcpyAsync(my_off, loff.data(), slot_off * 8, cudaMemcpyHostToDevice, s->stream));
  if (W > 1) COZO_NCCL(g_nccl.GroupStart());
  rc = group_all_gather(s, my_cost, dcost.p, slot_cost, ncclFloat32, 4);
  if (!rc) rc = group_all_gather(s, my_off, doff.p, slot_off, ncclUint64, 8);
  if (W > 1) COZO_NCCL(g_nccl.GroupEnd());
  if (rc) return rc;
  std::vector<float> hcost(W * slot_cost);
  std::vector<uint64_t> hoff(W * slot_off);
  COZO_CUDA(cudaMemcpyAsync(hcost.data(), dcost.p, hcost.size() * 4, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaMemcpyAsync(hoff.data(), doff.p, hoff.size() * 8, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  for (uint32_t r = 0; r < W; ++r)
    if (!hoff[r * slot_off + slot_off - 1])
      return set_error(COZO_GPU_ENOMEM, "sssp_goals_sharded: rank %u could not allocate the %llu-row exchange buffer", r,
                       (unsigned long long)total);
  for (uint32_t r = 0; r < W; ++r) {
    uint32_t a, b;
    source_slice(n_src, s->world, (int)r, a, b);
    std::copy(hcost.begin() + r * slot_cost, hcost.begin() + r * slot_cost + (uint64_t)(b - a) * n_goals,
              out_cost + (uint64_t)a * n_goals);
    const uint64_t* o = hoff.data() + r * slot_off;
    for (uint64_t i = 0; b > a && i <= (uint64_t)(b - a) * per_src; ++i) off_out[a * per_src + i] = o[i] + base[r];
  }
  off_out[n_off - 1] = total;
  if (!move_rows) return 0;
  // the rows: one broadcast per rank of its slice's rows, into place
  uint32_t* rows = drows.as<uint32_t>();
  if (W > 1) {
    COZO_NCCL(g_nccl.GroupStart());
    for (uint32_t r = 0; r < W; ++r) {
      const uint64_t cnt = base[r + 1] - base[r];
      if (!cnt) continue;
      uint32_t* dst = rows + base[r] * per_row;
      COZO_NCCL(g_nccl.Broadcast((int)r == s->rank ? dlocal.p : dst, dst, cnt * per_row, ncclUint32, (int)r, s->comm,
                                 s->stream));
    }
    COZO_NCCL(g_nccl.GroupEnd());
  } else {
    COZO_CUDA(cudaMemcpyAsync(rows, dlocal.p, total * per_row * 4, cudaMemcpyDeviceToDevice, s->stream));
  }
  COZO_CUDA(cudaMemcpyAsync(rows_out, rows, total * per_row * 4, cudaMemcpyDeviceToHost, s->stream));
  COZO_CUDA(cudaStreamSynchronize(s->stream));
  return 0;
}
