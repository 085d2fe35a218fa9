// hnsw_host.hpp — host-side state of a staged HNSW index (opaque cozo_gpu_hnsw_t).
#pragma once
#include <array>
#include <condition_variable>
#include <mutex>
#include <vector>

#include "hnsw_device.cuh"

struct HnswWorkspace {
  cudaStream_t stream = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  uint32_t* vis = nullptr;
  size_t vis_words = 0;  // total words allocated
  uint32_t* vlog = nullptr;
  size_t vlog_words = 0;
  uint32_t* counter = nullptr;
  // staging buffers of the host-pointer API
  float* q = nullptr;
  size_t q_floats = 0;
  uint32_t* ids = nullptr;
  float* dist = nullptr;
  uint32_t* count = nullptr;
  uint32_t* qstats = nullptr;
  size_t out_rows = 0, out_k = 0;
  uint32_t* mask = nullptr;  // row filter verdicts of the host-pointer call
  size_t mask_words = 0;
  // pinned mirrors
  float* h_q = nullptr;
  size_t h_q_floats = 0;
};

struct cozo_gpu_hnsw {
  cozo::HnswDev dev{};
  // owned device buffers
  float* d_vec = nullptr;
  bool vec_owned = true;
  // uint8 code rows of an L2 f32 index (hnsw_codes.cuh), one per row of d_vec, written wherever d_vec is;
  // dev.codes = nullptr when there are none (other metrics, F64, or an allocation that failed)
  uint8_t* d_codes = nullptr;
  uint32_t codes_rows = 0;     // allocated rows
  bool codes_failed = false;   // an allocation or a fill failed: the index stays without codes
  // F64 vector index (VecElementType::F64): payloads as doubles, searched by hnsw_f64.cu only
  double* d_vec64 = nullptr;
  uint32_t ld64 = 0;
  bool f64 = false;
  uint32_t* d_adj0 = nullptr;
  uint32_t* d_upper_off = nullptr;
  uint32_t* d_adj_up = nullptr;
  uint64_t up_rows = 0;
  // builder-only companions (distances of the stored edges, hnsw.rs:281-318 `dist`)
  float* d_adj0_dist = nullptr;
  float* d_adj_up_dist = nullptr;
  uint8_t* d_node_level = nullptr;
  uint32_t *d_deg0 = nullptr, *d_deg_up = nullptr;  // live out-degree of every row
  uint32_t* d_up_owner = nullptr;                   // node owning each upper-layer row
  uint8_t* d_dead = nullptr;                        // removed nodes (hnsw_remove)
  uint32_t cap_n = 0;                               // allocated rows (>= dev.n); 0 = staged, exact fit
  uint64_t cap_up = 0;
  bool build_state_ready = false;
  uint32_t ef_construction = 0;
  int keep_pruned = 0;
  int extend_candidates = 0;  // hnsw.rs:499-511: fidelity mode, one node per batch (hnsw_build.cu)
  uint64_t rng_state = 0x5EED0003ull;
  uint32_t n_live = 0;
  uint32_t borrowed_rows = 0;  // rows available in a borrowed vector buffer
  std::vector<uint8_t> live;
  // host copies
  std::vector<uint8_t> node_level;  // top layer index of each node (0 = layer 0 only)
  uint32_t n_levels = 1;
  uint32_t m_max0 = 0, m_max = 0;
  std::mutex mu;
  std::condition_variable cv;
  std::vector<HnswWorkspace*> pool;
  uint32_t n_workspaces = 0;  // created so far (bounded by the "hnsw.max_workspaces" option)
};

namespace cozo {
// One per-row device array of a handle: `row_bytes` per node row [0, n), or per upper-layer row [0, up_rows) when
// `upper`.  Rows from there up to the capacity are unused and hold `fill` bytes, the state append_nodes expects.
struct RowArray {
  void*& ptr;
  size_t row_bytes;
  bool upper;
  uint8_t fill;
};

// Every row array of an f32 handle.  Two of them keep rules of their own: vec may be borrowed from the caller
// (vec_owned = false) and is then never written, grown or freed; codes is optional (nullptr when the index has no code
// rows) and is grown by hnsw_codes_reserve, which drops it rather than failing.  vec64 is not listed: every
// maintenance call refuses F64 handles.
constexpr size_t kVecArray = 0, kCodesArray = 1;
inline std::array<RowArray, 12> row_arrays(cozo_gpu_hnsw* h) {
  const HnswDev& g = h->dev;
  const size_t vec = (size_t)g.ld * 4, adj0 = (size_t)g.s0 * 4, up = (size_t)g.su * 4;
  auto ref = [](auto*& p) -> void*& { return reinterpret_cast<void*&>(p); };
  return {{{ref(h->d_vec), vec, false, 0},
           {ref(h->d_codes), g.code_ld, false, 0},
           {ref(h->d_adj0), adj0, false, 0xFF},
           {ref(h->d_adj0_dist), adj0, false, 0},
           {ref(h->d_deg0), 4, false, 0},
           {ref(h->d_upper_off), 4, false, 0xFF},
           {ref(h->d_node_level), 1, false, 0},
           {ref(h->d_dead), 1, false, 0},
           {ref(h->d_adj_up), up, true, 0xFF},
           {ref(h->d_adj_up_dist), up, true, 0},
           {ref(h->d_deg_up), 4, true, 0},
           {ref(h->d_up_owner), 4, true, 0xFF}}};
}

// destinations of the fused exchange: the [n_slots][B][k] gather buffers of every rank, this rank's lists at `slot`
template <typename D>
struct ScatterDestT {
  uint32_t n_dest, slot;
  uint32_t* ids[COZO_GPU_MAX_PEERS];
  D* dist[COZO_GPU_MAX_PEERS];
};
using ScatterDest = ScatterDestT<float>;
using ScatterDest64 = ScatterDestT<double>;
int hnsw_launch_search(cozo_gpu_hnsw* h, HnswWorkspace* ws, const float* d_q, uint32_t B, uint32_t k, uint32_t ef,
                       double radius, uint32_t* d_ids, float* d_dist, uint32_t* d_count, uint32_t* d_qstats,
                       cudaStream_t stream, const ScatterDest* scatter, const uint32_t* d_filter_mask = nullptr);
// the asynchronous f32 search of cozo_gpu_hnsw_search_dev / _filtered_dev / _scatter_dev: checks the arguments, takes
// a workspace and hands it back after the kernel, in stream order
int hnsw_search_dev(cozo_gpu_hnsw* h, const float* d_q, uint32_t B, uint32_t k, uint32_t ef, double radius,
                    uint32_t* d_ids, float* d_dist, uint32_t* d_count, uint32_t* d_qstats, void* stream,
                    const ScatterDest* scatter, const uint32_t* d_filter_mask);
// the F64 search kernel on device buffers, on `stream`, with `ws` held by the caller until the kernel ends.  d_ids /
// d_dist [B*k] are always written, also when `scatter` is given; d_count, d_qstats, scatter and d_filter_mask nullable.
int hnsw_launch_search_f64(cozo_gpu_hnsw* h, HnswWorkspace* ws, const double* d_q, uint32_t B, uint32_t k, uint32_t ef,
                           double radius, uint32_t* d_ids, double* d_dist, uint32_t* d_count, uint32_t* d_qstats,
                           cudaStream_t stream, const ScatterDest64* scatter, const uint32_t* d_filter_mask);
// merge.cu: cozo_gpu_topk_merge_dev on F64 distances
int topk_merge_f64_dev(const double* dist_dev, const uint32_t* ids_dev, uint32_t n_shards, uint32_t B, uint32_t k,
                       const uint64_t* shard_offsets_dev, uint64_t* out_ids_dev, double* out_dist_dev, void* stream);
HnswWorkspace* hnsw_acquire_ws(cozo_gpu_hnsw* h);
void hnsw_release_ws(cozo_gpu_hnsw* h, HnswWorkspace* ws);
int hnsw_ws_reserve(HnswWorkspace* ws, size_t vis_words, size_t vlog_words, cudaStream_t stream);
int hnsw_ensure_build_state(cozo_gpu_hnsw* h);
void hnsw_codes_reserve(cozo_gpu_hnsw* h, uint32_t rows);
void hnsw_codes_fill(cozo_gpu_hnsw* h, uint32_t first, uint32_t count, const uint32_t* d_ids = nullptr);
}  // namespace cozo
