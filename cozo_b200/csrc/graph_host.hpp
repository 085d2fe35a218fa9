// graph_host.hpp — host-side state of a staged graph (opaque cozo_gpu_graph_t).
#pragma once
#include <functional>
#include <mutex>

#include "common.cuh"

namespace cozo {
struct PrState;  // PageRank's own layouts (pagerank.cu), built lazily by the first cozo_gpu_pagerank call
void pr_state_free(PrState* p);

// scoped device buffer
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  template <class T>
  T* as() {
    return static_cast<T*>(p);
  }
};

inline bool poisoned(const volatile int* p) { return p && *p != 0; }

// every call owns a stream: FixedRule::run is invoked concurrently from Rayon workers (query/eval.rs:199-202)
// and independent calls must not serialise on the legacy default stream
struct CallStream {
  cudaStream_t s = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  int init() {
    COZO_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    COZO_CUDA(cudaEventCreate(&e0));
    COZO_CUDA(cudaEventCreate(&e1));
    COZO_CUDA(cudaEventRecord(e0, s));
    return 0;
  }
  double stop() {
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
  }
  ~CallStream() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (s) cudaStreamDestroy(s);
  }
};
}  // namespace cozo

struct cozo_gpu_graph {
  uint32_t n = 0;
  uint64_t m = 0;
  bool weighted = false;
  // CSR exactly as GraphBuilder::csr_layout(Sorted) lays it out (fixed_rule/mod.rs:192-195, 318-321)
  uint32_t *out_ptr = nullptr, *out_idx = nullptr, *in_ptr = nullptr, *in_idx = nullptr;
  float* out_w = nullptr;
  std::mutex pr_mu;
  cozo::PrState* pr = nullptr;
  // graphs staged from node keys (cozo_gpu_graph_stage_keys): the n distinct keys sorted by (length, bytes) for
  // lookups — bytes key_bytes[key_off[i] .. key_off[i+1]) with dense id key_id[i] — and, per dense id, the endpoint
  // index where its key first appeared.  All null for a graph staged from dense ids (keyed = false) and for n = 0.
  bool keyed = false;
  uint8_t* key_bytes = nullptr;
  uint64_t* key_off = nullptr;
  uint32_t *key_id = nullptr, *node_first = nullptr;
};

namespace cozo {
// the dense path of both staging calls: device edge arrays (m = g->m entries, ids < g->n, weights nullable) -> the
// CSR on `g`, in `st`.  Validates ids and weights; returns 0 or a COZO_GPU_E* code with the message set.  The caller
// frees `g` on failure.
int graph_build_csr(cozo_gpu_graph_t* g, const uint32_t* dsrc, const uint32_t* ddst, const float* dw, cudaStream_t st);

// The source-parallel bodies of the all-source and many-source calls, over any slice of their sources, so that the
// single-GPU entry points (the whole range) and the sharded ones (graph replicated, sources split over the ranks,
// sharded.cu) run the same code.  All run on cs.s, poll `poison` between source chunks and return 0 or a
// COZO_GPU_E* code with the message set.
// closeness of the sources [lo, hi) into dout[0 .. hi - lo) (device memory)
int closeness_run(cozo_gpu_graph_t* g, CallStream& cs, uint32_t lo, uint32_t hi, float* dout,
                  const volatile int* poison);
// the dependencies of the sources [lo, hi) added to dbc[n] (device f64) one source after the other, in source order;
// *dcyc (device) is set when a zero-weight cycle of tied paths is met
int betweenness_run(cozo_gpu_graph_t* g, CallStream& cs, uint32_t lo, uint32_t hi, double* dbc, int* dcyc,
                    const volatile int* poison);
// cozo_gpu_sssp_goals' argument checks on sources and goals
int sssp_goals_check(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                     uint32_t n_goals);
// rows of one source chunk, on the device: rows [base, base + total) of the call's row list, each one path node (one
// u32) or one (v, p) tie edge (two u32), ordered on cs.s
using GoalRowSink = std::function<int(const uint32_t* drows, uint64_t base, uint64_t total)>;
// cozo_gpu_sssp_goals for the given sources (host memory, checked): costs into out_cost (host), offsets into off_out
// (host, n_src * n_goals + 1 or, with keep_ties, n_src + 1 entries, starting at 0).  The rows of every chunk go to
// `sink` while the rows so far fit `cap`; after the first chunk that does not fit, only costs and offsets follow.
int sssp_goals_run(cozo_gpu_graph_t* g, CallStream& cs, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                   uint32_t n_goals, bool keep_ties, float* out_cost, uint64_t* off_out, uint64_t cap,
                   const volatile int* poison, const GoalRowSink& sink);
}  // namespace cozo
