// fixed_rule.hpp — the FixedRule plugin boundary (fixed_rule/mod.rs:538-567) and the
// four graph rules of the hot path implemented over the C ABI of libcozo_gpu.so.
//
// Same names, argument meaning and error behaviour as the reference:
//   trait FixedRule { init_options, arity, run }            fixed_rule/mod.rs:538-567
//   FixedRulePayload option getters                          fixed_rule/mod.rs:331-535
//   FixedRuleInputRelation::{iter, as_directed_graph,
//       as_directed_weighted_graph}                          fixed_rule/mod.rs:86-103,136-328
//   RegularTempStore::put                                    runtime/temp_store.rs:58-60
//   Poison::check                                            runtime/db.rs:1926-1942
//   PageRank / ShortestPathDijkstra / ClosenessCentrality / BetweennessCentrality
//       (fixed_rule/algos/{pagerank,shortest_path_dijkstra,all_pairs_shortest_path}.rs)
#pragma once
#include <atomic>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>

#include "../../include/cozo_gpu.h"
#include "data_value.hpp"
#include "memcmp.hpp"

namespace cozo_host {

// ---- Poison (runtime/db.rs:1926-1942) -------------------------------------------
struct Poison {
  // an int-sized flag so that its address can be handed to the C ABI (`const volatile int*`)
  std::shared_ptr<std::atomic<int>> flag = std::make_shared<std::atomic<int>>(0);
  void check() const {
    if (flag->load()) throw CozoError("eval::killed", "Running query is killed before completion");
  }
  void kill() const { flag->store(1); }
  const volatile int* raw() const { return reinterpret_cast<const volatile int*>(flag.get()); }
};

// ---- RegularTempStore (runtime/temp_store.rs:27-29,58-60) --------------------------
struct RegularTempStore {
  std::map<Tuple, bool, TupleLess> inner;
  void put(Tuple t) { inner.emplace(std::move(t), false); }  // RegularTempStore::put (temp_store.rs:58-60)
  // Bulk fill for rules that emit one row per node: rows arrive in ascending key order (the glue walks its
  // key -> id dictionary in order), so every insert is an append at the end of the tree.  MEASURED on this
  // std::map twin (_cozo_host.bench_tempstore_fill, 2M rows): no gain — 1.3 s with put, 1.7 s through the
  // ordered walk; the time goes into materialising the tuples, not into the tree.  Kept for the record and not
  // used by the rules; whether Rust's BTreeMap bulk build (`from_iter` over a sorted iterator) does better is
  // unverified (INTEGRATION.md §3).
  template <class RowFn>  // row(i) -> Tuple for i in [0,n), ascending keys
  void put_sorted_bulk(size_t n, RowFn row) {
    for (size_t i = 0; i < n; ++i) inner.emplace_hint(inner.end(), row(i), false);  // a wrong hint only costs time
  }
  std::vector<Tuple> rows() const {
    std::vector<Tuple> r;
    for (auto& kv : inner) r.push_back(kv.first);
    return r;
  }
};

// the first field of every non-empty row: the node keys of a starting / termination relation
inline std::vector<const DataValue*> first_fields(const std::vector<Tuple>& rows) {
  std::vector<const DataValue*> out;
  for (const Tuple& t : rows)
    if (!t.empty()) out.push_back(&t[0]);
  return out;
}

inline void gpu_check(int rc) {
  if (rc == COZO_GPU_OK) return;
  const char* msg = cozo_gpu_last_error();
  if (rc == COZO_GPU_EKILLED) throw CozoError("eval::killed", "Running query is killed before completion");
  throw CozoError("gpu::error", std::string("cozo_gpu error ") + std::to_string(rc) + ": " + (msg ? msg : ""));
}

// The graph on the device: what GraphBuilder::edges / edges_with_values receives (fixed_rule/mod.rs:192-195,
// 318-321) after cozo_gpu_graph_stage_keys assigned the dense ids, plus the id -> key table.
struct StagedGraph {
  cozo_gpu_graph_t* g = nullptr;
  std::vector<DataValue> indices;  // id -> key
  uint64_t n_edges = 0;            // after mirroring
  uint32_t node_count() const { return (uint32_t)indices.size(); }
  // key -> id, COZO_GPU_NONE where the graph has no such node (cozo_gpu_graph_lookup_keys on memcmp encodings)
  std::vector<uint32_t> lookup(const std::vector<const DataValue*>& keys) const {
    std::string kb;
    std::vector<uint64_t> ko{0};
    for (const DataValue* k : keys) {
      memcmp_codec::encode_datavalue(kb, *k);
      ko.push_back(kb.size());
    }
    std::vector<uint32_t> ids(keys.size());
    if (!keys.empty())
      gpu_check(cozo_gpu_graph_lookup_keys(g, reinterpret_cast<const uint8_t*>(kb.data()), ko.data(),
                                           (uint32_t)keys.size(), ids.data()));
    return ids;
  }
  // the dense edge stream read back in out-CSR order: by (src, dst), parallel edges in input order
  void edges(std::vector<uint32_t>& src, std::vector<uint32_t>& dst, std::vector<float>& w) const {
    std::vector<uint32_t> ptr((size_t)node_count() + 1);
    src.resize(n_edges);
    dst.resize(n_edges);
    w.resize(n_edges);
    gpu_check(cozo_gpu_graph_export(g, ptr.data(), dst.data(), w.data(), nullptr, nullptr));
    for (uint32_t u = 0; u < node_count(); ++u)
      for (uint32_t e = ptr[u]; e < ptr[u + 1]; ++e) src[e] = u;
  }
  StagedGraph() = default;
  StagedGraph(const StagedGraph&) = delete;
  StagedGraph& operator=(const StagedGraph&) = delete;
  ~StagedGraph() {
    if (g) cozo_gpu_graph_free(g);
  }
};

// ---- FixedRuleInputRelation (fixed_rule/mod.rs:55-329) ------------------------------
struct FixedRuleInputRelation {
  const std::vector<Tuple>* tuples = nullptr;  // scan order (stored relation: key order)
  size_t declared_arity = 0;

  size_t arity() const { return declared_arity; }
  const std::vector<Tuple>& iter() const { return *tuples; }
  const FixedRuleInputRelation& ensure_min_len(size_t len) const {  // mod.rs:67-80
    if (declared_arity < len)
      throw CozoError("algo::input_relation_bad_arity", "Input relation to algorithm has insufficient arity");
    return *this;
  }

  // as_directed_graph (mod.rs:136-200) / as_directed_weighted_graph (mod.rs:208-328)
  void as_graph(bool undirected, bool weighted, bool allow_negative_weights, StagedGraph& out) const {
    // endpoint keys as memcmp encodings (data/memcmp.rs: equal bytes <=> equal values); the device assigns the dense
    // ids in first-appearance order (mod.rs:164-179)
    std::string kb;
    std::vector<uint64_t> ko{0};
    std::vector<float> w;
    ko.reserve(tuples->size() * 2 + 1);
    std::unique_ptr<CozoError> error;  // the reference records the error and keeps scanning
    for (const Tuple& t : *tuples) {
      if (t.size() < 2) {  // mod.rs:150-163
        error.reset(new CozoError("algo::not_an_edge", "The relation cannot be interpreted as an edge"));
        continue;
      }
      float wv = 1.0f;  // mod.rs:254-255
      if (weighted && t.size() >= 3) {
        double x;
        if (!t[2].get_float(x) || !std::isfinite(x) || (x < 0. && !allow_negative_weights)) {  // mod.rs:256-303
          error.reset(new CozoError("algo::invalid_edge_weight",
                                    "The value " + t[2].repr() + " cannot be interpreted as an edge weight"));
          continue;
        }
        wv = (float)x;  // mod.rs:306
      }
      memcmp_codec::encode_datavalue(kb, t[0]);
      ko.push_back(kb.size());
      memcmp_codec::encode_datavalue(kb, t[1]);
      ko.push_back(kb.size());
      if (weighted) w.push_back(wv);
    }
    if (error) throw *error;
    // no error: edge e is tuple e, so endpoint i is field i % 2 of tuple i / 2
    const uint64_t m = (ko.size() - 1) / 2;
    uint32_t n = 0;
    gpu_check(cozo_gpu_graph_stage_keys(&out.g, m, reinterpret_cast<const uint8_t*>(kb.data()), ko.data(),
                                        weighted ? w.data() : nullptr, undirected ? 1 : 0, &n));
    out.n_edges = undirected ? 2 * m : m;  // mod.rs:187-191, 313-317 (mirrored on the device)
    std::vector<uint64_t> first(n);
    gpu_check(cozo_gpu_graph_node_endpoints(out.g, first.data()));
    out.indices.reserve(n);
    for (uint64_t ep : first) out.indices.push_back((*tuples)[ep / 2][ep % 2]);
  }
  void as_directed_graph(bool undirected, StagedGraph& out) const { as_graph(undirected, false, false, out); }
  void as_directed_weighted_graph(bool undirected, bool allow_negative_weights, StagedGraph& out) const {
    as_graph(undirected, true, allow_negative_weights, out);
  }
};

// ---- FixedRulePayload (fixed_rule/mod.rs:47-51, 331-535) -----------------------------
using Options = std::map<std::string, DataValue>;  // BTreeMap<SmartString, Expr>, constants only

struct FixedRulePayload {
  std::string rule_name;
  std::vector<FixedRuleInputRelation> inputs;
  Options options;

  size_t inputs_count() const { return inputs.size(); }
  const FixedRuleInputRelation& get_input(size_t idx) const {
    if (idx >= inputs.size())
      throw CozoError("algo::not_enough_args", "Cannot find a required positional argument at index " +
                                                   std::to_string(idx) + " for '" + rule_name + "'");
    return inputs[idx];
  }
  bool has_input(size_t idx) const { return idx < inputs.size(); }
  const std::string& name() const { return rule_name; }

  [[noreturn]] void not_found(const std::string& n) const {
    throw CozoError("fixed_rule::specified_option_not_found",
                    "Cannot find a required named option '" + n + "' for '" + rule_name + "'");
  }
  [[noreturn]] void wrong(const std::string& n, const std::string& help) const {
    throw CozoError("fixed_rule::arg_wrong", "Wrong value for option '" + n + "' of '" + rule_name + "': " + help);
  }
  int64_t integer_option(const std::string& n, const int64_t* dflt) const {  // mod.rs:405-437
    auto it = options.find(n);
    if (it == options.end()) {
      if (dflt) return *dflt;
      not_found(n);
    }
    if (it->second.kind != DataValue::Num) wrong(n, "an integer is required");
    int64_t v;
    if (!it->second.get_int(v)) not_found(n);  // sic: the reference reports "not found" here
    return v;
  }
  size_t pos_integer_option(const std::string& n, const size_t* dflt) const {  // mod.rs:438-450
    int64_t d = dflt ? (int64_t)*dflt : 0;
    int64_t v = integer_option(n, dflt ? &d : nullptr);
    if (!(v > 0)) wrong(n, "a positive integer is required");
    return (size_t)v;
  }
  size_t non_neg_integer_option(const std::string& n, const size_t* dflt) const {  // mod.rs:451-463
    int64_t d = dflt ? (int64_t)*dflt : 0;
    int64_t v = integer_option(n, dflt ? &d : nullptr);
    if (!(v >= 0)) wrong(n, "a non-negative integer is required");
    return (size_t)v;
  }
  double float_option(const std::string& n, const double* dflt) const {  // mod.rs:464-491
    auto it = options.find(n);
    if (it == options.end()) {
      if (dflt) return *dflt;
      not_found(n);
    }
    double v;
    if (!it->second.get_float(v)) wrong(n, "a floating number is required");
    return v;
  }
  double unit_interval_option(const std::string& n, const double* dflt) const {  // mod.rs:492-504
    double v = float_option(n, dflt);
    if (!(v >= 0. && v <= 1.)) wrong(n, "a number between 0. and 1. is required");
    return v;
  }
  bool bool_option(const std::string& n, const bool* dflt) const {  // mod.rs:505-533
    auto it = options.find(n);
    if (it == options.end()) {
      if (dflt) return *dflt;
      not_found(n);
    }
    bool v;
    if (!it->second.get_bool(v)) wrong(n, "a boolean value is required");
    return v;
  }
  std::string string_option(const std::string& n, const char* dflt) const {  // mod.rs:362-391
    auto it = options.find(n);
    if (it == options.end()) {
      if (dflt) return dflt;
      not_found(n);
    }
    if (it->second.kind != DataValue::Str) wrong(n, "a string is required");
    return it->second.s;
  }
};

// ---- trait FixedRule (fixed_rule/mod.rs:538-567) ---------------------------------------
struct FixedRule {
  virtual ~FixedRule() = default;
  virtual void init_options(Options&) const {}
  virtual size_t arity(const Options& options, const std::vector<std::string>& rule_head) const = 0;
  virtual void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const = 0;
};

// SimpleFixedRule (fixed_rule/mod.rs:571-689): arity + a callback over (inputs, options)
struct SimpleFixedRule : FixedRule {
  using Fn = std::function<std::vector<Tuple>(const std::vector<std::vector<Tuple>>&, const Options&)>;
  size_t return_arity;
  Fn rule;
  SimpleFixedRule(size_t a, Fn f) : return_arity(a), rule(std::move(f)) {}
  size_t arity(const Options&, const std::vector<std::string>&) const override { return return_arity; }
  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison&) const override {
    std::vector<std::vector<Tuple>> ins;
    for (auto& r : payload.inputs) ins.push_back(r.iter());
    for (auto& row : rule(ins, payload.options)) {
      if (row.size() != return_arity)  // mod.rs:672-680
        throw CozoError("parser::simple_fixed_rule_bad_arity", "arity mismatch: expect " +
                                                                   std::to_string(return_arity) + ", got " +
                                                                   std::to_string(row.size()));
      out.put(row);
    }
  }
};

// ---- PageRank (fixed_rule/algos/pagerank.rs:25-66) --------------------------------------
struct PageRank : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 2; }
  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    const bool f = false;
    const double th = 0.85, ep = 0.0001;
    const size_t it10 = 10;
    bool undirected = payload.bool_option("undirected", &f);              // pagerank.rs:36
    float theta = (float)payload.unit_interval_option("theta", &th);      // :37
    float epsilon = (float)payload.unit_interval_option("epsilon", &ep);  // :38
    size_t iterations = payload.pos_integer_option("iterations", &it10);  // :39
    StagedGraph g;
    edges.as_directed_graph(undirected, g);
    if (g.indices.empty()) return;  // :43-45
    std::vector<float> ranks(g.node_count());
    uint32_t n_run = 0;
    double err = 0;
    gpu_check(cozo_gpu_pagerank(g.g, theta, (double)epsilon, (uint32_t)iterations, ranks.data(), &n_run, &err, nullptr,
                                poison.raw()));
    for (size_t idx = 0; idx < ranks.size(); ++idx)  // :52-54
      out.put({g.indices[idx], DataValue::from_float((double)ranks[idx])});
  }
};

// ---- ShortestPathDijkstra (fixed_rule/algos/shortest_path_dijkstra.rs:30-163) -----------
struct ShortestPathDijkstra : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 4; }

  // every tied shortest path start -> target over the tied-predecessor edges of one source (cozo_gpu_sssp_goals with
  // keep_ties; the reference keeps predecessor lists while searching, :372-380, and enumerates them at :397-426).
  // `tied` = (v, p) pairs sorted by v.
  static void collect(const std::vector<std::pair<uint32_t, uint32_t>>& tied, uint32_t start,
                      std::vector<uint32_t>& chain, std::vector<std::vector<uint32_t>>& paths, const Poison& poison) {
    const uint32_t last = chain.back();
    auto it = std::lower_bound(tied.begin(), tied.end(), std::make_pair(last, 0u));
    for (; it != tied.end() && it->first == last; ++it) {
      const uint32_t p = it->second;
      poison.check();
      chain.push_back(p);
      if (p == start) {
        paths.emplace_back(chain.rbegin(), chain.rend());
      } else {
        collect(tied, start, chain, paths, poison);
      }
      chain.pop_back();
    }
  }

  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    const auto& starting = payload.get_input(1);
    const bool f = false;
    bool undirected = payload.bool_option("undirected", &f);  // :42
    bool keep_ties = payload.bool_option("keep_ties", &f);    // :43
    StagedGraph g;
    edges.as_directed_weighted_graph(undirected, false, g);
    std::set<uint32_t> starting_nodes;  // BTreeSet, :47-54
    for (uint32_t id : g.lookup(first_fields(starting.iter())))
      if (id != COZO_GPU_NONE) starting_nodes.insert(id);
    bool has_term = payload.has_input(2);  // `termination` is optional, :41,55-68
    std::set<uint32_t> termination_nodes;
    if (has_term)
      for (uint32_t id : g.lookup(first_fields(payload.get_input(2).iter())))
        if (id != COZO_GPU_NONE) termination_nodes.insert(id);
    if (starting_nodes.empty()) return;
    const uint32_t n = g.node_count();
    std::vector<uint32_t> sources(starting_nodes.begin(), starting_nodes.end());
    auto put = [&](uint32_t start, uint32_t target, float cost, const uint32_t* path, size_t len) {
      std::vector<DataValue> pl;
      for (size_t i = 0; i < len; ++i) pl.push_back(g.indices[path[i]]);
      out.put({g.indices[start], g.indices[target], DataValue::from_float((double)cost),
               DataValue::from_list(std::move(pl))});  // :88-99
    };
    if (!has_term) {
      // Goal for (): every node, 0..total (:233-235); keep_ties falls back to plain dijkstra (:85-87)
      std::vector<float> dist((size_t)sources.size() * n);
      std::vector<uint32_t> pred((size_t)sources.size() * n);
      gpu_check(cozo_gpu_sssp_multi(g.g, sources.data(), (uint32_t)sources.size(), dist.data(), pred.data(), nullptr,
                                    poison.raw()));
      std::vector<uint32_t> path;
      for (size_t si = 0; si < sources.size(); ++si) {
        const uint32_t start = sources[si];
        const float* d = dist.data() + si * n;
        const uint32_t* p = pred.data() + si * n;
        for (uint32_t t = 0; t < n; ++t) {
          path.clear();
          if (std::isfinite(d[t])) {  // :325-333; unreachable: (inf, []) :322-323
            for (uint32_t cur = t; cur != start; cur = p[cur]) path.push_back(cur);
            path.push_back(start);
            std::reverse(path.begin(), path.end());
          }
          put(start, t, d[t], path.data(), path.size());
        }
        poison.check();
      }
      return;
    }
    // an empty termination set means "already exhausted": the search stops after the start
    // node and the goal iterator is empty (Goal for BTreeSet, :260-272) => no rows.
    if (termination_nodes.empty()) return;
    // with goals, each search stops once they are settled (is_exhausted, :312-315): only the goal answers come back
    const std::vector<uint32_t> goals(termination_nodes.begin(), termination_nodes.end());
    const size_t ns = sources.size(), ng = goals.size();
    std::vector<float> cost(ns * ng);
    std::vector<uint64_t> off(keep_ties ? ns + 1 : ns * ng + 1);
    std::vector<uint32_t> rows;
    for (uint64_t cap = 16 * ns * ng;;) {  // a first guess; the call reports the total when it does not fit
      rows.resize(std::max<uint64_t>(cap, 1) * (keep_ties ? 2 : 1));
      gpu_check(cozo_gpu_sssp_goals(g.g, sources.data(), (uint32_t)ns, goals.data(), (uint32_t)ng, keep_ties ? 1 : 0,
                                    cost.data(), keep_ties ? nullptr : off.data(), keep_ties ? nullptr : rows.data(),
                                    keep_ties ? 0 : cap, keep_ties ? off.data() : nullptr,
                                    keep_ties ? rows.data() : nullptr, keep_ties ? cap : 0, nullptr, poison.raw()));
      if (off.back() <= cap) break;
      cap = off.back();
    }
    std::vector<std::pair<uint32_t, uint32_t>> tied;
    std::vector<std::vector<uint32_t>> paths;
    for (size_t si = 0; si < ns; ++si) {
      const uint32_t start = sources[si];
      if (keep_ties) {
        tied.clear();
        for (uint64_t e = off[si]; e < off[si + 1]; ++e) tied.push_back({rows[2 * e], rows[2 * e + 1]});
        std::sort(tied.begin(), tied.end());
      }
      for (size_t gi = 0; gi < ng; ++gi) {
        const uint32_t target = goals[gi];
        const float c = cost[si * ng + gi];
        if (!std::isfinite(c)) {  // :322-323
          put(start, target, c, nullptr, 0);
        } else if (!keep_ties) {  // :325-333
          const uint64_t b = off[si * ng + gi];
          put(start, target, c, rows.data() + b, off[si * ng + gi + 1] - b);
        } else if (target != start) {  // collect() finds no predecessor of the start (:410-421)
          paths.clear();
          std::vector<uint32_t> chain{target};
          collect(tied, start, chain, paths, poison);
          for (auto& path : paths) put(start, target, c, path.data(), path.size());
        }
      }
      poison.check();
    }
  }
};

// ---- ClosenessCentrality (fixed_rule/algos/all_pairs_shortest_path.rs:97-143) ------------
struct ClosenessCentrality : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 2; }
  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    const bool f = false;
    bool undirected = payload.bool_option("undirected", &f);  // :107
    StagedGraph g;
    edges.as_directed_weighted_graph(undirected, false, g);
    const uint32_t n = g.node_count();
    if (n == 0) return;  // :111-113
    std::vector<float> res(n);
    gpu_check(cozo_gpu_closeness(g.g, res.data(), nullptr, poison.raw()));
    for (uint32_t idx = 0; idx < n; ++idx) {  // :125-131
      out.put({g.indices[idx], DataValue::from_float((double)res[idx])});
      poison.check();
    }
  }
};

// ---- BetweennessCentrality (fixed_rule/algos/all_pairs_shortest_path.rs:29-95) -----------
struct BetweennessCentrality : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 2; }
  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    const bool f = false;
    bool undirected = payload.bool_option("undirected", &f);  // :39
    StagedGraph g;
    edges.as_directed_weighted_graph(undirected, false, g);
    const uint32_t n = g.node_count();
    if (n == 0) return;  // :43-46
    std::vector<float> c(n);
    gpu_check(cozo_gpu_betweenness(g.g, c.data(), nullptr, poison.raw()));
    for (uint32_t i = 0; i < n; ++i) out.put({g.indices[i], DataValue::from_float((double)c[i])});  // :79-82
  }
};

// ---- ClusteringCoefficients (fixed_rule/algos/triangles.rs:25-57) ------------------------------
struct ClusteringCoefficients : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 4; }
  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    StagedGraph g;
    edges.as_directed_graph(true, g);  // always undirected, triangles.rs:35
    const uint32_t n = g.node_count();
    if (n == 0) return;
    std::vector<double> cc(n);
    std::vector<uint64_t> nt(n), deg(n);
    gpu_check(cozo_gpu_clustering(g.g, cc.data(), nt.data(), deg.data(), nullptr, poison.raw()));
    for (uint32_t idx = 0; idx < n; ++idx)  // triangles.rs:37-44
      out.put({g.indices[idx], DataValue::from_float(cc[idx]), DataValue::from_int((int64_t)nt[idx]),
               DataValue::from_int((int64_t)deg[idx])});
  }
};

// ---- KShortestPathYen (fixed_rule/algos/yen.rs:26-211) ------------------------------------------
// The control flow of k_shortest_path_yen is the reference's; what changes is that the dijkstra
// calls of one round — every spur node of every (start, goal) pair, which the reference runs one
// after another (pairs in parallel via par_bridge, yen.rs:85) — go to the device as ONE batch of
// goal-directed searches with their ForbiddenEdge / ForbiddenNode sets (cozo_gpu_sssp_paths).
struct KShortestPathYen : FixedRule {
  size_t arity(const Options&, const std::vector<std::string>&) const override { return 4; }

  struct PairState {
    uint32_t start, goal;
    std::vector<std::pair<float, std::vector<uint32_t>>> k_shortest, candidates;
    bool done = false;
  };
  struct Search {
    size_t pair;
    size_t i;  // spur index, or SIZE_MAX for the initial search
    uint32_t from;
    std::vector<uint32_t> fn;
    std::vector<std::pair<uint32_t, uint32_t>> fe;
  };

  static void run_batch(const StagedGraph& g, const std::vector<PairState>& ps, const std::vector<Search>& batch,
                        std::vector<std::pair<float, std::vector<uint32_t>>>& res, const Poison& poison) {
    const uint32_t k = (uint32_t)batch.size();
    res.assign(k, {});
    if (!k) return;
    std::vector<uint32_t> src(k), goal(k), fnp(k + 1, 0), fep(k + 1, 0), fnn, fes, fed;
    for (uint32_t b = 0; b < k; ++b) {
      src[b] = batch[b].from;
      goal[b] = ps[batch[b].pair].goal;
      for (uint32_t v : batch[b].fn) fnn.push_back(v);
      for (auto& e : batch[b].fe) {
        fes.push_back(e.first);
        fed.push_back(e.second);
      }
      fnp[b + 1] = (uint32_t)fnn.size();
      fep[b + 1] = (uint32_t)fes.size();
    }
    if (fnn.empty()) fnn.push_back(0);
    if (fes.empty()) {
      fes.push_back(0);
      fed.push_back(0);
    }
    uint32_t max_len = 64;
    for (;;) {
      std::vector<float> cost(k);
      std::vector<uint32_t> len(k), paths((size_t)k * max_len);
      gpu_check(cozo_gpu_sssp_paths(g.g, src.data(), goal.data(), k, fnp.data(), fnn.data(), fep.data(), fes.data(),
                                    fed.data(), max_len, cost.data(), len.data(), paths.data(), nullptr, poison.raw()));
      uint32_t need = 0;
      for (uint32_t b = 0; b < k; ++b) need = std::max(need, len[b]);
      if (need > max_len) {
        max_len = need;
        continue;
      }
      for (uint32_t b = 0; b < k; ++b)
        res[b] = {cost[b], std::vector<uint32_t>(paths.begin() + (size_t)b * max_len,
                                                 paths.begin() + (size_t)b * max_len + len[b])};
      return;
    }
  }

  void run(const FixedRulePayload& payload, RegularTempStore& out, const Poison& poison) const override {
    const auto& edges = payload.get_input(0);
    const auto& starting = payload.get_input(1);
    const auto& termination = payload.get_input(2);
    const bool f = false;
    bool undirected = payload.bool_option("undirected", &f);  // yen.rs:38
    size_t k = payload.pos_integer_option("k", nullptr);      // yen.rs:39 (required)
    StagedGraph g;
    edges.as_directed_weighted_graph(undirected, false, g);
    std::set<uint32_t> starts, goals;  // BTreeSets, yen.rs:43-58
    for (uint32_t id : g.lookup(first_fields(starting.iter())))
      if (id != COZO_GPU_NONE) starts.insert(id);
    for (uint32_t id : g.lookup(first_fields(termination.iter())))
      if (id != COZO_GPU_NONE) goals.insert(id);
    std::vector<PairState> ps;
    for (uint32_t s0 : starts)
      for (uint32_t g0 : goals) {
        PairState p;
        p.start = s0;
        p.goal = g0;
        ps.push_back(std::move(p));
      }
    if (ps.empty()) return;
    // first edge s->d in adjacency order supplies the root-path cost (yen.rs:171-183); the CSR keeps parallel edges
    // in input order
    std::map<std::pair<uint32_t, uint32_t>, float> first_edge;
    {
      std::vector<uint32_t> es, ed;
      std::vector<float> ew;
      g.edges(es, ed, ew);
      for (size_t e = 0; e < es.size(); ++e) first_edge.emplace(std::make_pair(es[e], ed[e]), ew[e]);
    }

    std::vector<Search> batch;
    std::vector<std::pair<float, std::vector<uint32_t>>> res;
    for (size_t pi = 0; pi < ps.size(); ++pi) batch.push_back({pi, SIZE_MAX, ps[pi].start, {}, {}});
    run_batch(g, ps, batch, res, poison);
    for (size_t b = 0; b < batch.size(); ++b) ps[batch[b].pair].k_shortest.push_back(res[b]);  // yen.rs:130-136

    for (size_t it = 1; it < k; ++it) {  // yen.rs:138
      batch.clear();
      for (size_t pi = 0; pi < ps.size(); ++pi) {
        PairState& p = ps[pi];
        if (p.done) continue;
        const std::vector<uint32_t>& prev = p.k_shortest.back().second;
        for (size_t i = 0; i + 1 < prev.size(); ++i) {
          Search sr;
          sr.pair = pi;
          sr.i = i;
          sr.from = prev[i];
          for (auto& cp : p.k_shortest) {  // yen.rs:147-155
            const auto& path = cp.second;
            if (path.size() < i + 2) continue;
            if (std::equal(prev.begin(), prev.begin() + i + 1, path.begin())) sr.fe.push_back({path[i], path[i + 1]});
          }
          sr.fn.assign(prev.begin(), prev.begin() + i);  // yen.rs:156-159
          batch.push_back(std::move(sr));
        }
      }
      run_batch(g, ps, batch, res, poison);
      for (size_t b = 0; b < batch.size(); ++b) {
        PairState& p = ps[batch[b].pair];
        const std::vector<uint32_t>& prev = p.k_shortest.back().second;
        const size_t i = batch[b].i;
        float total = res[b].first;
        for (size_t j = 0; j < i; ++j) {
          auto fe = first_edge.find({prev[j], prev[j + 1]});
          if (fe != first_edge.end()) total += fe->second;
        }
        std::vector<uint32_t> total_path(prev.begin(), prev.begin() + i);
        total_path.insert(total_path.end(), res[b].second.begin(), res[b].second.end());
        bool dup = false;
        for (auto& c : p.candidates)
          if (c.second == total_path) dup = true;
        if (!dup) p.candidates.push_back({total, std::move(total_path)});  // yen.rs:187-189
      }
      poison.check();
      for (PairState& p : ps) {
        if (p.done) continue;
        if (p.candidates.empty()) {  // yen.rs:194-196
          p.done = true;
          continue;
        }
        std::stable_sort(p.candidates.begin(), p.candidates.end(),
                         [](const auto& a, const auto& b) { return b.first < a.first; });  // yen.rs:197
        auto shortest = p.candidates.back();
        p.candidates.pop_back();
        if (std::isfinite(shortest.first)) p.k_shortest.push_back(std::move(shortest));  // yen.rs:200-203
      }
    }
    for (const PairState& p : ps)
      for (auto& cp : p.k_shortest) {  // yen.rs:62-77, 103-117
        std::vector<DataValue> pl;
        for (uint32_t u : cp.second) pl.push_back(g.indices[u]);
        out.put({g.indices[p.start], g.indices[p.goal], DataValue::from_float((double)cp.first),
                 DataValue::from_list(std::move(pl))});
      }
  }
};

// ---- registry (fixed_rule/mod.rs:705-836; Db::register_fixed_rule runtime/db.rs:760-784) ---
struct FixedRuleRegistry {
  std::map<std::string, std::shared_ptr<FixedRule>> rules;
  std::set<std::string> builtin;
  FixedRuleRegistry() {
    add_builtin("PageRank", std::make_shared<PageRank>());
    add_builtin("ShortestPathDijkstra", std::make_shared<ShortestPathDijkstra>());
    add_builtin("ClosenessCentrality", std::make_shared<ClosenessCentrality>());
    add_builtin("BetweennessCentrality", std::make_shared<BetweennessCentrality>());
    add_builtin("ClusteringCoefficients", std::make_shared<ClusteringCoefficients>());
    add_builtin("KShortestPathYen", std::make_shared<KShortestPathYen>());
  }
  void add_builtin(const std::string& n, std::shared_ptr<FixedRule> r) {
    rules[n] = std::move(r);
    builtin.insert(n);
  }
  void register_fixed_rule(const std::string& n, std::shared_ptr<FixedRule> r) {  // db.rs:760-776
    if (rules.count(n)) throw CozoError("", "A fixed rule with the name `" + n + "` is already registered");
    rules[n] = std::move(r);
  }
  bool unregister_fixed_rule(const std::string& n) {  // db.rs:779-784
    if (builtin.count(n)) throw CozoError("", "Cannot unregister builtin fixed rule `" + n + "`");
    return rules.erase(n) > 0;
  }
  // what parse_fixed_rule + eval.rs:170-180 do for `?[..] <~ Name(inputs.., opts..)`:
  // init_options, exact arity check against the rule head, one run in epoch 0
  std::vector<Tuple> run(const std::string& n, const std::vector<std::vector<Tuple>>& inputs,
                         const std::vector<size_t>& input_arities, Options options, size_t head_arity,
                         const Poison& poison) const {
    auto it = rules.find(n);
    if (it == rules.end())
      throw CozoError("parser::fixed_rule_not_found", "Fixed rule '" + n + "' not found");
    it->second->init_options(options);
    size_t ar = it->second->arity(options, {});
    if (head_arity != 0 && head_arity != ar)  // parse/query.rs:1010-1019
      throw CozoError("parser::fixed_rule_head_arity_mismatch",
                      "Fixed rule head arity mismatch: expected " + std::to_string(ar) + ", found " +
                          std::to_string(head_arity));
    FixedRulePayload p;
    p.rule_name = n;
    p.options = std::move(options);
    for (size_t i = 0; i < inputs.size(); ++i) {
      FixedRuleInputRelation r;
      r.tuples = &inputs[i];
      r.declared_arity = i < input_arities.size() ? input_arities[i] : (inputs[i].empty() ? 0 : inputs[i][0].size());
      p.inputs.push_back(r);
    }
    RegularTempStore out;
    it->second->run(p, out, poison);
    return out.rows();
  }
};

}  // namespace cozo_host
