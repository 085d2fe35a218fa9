// cozo_oracle.cpp — CPU ORACLE (test infrastructure, NOT product code).
//
// A single-file C++17 restatement of the CozoDB v0.7.6 algorithms on the
// north-star hot path.  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library; the product
// (cozo_b200/csrc) never links, imports or calls it.
//
// PARITY UNPINNED: the reference ships no golden vector / known-answer test for
// any function restated here (SURVEY.md §4, §8c) and cannot be compiled in this
// environment (no Rust toolchain).  Correctness of this file is anchored on the
// algorithm text cited per function, and cross-checked in tests/ against
// independent implementations (brute force, scipy, networkx).
//
// Build: see oracle/Makefile  (-O2 -ffp-contract=off so f32 results do not
// depend on FMA contraction; the reference is Rust, which never contracts).
//
// Reference citations are `path:line` under /root/reference/cozo-core/src/.

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <set>
#include <thread>
#include <unordered_set>
#include <vector>

namespace {

// ---------------------------------------------------------------------------
// a1. distances — runtime/hnsw.rs:66-109 (VectorCache::dist)
// f32 arithmetic as ndarray 0.15.6 does it (Cargo.lock:2349): `a - b` is an
// elementwise f32 subtraction into a temporary; `dot` is numeric_util::
// unrolled_dot: eight independent accumulators over chunks of 8, combined as
// sum += (p0+p4); sum += (p1+p5); sum += (p2+p6); sum += (p3+p7); then the
// (<8) tail elements are added one by one.  Result cast to f64.
// ---------------------------------------------------------------------------
static float unrolled_dot(const float* x, const float* y, size_t n) {
  float p0 = 0, p1 = 0, p2 = 0, p3 = 0, p4 = 0, p5 = 0, p6 = 0, p7 = 0;
  size_t i = 0;
  for (; i + 8 <= n; i += 8) {
    p0 = p0 + x[i + 0] * y[i + 0];
    p1 = p1 + x[i + 1] * y[i + 1];
    p2 = p2 + x[i + 2] * y[i + 2];
    p3 = p3 + x[i + 3] * y[i + 3];
    p4 = p4 + x[i + 4] * y[i + 4];
    p5 = p5 + x[i + 5] * y[i + 5];
    p6 = p6 + x[i + 6] * y[i + 6];
    p7 = p7 + x[i + 7] * y[i + 7];
  }
  float sum = 0;
  sum = sum + (p0 + p4);
  sum = sum + (p1 + p5);
  sum = sum + (p2 + p6);
  sum = sum + (p3 + p7);
  for (; i < n; ++i) sum = sum + x[i] * y[i];
  return sum;
}

// L2 needs the temporary `diff` array (hnsw.rs:70).  Same accumulator
// structure as unrolled_dot(diff, diff), without materialising diff.
static float unrolled_sqdiff(const float* a, const float* b, size_t n) {
  float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  size_t i = 0;
  for (; i + 8 <= n; i += 8) {
    for (int j = 0; j < 8; ++j) {
      float d = a[i + j] - b[i + j];
      p[j] = p[j] + d * d;
    }
  }
  float sum = 0;
  sum = sum + (p[0] + p[4]);
  sum = sum + (p[1] + p[5]);
  sum = sum + (p[2] + p[6]);
  sum = sum + (p[3] + p[7]);
  for (; i < n; ++i) {
    float d = a[i] - b[i];
    sum = sum + d * d;
  }
  return sum;
}

enum Metric { L2 = 0, COSINE = 1, IP = 2 };  // parse/sys.rs:94-98

static double vec_dist(int metric, const float* a, const float* b, size_t n) {
  switch (metric) {
    case L2:  // hnsw.rs:68-72  (squared, no sqrt)
      return (double)unrolled_sqdiff(a, b, n);
    case COSINE: {  // hnsw.rs:79-85
      double an = (double)unrolled_dot(a, a, n);
      double bn = (double)unrolled_dot(b, b, n);
      double dot = (double)unrolled_dot(a, b, n);
      return 1.0 - dot / std::sqrt(an * bn);
    }
    default: {  // hnsw.rs:97-101
      float dot = unrolled_dot(a, b, n);
      return 1.0 - (double)dot;
    }
  }
}

// F64 vector indexes (hnsw.rs:73-76, 86-93, 102-107): the same expressions with f64 operands throughout;
// ndarray's unrolled_dot is generic over the element type, so the accumulator structure is the same.
static double unrolled_dot64(const double* x, const double* y, size_t n) {
  double p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  size_t i = 0;
  for (; i + 8 <= n; i += 8)
    for (int j = 0; j < 8; ++j) p[j] = p[j] + x[i + j] * y[i + j];
  double sum = 0;
  sum = sum + (p[0] + p[4]);
  sum = sum + (p[1] + p[5]);
  sum = sum + (p[2] + p[6]);
  sum = sum + (p[3] + p[7]);
  for (; i < n; ++i) sum = sum + x[i] * y[i];
  return sum;
}
static double vec_dist64(int metric, const double* a, const double* b, size_t n) {
  switch (metric) {
    case L2: {  // hnsw.rs:73-76: diff = a - b (materialised), diff.dot(&diff)
      std::vector<double> diff(n);
      for (size_t i = 0; i < n; ++i) diff[i] = a[i] - b[i];
      return unrolled_dot64(diff.data(), diff.data(), n);
    }
    case COSINE: {  // hnsw.rs:86-91
      double an = unrolled_dot64(a, a, n), bn = unrolled_dot64(b, b, n), dot = unrolled_dot64(a, b, n);
      return 1.0 - dot / std::sqrt(an * bn);
    }
    default:  // hnsw.rs:102-105
      return 1.0 - unrolled_dot64(a, b, n);
  }
}

// ---------------------------------------------------------------------------
// priority-queue 1.4.0 stand-in (Cargo.lock:2836).  push = insert-or-replace,
// pop/peek = max priority.  Order among EQUAL priorities is unspecified in the
// crate (heap-shape dependent); here it is made deterministic: larger id wins
// in a max-queue.  Tests therefore use tie-free data (SURVEY.md §7 hard parts).
// Priorities compare as OrderedFloat<f64>: NaN is greater than every number
// (+inf included) and equal to NaN, so a NaN key is an ordinary priority.
// ---------------------------------------------------------------------------
struct OrderedLess {
  bool operator()(const std::pair<double, uint32_t>& a, const std::pair<double, uint32_t>& b) const {
    const bool an = std::isnan(a.first), bn = std::isnan(b.first);
    if (an != bn) return bn;
    if (!an && a.first != b.first) return a.first < b.first;
    return a.second < b.second;
  }
};
using PQSet = std::set<std::pair<double, uint32_t>, OrderedLess>;
struct MaxPQ {
  PQSet s;
  std::map<uint32_t, double> pr;
  size_t size() const { return s.size(); }
  bool empty() const { return s.empty(); }
  void push(uint32_t k, double p) {
    auto it = pr.find(k);
    if (it != pr.end()) {
      s.erase({it->second, k});
      it->second = p;
    } else {
      pr.emplace(k, p);
    }
    s.insert({p, k});
  }
  std::pair<uint32_t, double> peek() const {
    auto it = std::prev(s.end());
    return {it->second, it->first};
  }
  std::pair<uint32_t, double> pop() {
    auto it = std::prev(s.end());
    auto r = std::make_pair(it->second, it->first);
    pr.erase(it->second);
    s.erase(it);
    return r;
  }
  bool contains(uint32_t k) const { return pr.count(k) != 0; }
};
// Min-queue = PriorityQueue<_, Reverse<OrderedFloat>>; smaller id wins ties.
struct MinPQ {
  PQSet s;
  std::map<uint32_t, double> pr;
  size_t size() const { return s.size(); }
  bool empty() const { return s.empty(); }
  void push(uint32_t k, double p) {
    auto it = pr.find(k);
    if (it != pr.end()) {
      s.erase({it->second, k});
      it->second = p;
    } else {
      pr.emplace(k, p);
    }
    s.insert({p, k});
  }
  // push_increase on Reverse priority == keep the smaller cost
  void push_decrease_cost(uint32_t k, double p) {
    auto it = pr.find(k);
    if (it != pr.end() && !(p < it->second)) return;
    push(k, p);
  }
  std::pair<uint32_t, double> pop() {
    auto it = s.begin();
    auto r = std::make_pair(it->second, it->first);
    pr.erase(it->second);
    s.erase(it);
    return r;
  }
};

// ---------------------------------------------------------------------------
// Flat, read-only view of an HNSW index after the reading rules of
// hnsw_get_neighbours(include_deleted=false) (hnsw.rs:588-629) were applied:
// self-loops / same-row edges and ignore_link edges removed, neighbours in key
// order (= ascending dense id).  Level index L here means reference layer -L.
// ---------------------------------------------------------------------------
struct LevelView {
  std::vector<uint32_t> node_ids;  // ascending; empty on level 0 (identity)
  std::vector<uint64_t> row_ptr;
  std::vector<uint32_t> col_idx;
  bool identity = false;
  uint32_t n_rows() const { return (uint32_t)(row_ptr.size() - 1); }
  // returns [begin,end) into col_idx, or empty if node not on this level
  std::pair<uint64_t, uint64_t> row(uint32_t id) const {
    if (identity) {
      if (id + 1 >= row_ptr.size()) return {0, 0};
      return {row_ptr[id], row_ptr[id + 1]};
    }
    auto it = std::lower_bound(node_ids.begin(), node_ids.end(), id);
    if (it == node_ids.end() || *it != id) return {0, 0};
    size_t r = it - node_ids.begin();
    return {row_ptr[r], row_ptr[r + 1]};
  }
};

struct HnswView {
  uint32_t n = 0, dim = 0;
  int metric = L2;
  const float* vectors = nullptr;  // borrowed [n x dim]
  std::vector<float> owned;        // or owned copy
  std::vector<LevelView> levels;   // levels[0] = bottom
  uint32_t entry = UINT32_MAX;     // dense id; lives on top level
  bool empty_index = true;
  const float* vec(uint32_t id) const { return vectors + (size_t)id * dim; }
};

struct SearchStats {
  uint64_t dist_evals = 0;      // calls to dist() (incl. entry point)
  uint64_t nodes_expanded = 0;  // candidates whose neighbour list was read
  uint64_t nbr_reads = 0;       // neighbour ids read (sum of degrees)
};

// a4. hnsw_search_level — hnsw.rs:539-587
template <class Dist>  // Dist: double(uint32_t id) = VectorCache::v_dist(q, id)
static void search_level(const HnswView& ix, Dist&& dist_to, size_t ef, uint32_t level,
                         MaxPQ& found_nn, SearchStats& st) {
  std::unordered_set<uint32_t> visited;
  MinPQ candidates;
  for (auto& e : found_nn.s) {  // hnsw.rs:554-557
    visited.insert(e.second);
    candidates.push(e.second, e.first);
  }
  const LevelView& lv = ix.levels[level];
  while (!candidates.empty()) {
    auto [cand, cand_dist] = candidates.pop();  // hnsw.rs:559
    double furthest = found_nn.peek().second;
    if (cand_dist > furthest) break;  // strict, hnsw.rs:562
    auto [b, e] = lv.row(cand);
    st.nodes_expanded++;
    st.nbr_reads += (e - b);
    for (uint64_t i = b; i < e; ++i) {  // key order, hnsw.rs:566
      uint32_t nb = lv.col_idx[i];
      if (visited.count(nb)) continue;
      double d = dist_to(nb);
      st.dist_evals++;
      double far = found_nn.peek().second;  // read BEFORE insertion, hnsw.rs:574
      if (found_nn.size() < ef || d < far) {
        candidates.push(nb, d);
        found_nn.push(nb, d);
        if (found_nn.size() > ef) found_nn.pop();
      }
      visited.insert(nb);
    }
  }
}

// a5. hnsw_knn — hnsw.rs:869-1012, minus the base-row fetch / bind_* columns /
// filter bytecode which are host-engine work.  `k_eff` is k, or ef when a
// filter is present (hnsw.rs:943-947).  Output nearest-first (hnsw.rs:1005).
template <class Dist>
static uint32_t hnsw_knn_with(const HnswView& ix, Dist&& dist_to, uint32_t k, uint32_t ef, double radius,
                              bool has_radius, uint32_t* out_ids, double* out_dist, SearchStats& st) {
  if (ix.empty_index || ix.entry == UINT32_MAX) return 0;  // hnsw.rs:903-909,1009
  MaxPQ found_nn;
  double ep_d = dist_to(ix.entry);
  st.dist_evals++;
  found_nn.push(ix.entry, ep_d);  // hnsw.rs:916-918
  for (uint32_t lvl = (uint32_t)ix.levels.size() - 1; lvl >= 1; --lvl)  // hnsw.rs:919-929
    search_level(ix, dist_to, 1, lvl, found_nn, st);
  search_level(ix, dist_to, ef, 0, found_nn, st);  // hnsw.rs:930-938
  while (found_nn.size() > k) found_nn.pop();  // hnsw.rs:943-947
  std::vector<std::pair<uint32_t, double>> ret;
  while (!found_nn.empty()) {  // hnsw.rs:951-1004
    auto [id, d] = found_nn.pop();
    if (has_radius && d > radius) continue;  // hnsw.rs:952-956
    ret.push_back({id, d});
  }
  std::reverse(ret.begin(), ret.end());  // hnsw.rs:1005
  if (ret.size() > k) ret.resize(k);     // hnsw.rs:1006
  for (size_t i = 0; i < ret.size(); ++i) {
    out_ids[i] = ret[i].first;
    out_dist[i] = ret[i].second;
  }
  return (uint32_t)ret.size();
}

static uint32_t hnsw_knn(const HnswView& ix, const float* q, uint32_t k, uint32_t ef, double radius,
                         bool has_radius, uint32_t* out_ids, double* out_dist, SearchStats& st) {
  return hnsw_knn_with(ix, [&](uint32_t id) { return vec_dist(ix.metric, q, ix.vec(id), ix.dim); }, k, ef, radius,
                       has_radius, out_ids, out_dist, st);
}

// ---------------------------------------------------------------------------
// Faithful index builder: the index *relation* (runtime/relation.rs:1064-1126)
// kept as ordered maps so that scans see key order.  Dense id == key order of
// the base relation key (single vector field, sub-index -1), so "to_k != fr_k"
// (hnsw.rs:609) is `to != fr`.
// ---------------------------------------------------------------------------
struct EdgeVal {
  double dist;
  bool ignore_link;
};
struct LevelRel {
  std::map<uint32_t, double> self_degree;                   // self-loop rows: node -> degree
  std::map<uint32_t, std::map<uint32_t, EdgeVal>> edges;    // (fr, to) -> value, to != fr
};

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

struct HnswBuilder {
  uint32_t dim, n_max;
  int metric;
  uint32_t m, m_max, m_max0, ef_construction;  // relation.rs:1145-1147
  double level_multiplier;
  bool extend_candidates, keep_pruned;
  SplitMix64 rng;  // replaces rand::thread_rng (hnsw.rs:47), seeded for repeatability
  std::vector<float> vectors;
  std::vector<uint8_t> present;
  std::map<int64_t, LevelRel> rel;  // layer (<=0) -> rows; key order = most negative first
  uint64_t dist_evals = 0;

  const float* vec(uint32_t id) const { return vectors.data() + (size_t)id * dim; }
  double dist(const float* a, const float* b) {
    dist_evals++;
    return vec_dist(metric, a, b, dim);
  }

  int64_t random_level() {  // hnsw.rs:46-52
    double u = rng.uniform();
    double r = -std::log(u) * level_multiplier;
    if (!(r < 1e6)) r = 1e6;  // u==0 guard; reference would saturate
    return -(int64_t)std::floor(r);
  }

  // hnsw_get_neighbours — hnsw.rs:588-629
  std::vector<std::pair<uint32_t, double>> neighbours(uint32_t key, int64_t level, bool include_deleted) const {
    std::vector<std::pair<uint32_t, double>> out;
    auto li = rel.find(level);
    if (li == rel.end()) return out;
    auto ei = li->second.edges.find(key);
    if (ei == li->second.edges.end()) return out;
    for (auto& kv : ei->second) {
      if (!include_deleted && kv.second.ignore_link) continue;
      out.push_back({kv.first, kv.second.dist});
    }
    return out;
  }

  // entry point for insertion: first row with layer in [i64::MIN, 0] — hnsw.rs:184-191
  bool entry_point(int64_t& bottom_level, uint32_t& ep) const {
    for (auto& lr : rel) {
      if (!lr.second.self_degree.empty()) {
        bottom_level = lr.first;
        uint32_t first_self = lr.second.self_degree.begin()->first;
        // rows (level, fr, to): the smallest `fr` on this level.  Every node on a
        // level has a self-loop row, so the smallest fr is the smallest self key.
        ep = first_self;
        return true;
      }
    }
    return false;
  }

  void search_level_b(const float* q, size_t ef, int64_t level, MaxPQ& found_nn) {  // hnsw.rs:539-587
    std::unordered_set<uint32_t> visited;
    MinPQ candidates;
    for (auto& e : found_nn.s) {
      visited.insert(e.second);
      candidates.push(e.second, e.first);
    }
    while (!candidates.empty()) {
      auto [cand, cand_dist] = candidates.pop();
      double furthest = found_nn.peek().second;
      if (cand_dist > furthest) break;
      for (auto& nbd : neighbours(cand, level, false)) {
        uint32_t nb = nbd.first;
        if (visited.count(nb)) continue;
        double d = dist(q, vec(nb));
        double far = found_nn.peek().second;
        if (found_nn.size() < ef || d < far) {
          candidates.push(nb, d);
          found_nn.push(nb, d);
          if (found_nn.size() > ef) found_nn.pop();
        }
        visited.insert(nb);
      }
    }
  }

  // hnsw_select_neighbours_heuristic — hnsw.rs:470-538.  Returns nearest-first
  // (the iteration order of `ret`, which is only ever pushed to).
  std::vector<std::pair<uint32_t, double>> select_heuristic(const float* q, uint32_t q_self,
                                                            const std::vector<std::pair<uint32_t, double>>& found,
                                                            size_t mm, int64_t level) {
    MinPQ candidates;
    for (auto& f : found) candidates.push(f.first, f.second);  // hnsw.rs:495-498
    if (extend_candidates) {                                   // hnsw.rs:499-511
      for (auto& f : found)
        for (auto& nbd : neighbours(f.first, level, false)) {
          // NOTE: the reference would also admit the shrink target itself here
          // (and then overwrite its self-loop row, hnsw.rs:413-432); that corner
          // is treated as a reference defect and the self key is skipped.
          if (nbd.first == q_self) continue;
          candidates.push(nbd.first, dist(q, vec(nbd.first)));
        }
    }
    std::vector<std::pair<uint32_t, double>> ret;
    MinPQ discarded;
    while (!candidates.empty() && ret.size() < mm) {  // hnsw.rs:512-529
      auto [ck, cd] = candidates.pop();
      bool should_add = true;
      for (auto& ex : ret) {
        double de = dist(vec(ex.first), vec(ck));
        if (de < cd) {  // strict, hnsw.rs:519
          should_add = false;
          break;
        }
      }
      if (should_add)
        ret.push_back({ck, cd});
      else if (keep_pruned)
        discarded.push(ck, cd);
    }
    if (keep_pruned)  // hnsw.rs:530-536
      while (!discarded.empty() && ret.size() < mm) {
        auto [k2, d2] = discarded.pop();
        ret.push_back({k2, d2});
      }
    return ret;
  }

  // hnsw_shrink_neighbour — hnsw.rs:376-469
  size_t shrink(uint32_t target, size_t mm, int64_t level) {
    auto cand = neighbours(target, level, false);  // stored distances, hnsw.rs:389-393
    auto sel = select_heuristic(vec(target), target, cand, mm, level);
    std::set<uint32_t> oldset, newset;
    for (auto& c : cand) oldset.insert(c.first);
    for (auto& c : sel) newset.insert(c.first);
    auto& rows = rel[level].edges[target];
    for (auto& c : sel)
      if (!oldset.count(c.first)) rows[c.first] = EdgeVal{c.second, false};  // hnsw.rs:413-433
    for (auto& c : cand)
      if (!newset.count(c.first)) {  // hnsw.rs:434-465
        auto it = rows.find(c.first);
        if (it->second.ignore_link)
          rows.erase(it);
        else
          it->second = EdgeVal{c.second, true};
      }
    return sel.size();
  }

  void put_fresh_at_levels(uint32_t id, int64_t bottom, int64_t top) {  // hnsw.rs:630-678
    for (int64_t l = bottom; l <= top; ++l) rel[l].self_degree[id] = 0.0;
  }

  // hnsw_put_vector — hnsw.rs:155-375 (fresh key; re-put of an existing key with
  // a changed vector goes through remove() first, hnsw.rs:175-182)
  int insert(uint32_t id, const float* v, int64_t forced_level) {
    if (id >= n_max) return -1;
    if (present[id]) {
      if (std::memcmp(vec(id), v, dim * sizeof(float)) == 0) return 0;  // same hash, hnsw.rs:176-179
      remove(id);
    }
    std::memcpy(vectors.data() + (size_t)id * dim, v, dim * sizeof(float));
    present[id] = 1;
    const float* q = vec(id);
    int64_t bottom_level;
    uint32_t ep;
    if (!entry_point(bottom_level, ep)) {  // first vector, hnsw.rs:360-373
      int64_t level = forced_level <= 0 ? forced_level : random_level();
      put_fresh_at_levels(id, level, 0);
      return 0;
    }
    MaxPQ found_nn;
    found_nn.push(ep, dist(q, vec(ep)));  // hnsw.rs:200-204
    int64_t target_level = forced_level <= 0 ? forced_level : random_level();
    if (target_level < bottom_level) put_fresh_at_levels(id, target_level, bottom_level - 1);  // hnsw.rs:206-218
    for (int64_t cur = bottom_level; cur < target_level; ++cur) search_level_b(q, 1, cur, found_nn);  // 219-229
    for (int64_t cur = std::max(target_level, bottom_level); cur <= 0; ++cur) {  // hnsw.rs:242-359
      size_t mm = cur == 0 ? m_max0 : m_max;
      search_level_b(q, ef_construction, cur, found_nn);
      std::vector<std::pair<uint32_t, double>> found;
      for (auto& e : found_nn.s) found.push_back({e.second, e.first});
      auto nbrs = select_heuristic(q, id, found, mm, cur);
      LevelRel& lr = rel[cur];
      lr.self_degree[id] = (double)nbrs.size();  // hnsw.rs:269-277
      for (auto& nd : nbrs) {
        lr.edges[id][nd.first] = EdgeVal{nd.second, false};   // out edge, hnsw.rs:281-298
        lr.edges[nd.first][id] = EdgeVal{nd.second, false};   // in edge, hnsw.rs:300-318
        size_t target_degree = (size_t)lr.self_degree[nd.first] + 1;  // hnsw.rs:338
        if (target_degree > mm) target_degree = shrink(nd.first, mm, cur);
        lr.self_degree[nd.first] = (double)target_degree;  // hnsw.rs:352-357
      }
    }
    return 0;
  }

  // hnsw_remove_vec — hnsw.rs:754-868
  void remove(uint32_t id) {
    if (id >= n_max || !present[id]) return;
    for (int64_t layer = 0;; --layer) {
      auto li = rel.find(layer);
      if (li == rel.end() || !li->second.self_degree.count(id)) break;
      li->second.self_degree.erase(id);
      auto nbrs = neighbours(id, layer, true);
      for (auto& nd : nbrs) {
        li->second.edges[id].erase(nd.first);
        auto& back = li->second.edges[nd.first];
        back.erase(id);
        li->second.self_degree[nd.first] -= 1.0;  // hnsw.rs:820
      }
      li->second.edges.erase(id);
      if (li->second.self_degree.empty()) rel.erase(li);
    }
    present[id] = 0;
  }

  // Export with the reading rules of hnsw_get_neighbours(include_deleted=false)
  void to_view(HnswView& v) const {
    v.n = n_max;
    v.dim = dim;
    v.metric = metric;
    v.owned = vectors;
    v.vectors = v.owned.data();
    v.levels.clear();
    int64_t bottom;
    uint32_t ep;
    if (!entry_point(bottom, ep)) {
      v.empty_index = true;
      v.entry = UINT32_MAX;
      v.levels.resize(1);
      v.levels[0].identity = true;
      v.levels[0].row_ptr.assign(n_max + 1, 0);
      return;
    }
    v.empty_index = false;
    v.entry = ep;
    size_t nl = (size_t)(-bottom) + 1;
    v.levels.resize(nl);
    for (size_t L = 0; L < nl; ++L) {
      LevelView& lv = v.levels[L];
      auto li = rel.find(-(int64_t)L);
      if (L == 0) {
        lv.identity = true;
        lv.row_ptr.assign(n_max + 1, 0);
        if (li != rel.end())
          for (uint32_t i = 0; i < n_max; ++i) {
            auto ei = li->second.edges.find(i);
            if (ei != li->second.edges.end())
              for (auto& kv : ei->second)
                if (!kv.second.ignore_link) lv.col_idx.push_back(kv.first);
            lv.row_ptr[i + 1] = lv.col_idx.size();
          }
        else
          for (uint32_t i = 0; i < n_max; ++i) lv.row_ptr[i + 1] = 0;
      } else {
        lv.identity = false;
        lv.row_ptr.push_back(0);
        if (li != rel.end())
          for (auto& sd : li->second.self_degree) {
            lv.node_ids.push_back(sd.first);
            auto ei = li->second.edges.find(sd.first);
            if (ei != li->second.edges.end())
              for (auto& kv : ei->second)
                if (!kv.second.ignore_link) lv.col_idx.push_back(kv.first);
            lv.row_ptr.push_back(lv.col_idx.size());
          }
      }
    }
  }
};

// ---------------------------------------------------------------------------
// Graph side.  CSR as graph_builder 0.4.0 builds it with CsrLayout::Sorted
// (fixed_rule/mod.rs:192-195, 318-321): node_count = max id + 1, adjacency
// sorted by target, parallel edges kept.
// ---------------------------------------------------------------------------
struct Csr {
  uint32_t n = 0;
  std::vector<uint64_t> out_ptr, in_ptr;
  std::vector<uint32_t> out_idx, in_idx;
  std::vector<float> out_w;
};

static void build_csr(Csr& g, uint32_t n, uint64_t m, const uint32_t* src, const uint32_t* dst, const float* w) {
  g.n = n;
  g.out_ptr.assign((size_t)n + 1, 0);
  g.in_ptr.assign((size_t)n + 1, 0);
  for (uint64_t e = 0; e < m; ++e) {
    g.out_ptr[src[e] + 1]++;
    g.in_ptr[dst[e] + 1]++;
  }
  for (uint32_t i = 0; i < n; ++i) {
    g.out_ptr[i + 1] += g.out_ptr[i];
    g.in_ptr[i + 1] += g.in_ptr[i];
  }
  g.out_idx.resize(m);
  g.in_idx.resize(m);
  if (w) g.out_w.resize(m);
  std::vector<uint64_t> po(g.out_ptr.begin(), g.out_ptr.end() - 1), pi(g.in_ptr.begin(), g.in_ptr.end() - 1);
  for (uint64_t e = 0; e < m; ++e) {
    uint64_t o = po[src[e]]++;
    g.out_idx[o] = dst[e];
    if (w) g.out_w[o] = w[e];
    g.in_idx[pi[dst[e]]++] = src[e];
  }
  // Sorted layout: by target (stable w.r.t. input order for equal targets)
  std::vector<std::pair<uint32_t, float>> tmp;
  for (uint32_t i = 0; i < n; ++i) {
    uint64_t b = g.out_ptr[i], e = g.out_ptr[i + 1];
    if (w) {
      tmp.clear();
      for (uint64_t k = b; k < e; ++k) tmp.push_back({g.out_idx[k], g.out_w[k]});
      std::stable_sort(tmp.begin(), tmp.end(), [](auto& a, auto& b2) { return a.first < b2.first; });
      for (uint64_t k = b; k < e; ++k) {
        g.out_idx[k] = tmp[k - b].first;
        g.out_w[k] = tmp[k - b].second;
      }
    } else {
      std::sort(g.out_idx.begin() + b, g.out_idx.begin() + e);
    }
    std::sort(g.in_idx.begin() + g.in_ptr[i], g.in_idx.begin() + g.in_ptr[i + 1]);
  }
}

// a8. PageRank — fixed_rule/algos/pagerank.rs:47-50 calls graph::page_rank of
// the UN-VENDORED crate `graph 0.3.1` (Cargo.lock:1562-1575).  Its published
// algorithm is the GAP benchmark-suite pull PageRank: f32 scores, init 1/N,
// base (1-d)/N, no dangling redistribution, f64 L1 error, stop when
// error < tolerance or iteration == max_iterations.
//   variant 0 ("jacobi"): GAP pr (classic): contributions recomputed from the
//       previous iteration's scores at the start of every iteration.
//   variant 1 ("gs"): GAP PageRankPullGS: contribution of u overwritten in
//       place right after its score (chunks of 16384 nodes raced over by Rayon
//       workers in the crate; here executed in node order on one thread, which
//       is the crate's behaviour with RAYON_NUM_THREADS=1).
// Both share one fixed point; see DESIGN.md "PageRank parity".
static uint32_t pagerank(const Csr& g, float damping, double tol, uint32_t max_iter, int variant, float* scores,
                         double* out_err, unsigned n_threads) {
  const uint32_t n = g.n;
  if (n == 0) {
    *out_err = 0;
    return 0;
  }
  const float init = 1.0f / (float)n;
  const float base = (1.0f - damping) / (float)n;
  std::vector<float> contrib(n);
  for (uint32_t v = 0; v < n; ++v) {
    scores[v] = init;
    contrib[v] = init / (float)(g.out_ptr[v + 1] - g.out_ptr[v]);
  }
  uint32_t iter = 0;
  double err = 0;
  std::vector<float> next(variant == 0 ? n : 0);
  for (;;) {
    err = 0;
    if (variant == 1) {
      for (uint32_t u = 0; u < n; ++u) {
        float tot = 0.0f;
        for (uint64_t k = g.in_ptr[u]; k < g.in_ptr[u + 1]; ++k) tot += contrib[g.in_idx[k]];
        float old = scores[u];
        float nw = base + damping * tot;
        scores[u] = nw;
        err += (double)std::fabs(nw - old);
        contrib[u] = nw / (float)(g.out_ptr[u + 1] - g.out_ptr[u]);
      }
    } else {
      unsigned T = std::max(1u, n_threads);
      std::vector<double> errs(T, 0.0);
      auto work = [&](unsigned t) {
        uint32_t lo = (uint32_t)((uint64_t)n * t / T), hi = (uint32_t)((uint64_t)n * (t + 1) / T);
        double e = 0;
        for (uint32_t u = lo; u < hi; ++u) {
          float tot = 0.0f;
          for (uint64_t k = g.in_ptr[u]; k < g.in_ptr[u + 1]; ++k) tot += contrib[g.in_idx[k]];
          float nw = base + damping * tot;
          e += (double)std::fabs(nw - scores[u]);
          next[u] = nw;
        }
        errs[t] = e;
      };
      if (T == 1)
        work(0);
      else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < T; ++t) th.emplace_back(work, t);
        for (auto& x : th) x.join();
      }
      for (unsigned t = 0; t < T; ++t) err += errs[t];
      for (uint32_t u = 0; u < n; ++u) {
        scores[u] = next[u];
        contrib[u] = next[u] / (float)(g.out_ptr[u + 1] - g.out_ptr[u]);
      }
    }
    iter++;
    if (err < tol || iter == max_iter) break;
  }
  *out_err = err;
  return iter;
}

// a10. dijkstra_cost_only — all_pairs_shortest_path.rs:145-176
static void dijkstra_cost_only(const Csr& g, uint32_t start, float* distance) {
  for (uint32_t i = 0; i < g.n; ++i) distance[i] = INFINITY;
  MinPQ pq;
  distance[start] = 0.f;
  pq.push(start, 0.0);
  while (!pq.empty()) {
    auto [node, costd] = pq.pop();
    float cost = (float)costd;
    if (cost > distance[node]) continue;
    for (uint64_t k = g.out_ptr[node]; k < g.out_ptr[node + 1]; ++k) {
      uint32_t nx = g.out_idx[k];
      float nc = cost + g.out_w[k];  // f32 sum, :163
      if (nc < distance[nx]) {
        pq.push_decrease_cost(nx, (double)nc);
        distance[nx] = nc;
      }
    }
  }
}

// a10. dijkstra — shortest_path_dijkstra.rs:274-339.  goals == nullptr means
// Goal=() (all nodes, never exhausted); otherwise a set (BTreeSet / Option).
static void dijkstra(const Csr& g, uint32_t start, const std::set<uint32_t>* goals, float* distance,
                     uint32_t* back) {
  for (uint32_t i = 0; i < g.n; ++i) {
    distance[i] = INFINITY;
    back[i] = UINT32_MAX;
  }
  MinPQ pq;
  distance[start] = 0.f;
  pq.push(start, 0.0);
  std::set<uint32_t> remaining;
  if (goals) remaining = *goals;
  while (!pq.empty()) {
    auto [node, costd] = pq.pop();
    float cost = (float)costd;
    if (cost > distance[node]) continue;
    for (uint64_t k = g.out_ptr[node]; k < g.out_ptr[node + 1]; ++k) {
      uint32_t nx = g.out_idx[k];
      float nc = cost + g.out_w[k];
      if (nc < distance[nx]) {  // strict, :305
        pq.push_decrease_cost(nx, (double)nc);
        distance[nx] = nc;
        back[nx] = node;
      }
    }
    if (goals) {  // :312-315
      remaining.erase(node);
      if (remaining.empty()) break;
    }
  }
}

// dijkstra with ForbiddenEdge / ForbiddenNode sets and a single Option<u32> goal, as
// KShortestPathYen calls it (yen.rs:138, 168; shortest_path_dijkstra.rs:188-218, 274-339).
// Returns the (goal, cost, path) triple of `.into_iter().next()`.
static void dijkstra_forbidden(const Csr& g, uint32_t start, uint32_t goal,
                               const std::set<std::pair<uint32_t, uint32_t>>& fe, const std::set<uint32_t>& fn,
                               float& cost_out, std::vector<uint32_t>& path_out) {
  std::vector<float> distance(g.n, INFINITY);
  std::vector<uint32_t> back(g.n, UINT32_MAX);
  MinPQ pq;
  distance[start] = 0.f;
  pq.push(start, 0.0);
  bool goal_left = true;
  while (!pq.empty()) {
    auto [node, costd] = pq.pop();
    float cost = (float)costd;
    if (cost > distance[node]) continue;
    for (uint64_t k = g.out_ptr[node]; k < g.out_ptr[node + 1]; ++k) {
      uint32_t nx = g.out_idx[k];
      if (fn.count(nx)) continue;          // :298-300
      if (fe.count({node, nx})) continue;  // :301-303
      float nc = cost + g.out_w[k];
      if (nc < distance[nx]) {
        pq.push_decrease_cost(nx, (double)nc);
        distance[nx] = nc;
        back[nx] = node;
      }
    }
    if (node == goal) goal_left = false;  // Goal for Option<u32>, :238-258
    if (!goal_left) break;
  }
  cost_out = distance[goal];
  path_out.clear();
  if (!std::isfinite(cost_out)) return;  // (target, inf, [])
  uint32_t cur = goal;
  while (cur != start) {
    path_out.push_back(cur);
    cur = back[cur];
  }
  path_out.push_back(start);
  std::reverse(path_out.begin(), path_out.end());
}

// k_shortest_path_yen — fixed_rule/algos/yen.rs:120-211, quirks included (unreachable spur
// results enter `candidates` with infinite cost and a truncated path; only finite ones are kept).
static std::vector<std::pair<float, std::vector<uint32_t>>> k_shortest_path_yen(const Csr& g, size_t k, uint32_t start,
                                                                                uint32_t goal) {
  std::vector<std::pair<float, std::vector<uint32_t>>> k_shortest, candidates;
  {
    float c;
    std::vector<uint32_t> p;
    dijkstra_forbidden(g, start, goal, {}, {}, c, p);
    k_shortest.push_back({c, p});  // yen.rs:130-136 (the goal iterator always yields one triple)
  }
  for (size_t it = 1; it < k; ++it) {
    const std::vector<uint32_t> prev_path = k_shortest.back().second;
    for (size_t i = 0; i + 1 < prev_path.size(); ++i) {  // 0..prev_path.len()-1, yen.rs:140
      uint32_t spur_node = prev_path[i];
      std::vector<uint32_t> root_path(prev_path.begin(), prev_path.begin() + i + 1);
      std::set<std::pair<uint32_t, uint32_t>> fe;
      for (auto& cp : k_shortest) {  // yen.rs:147-155
        const auto& p = cp.second;
        if (p.size() < root_path.size() + 1) continue;
        if (std::equal(root_path.begin(), root_path.end(), p.begin())) fe.insert({p[i], p[i + 1]});
      }
      std::set<uint32_t> fn(prev_path.begin(), prev_path.begin() + i);  // yen.rs:156-159
      float spur_cost;
      std::vector<uint32_t> spur_path;
      dijkstra_forbidden(g, spur_node, goal, fe, fn, spur_cost, spur_path);
      float total_cost = spur_cost;
      for (size_t j = 0; j + 1 < root_path.size(); ++j) {  // yen.rs:171-183: first edge s->d in adjacency order
        uint32_t sN = root_path[j], dN = root_path[j + 1];
        for (uint64_t e = g.out_ptr[sN]; e < g.out_ptr[sN + 1]; ++e)
          if (g.out_idx[e] == dN) {
            total_cost += g.out_w[e];
            break;
          }
      }
      std::vector<uint32_t> total_path(root_path.begin(), root_path.end() - 1);
      total_path.insert(total_path.end(), spur_path.begin(), spur_path.end());
      bool dup = false;
      for (auto& c : candidates)
        if (c.second == total_path) dup = true;
      if (!dup) candidates.push_back({total_cost, total_path});  // yen.rs:187-189
    }
    if (candidates.empty()) break;
    // sort_by(|a,b| b.total_cmp(a)) then pop(): the smallest cost; stable sort keeps insertion order of ties
    std::stable_sort(candidates.begin(), candidates.end(), [](const auto& a, const auto& b) {
      // total_cmp on f32: order by bits with sign handling; costs are >= 0 or +inf/NaN-free here
      return b.first < a.first;
    });
    auto shortest = candidates.back();
    candidates.pop_back();
    if (std::isfinite(shortest.first)) k_shortest.push_back(shortest);  // yen.rs:205-207
  }
  return k_shortest;
}

// a10. dijkstra_keep_ties — shortest_path_dijkstra.rs:341-432 (search part).
// back-pointer lists are returned CSR-style.  A settled node that is re-pushed
// through an equal-cost relaxation (possible only with zero-weight edges) is
// re-expanded by the reference; a pop budget guards the zero-weight-cycle
// non-termination of the reference.
static int dijkstra_keep_ties(const Csr& g, uint32_t start, const std::set<uint32_t>* goals, float* distance,
                              std::vector<std::vector<uint32_t>>& back) {
  back.assign(g.n, {});
  for (uint32_t i = 0; i < g.n; ++i) distance[i] = INFINITY;
  MinPQ pq;
  distance[start] = 0.f;
  pq.push(start, 0.0);
  std::set<uint32_t> remaining;
  if (goals) remaining = *goals;
  uint64_t pops = 0, budget = 64ull * (g.out_idx.size() + g.n + 16);
  while (!pq.empty()) {
    if (++pops > budget) return -1;
    auto [node, costd] = pq.pop();
    float cost = (float)costd;
    if (cost > distance[node]) continue;
    for (uint64_t k = g.out_ptr[node]; k < g.out_ptr[node + 1]; ++k) {
      uint32_t nx = g.out_idx[k];
      float nc = cost + g.out_w[k];
      if (nc < distance[nx]) {
        pq.push_decrease_cost(nx, (double)nc);
        distance[nx] = nc;
        back[nx].clear();
        back[nx].push_back(node);
      } else if (nc == distance[nx]) {  // :377-380
        pq.push_decrease_cost(nx, (double)nc);
        back[nx].push_back(node);
      }
    }
    if (goals) {
      remaining.erase(node);
      if (remaining.empty()) break;
    }
  }
  return 0;
}

// path enumeration of keep_ties — shortest_path_dijkstra.rs:397-426
static void collect_paths(std::vector<uint32_t>& chain, uint32_t start, const std::vector<std::vector<uint32_t>>& back,
                          std::vector<std::vector<uint32_t>>& out, size_t cap) {
  if (out.size() >= cap) return;
  uint32_t last = chain.back();
  for (uint32_t nxt : back[last]) {
    chain.push_back(nxt);
    if (nxt == start) {
      std::vector<uint32_t> r(chain.rbegin(), chain.rend());
      out.push_back(std::move(r));
    } else {
      collect_paths(chain, start, back, out, cap);
    }
    chain.pop_back();
    if (out.size() >= cap) return;
  }
}

struct GraphHandle {
  Csr g;
};

struct HnswHandle {
  HnswBuilder* b = nullptr;
  HnswView view;
  bool view_valid = false;
  void ensure_view() {
    if (b && !view_valid) {
      b->to_view(view);
      view_valid = true;
    }
  }
};

template <class F>
static void parallel_for(uint32_t n, unsigned T, F f) {
  T = std::max(1u, std::min<unsigned>(T, n ? n : 1));
  if (T == 1) {
    for (uint32_t i = 0; i < n; ++i) f(i, 0u);
    return;
  }
  std::atomic<uint32_t> next{0};
  std::vector<std::thread> th;
  for (unsigned t = 0; t < T; ++t)
    th.emplace_back([&, t] {
      for (;;) {
        uint32_t i = next.fetch_add(1);
        if (i >= n) break;
        f(i, t);
      }
    });
  for (auto& x : th) x.join();
}

}  // namespace

// ===========================================================================
// C entry points (ctypes).  All ids are dense u32; level L >= 0 == layer -L.
// ===========================================================================
extern "C" {

double orc_vec_dist(int metric, const float* a, const float* b, uint32_t n) { return vec_dist(metric, a, b, n); }

// -- HNSW builder ----------------------------------------------------------
void* orc_hnsw_new(uint32_t n_max, uint32_t dim, int metric, uint32_t m, uint32_t ef_construction,
                   int extend_candidates, int keep_pruned, uint64_t level_seed) {
  auto* h = new HnswHandle();
  auto* b = new HnswBuilder();
  b->dim = dim;
  b->n_max = n_max;
  b->metric = metric;
  b->m = m;
  b->m_max = m;
  b->m_max0 = 2 * m;
  b->ef_construction = ef_construction;
  b->level_multiplier = 1.0 / std::log((double)m);
  b->extend_candidates = extend_candidates != 0;
  b->keep_pruned = keep_pruned != 0;
  b->rng.s = level_seed;
  b->vectors.assign((size_t)n_max * dim, 0.f);
  b->present.assign(n_max, 0);
  h->b = b;
  return h;
}

// forced_level: <= 0 forces that layer, > 0 draws from the seeded RNG.
int orc_hnsw_insert(void* hp, uint32_t id, const float* v, int64_t forced_level) {
  auto* h = (HnswHandle*)hp;
  if (!h->b) return -2;
  h->view_valid = false;
  return h->b->insert(id, v, forced_level);
}

int orc_hnsw_remove(void* hp, uint32_t id) {
  auto* h = (HnswHandle*)hp;
  if (!h->b) return -2;
  h->view_valid = false;
  h->b->remove(id);
  return 0;
}

uint64_t orc_hnsw_build_dist_evals(void* hp) {
  auto* h = (HnswHandle*)hp;
  return h->b ? h->b->dist_evals : 0;
}

// Raw rows of the index relation (runtime/relation.rs:1064-1126) in key order, for tests of
// the host-side stager: self-loop rows (fr == to, value = degree), live and soft-deleted
// edge rows.  The canary row (1, Null..) is added by the caller.  Returns the row count;
// arrays may be NULL to size them.
uint64_t orc_hnsw_relation_rows(void* hp, int64_t* layer, uint32_t* fr, uint32_t* to, double* dist,
                                uint8_t* ignore_link) {
  auto* h = (HnswHandle*)hp;
  if (!h->b) return 0;
  uint64_t c = 0;
  for (auto& lr : h->b->rel) {  // most negative layer first
    const LevelRel& L = lr.second;
    for (auto& sd : L.self_degree) {
      const uint32_t node = sd.first;
      auto ei = L.edges.find(node);
      bool self_done = false;
      auto emit_self = [&] {
        if (layer) {
          layer[c] = lr.first;
          fr[c] = node;
          to[c] = node;
          dist[c] = sd.second;
          ignore_link[c] = 0;
        }
        ++c;
        self_done = true;
      };
      if (ei != L.edges.end())
        for (auto& kv : ei->second) {
          if (!self_done && kv.first > node) emit_self();
          if (layer) {
            layer[c] = lr.first;
            fr[c] = node;
            to[c] = kv.first;
            dist[c] = kv.second.dist;
            ignore_link[c] = kv.second.ignore_link ? 1 : 0;
          }
          ++c;
        }
      if (!self_done) emit_self();
    }
  }
  return c;
}

// -- read-only view from flat arrays (to search graphs built elsewhere) ------
// level_nodes[L]: n rows on level L; node_ids[L] NULL for level 0 (identity).
void* orc_hnsw_from_csr(uint32_t n, uint32_t dim, int metric, const float* vectors, int copy_vectors,
                        uint32_t n_levels, const uint32_t* level_nodes, const uint32_t* const* node_ids,
                        const uint64_t* const* row_ptr, const uint32_t* const* col_idx, uint32_t entry) {
  auto* h = new HnswHandle();
  HnswView& v = h->view;
  v.n = n;
  v.dim = dim;
  v.metric = metric;
  if (copy_vectors) {
    v.owned.assign(vectors, vectors + (size_t)n * dim);
    v.vectors = v.owned.data();
  } else {
    v.vectors = vectors;
  }
  v.levels.resize(n_levels);
  for (uint32_t L = 0; L < n_levels; ++L) {
    LevelView& lv = v.levels[L];
    uint32_t rows = level_nodes[L];
    lv.identity = (L == 0);
    if (!lv.identity) lv.node_ids.assign(node_ids[L], node_ids[L] + rows);
    lv.row_ptr.assign(row_ptr[L], row_ptr[L] + rows + 1);
    lv.col_idx.assign(col_idx[L], col_idx[L] + lv.row_ptr[rows]);
  }
  v.entry = entry;
  v.empty_index = (entry == UINT32_MAX);
  h->view_valid = true;
  return h;
}

void orc_hnsw_free(void* hp) {
  auto* h = (HnswHandle*)hp;
  delete h->b;
  delete h;
}

uint32_t orc_hnsw_n_levels(void* hp) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  return (uint32_t)h->view.levels.size();
}
uint32_t orc_hnsw_entry(void* hp) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  return h->view.entry;
}
void orc_hnsw_level_size(void* hp, uint32_t L, uint32_t* n_rows, uint64_t* n_edges) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  *n_rows = h->view.levels[L].n_rows();
  *n_edges = h->view.levels[L].col_idx.size();
}
void orc_hnsw_export_level(void* hp, uint32_t L, uint32_t* node_ids, uint64_t* row_ptr, uint32_t* col_idx) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  const LevelView& lv = h->view.levels[L];
  if (node_ids) {
    if (lv.identity)
      for (uint32_t i = 0; i < lv.n_rows(); ++i) node_ids[i] = i;
    else
      std::copy(lv.node_ids.begin(), lv.node_ids.end(), node_ids);
  }
  std::copy(lv.row_ptr.begin(), lv.row_ptr.end(), row_ptr);
  std::copy(lv.col_idx.begin(), lv.col_idx.end(), col_idx);
}
const float* orc_hnsw_vectors(void* hp) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  return h->view.vectors;
}

// -- F64 index: the same graph, f64 payloads and queries (manifest.dtype == F64, hnsw.rs:879-884) -------------
int orc_hnsw_search_batch_f64(void* hp, const double* vectors64, const double* queries, uint32_t B, uint32_t k,
                              uint32_t ef, double radius, uint32_t* out_ids, double* out_dist, uint32_t* out_count,
                              uint64_t* stats, uint32_t n_threads) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  const HnswView& ix = h->view;
  parallel_for(B, n_threads, [&](uint32_t qi, unsigned) {
    SearchStats st;
    uint32_t* ids = out_ids + (size_t)qi * k;
    double* ds = out_dist + (size_t)qi * k;
    for (uint32_t j = 0; j < k; ++j) {
      ids[j] = UINT32_MAX;
      ds[j] = INFINITY;
    }
    const double* q = queries + (size_t)qi * ix.dim;
    uint32_t c = hnsw_knn_with(
        ix, [&](uint32_t id) { return vec_dist64(ix.metric, q, vectors64 + (size_t)id * ix.dim, ix.dim); }, k, ef, radius,
        radius >= 0, ids, ds, st);
    if (out_count) out_count[qi] = c;
    if (stats) {
      stats[(size_t)qi * 3 + 0] = st.dist_evals;
      stats[(size_t)qi * 3 + 1] = st.nodes_expanded;
      stats[(size_t)qi * 3 + 2] = st.nbr_reads;
    }
  });
  return 0;
}

// -- search -------------------------------------------------------------------
// radius < 0 => no radius.  stats: [B x 3] dist_evals, nodes_expanded, nbr_reads
// (nullable).  out_ids padded with UINT32_MAX, out_dist with +inf.
int orc_hnsw_search_batch(void* hp, const float* queries, uint32_t B, uint32_t k, uint32_t ef, double radius,
                          uint32_t* out_ids, double* out_dist, uint32_t* out_count, uint64_t* stats,
                          uint32_t n_threads) {
  auto* h = (HnswHandle*)hp;
  h->ensure_view();
  const HnswView& ix = h->view;
  parallel_for(B, n_threads, [&](uint32_t qi, unsigned) {
    SearchStats st;
    uint32_t* ids = out_ids + (size_t)qi * k;
    double* ds = out_dist + (size_t)qi * k;
    for (uint32_t j = 0; j < k; ++j) {
      ids[j] = UINT32_MAX;
      ds[j] = INFINITY;
    }
    uint32_t c = hnsw_knn(ix, queries + (size_t)qi * ix.dim, k, ef, radius, radius >= 0, ids, ds, st);
    if (out_count) out_count[qi] = c;
    if (stats) {
      stats[(size_t)qi * 3 + 0] = st.dist_evals;
      stats[(size_t)qi * 3 + 1] = st.nodes_expanded;
      stats[(size_t)qi * 3 + 2] = st.nbr_reads;
    }
  });
  return 0;
}

// exact brute-force k-NN with the same distance function (context recall only)
int orc_bruteforce_knn(const float* vectors, uint32_t n, uint32_t dim, int metric, const float* queries, uint32_t B,
                       uint32_t k, uint32_t* out_ids, double* out_dist, uint32_t n_threads) {
  parallel_for(B, n_threads, [&](uint32_t qi, unsigned) {
    std::vector<std::pair<double, uint32_t>> d(n);
    for (uint32_t i = 0; i < n; ++i)
      d[i] = {vec_dist(metric, queries + (size_t)qi * dim, vectors + (size_t)i * dim, dim), i};
    uint32_t kk = std::min(k, n);
    std::partial_sort(d.begin(), d.begin() + kk, d.end());
    for (uint32_t j = 0; j < k; ++j) {
      out_ids[(size_t)qi * k + j] = j < kk ? d[j].second : UINT32_MAX;
      out_dist[(size_t)qi * k + j] = j < kk ? d[j].first : INFINITY;
    }
  });
  return 0;
}

// -- graphs ---------------------------------------------------------------------
void* orc_graph_new(uint32_t n, uint64_t m, const uint32_t* src, const uint32_t* dst, const float* w) {
  auto* h = new GraphHandle();
  build_csr(h->g, n, m, src, dst, w);
  return h;
}
void orc_graph_free(void* gp) { delete (GraphHandle*)gp; }

void orc_graph_export(void* gp, uint64_t* out_ptr, uint32_t* out_idx, float* out_w, uint64_t* in_ptr,
                      uint32_t* in_idx) {
  const Csr& g = ((GraphHandle*)gp)->g;
  if (out_ptr) std::copy(g.out_ptr.begin(), g.out_ptr.end(), out_ptr);
  if (out_idx) std::copy(g.out_idx.begin(), g.out_idx.end(), out_idx);
  if (out_w && !g.out_w.empty()) std::copy(g.out_w.begin(), g.out_w.end(), out_w);
  if (in_ptr) std::copy(g.in_ptr.begin(), g.in_ptr.end(), in_ptr);
  if (in_idx) std::copy(g.in_idx.begin(), g.in_idx.end(), in_idx);
}

uint32_t orc_pagerank(void* gp, float damping, double tol, uint32_t max_iter, int variant, float* scores,
                      double* out_err, uint32_t n_threads) {
  return pagerank(((GraphHandle*)gp)->g, damping, tol, max_iter, variant, scores, out_err, n_threads);
}

// multi-source SSSP; out_dist [n_src x n], out_back [n_src x n] (nullable).
// goals: nullable; when given, each search stops once all goals are settled
// (distances of unsettled nodes are then tentative, exactly as the reference).
int orc_sssp(void* gp, const uint32_t* sources, uint32_t n_src, const uint32_t* goals, uint32_t n_goals,
             float* out_dist, uint32_t* out_back, uint32_t n_threads) {
  const Csr& g = ((GraphHandle*)gp)->g;
  std::set<uint32_t> gs;
  if (goals) gs.insert(goals, goals + n_goals);
  parallel_for(n_src, n_threads, [&](uint32_t si, unsigned) {
    std::vector<uint32_t> tmp;
    uint32_t* back = out_back ? out_back + (size_t)si * g.n : (tmp.resize(g.n), tmp.data());
    dijkstra(g, sources[si], goals ? &gs : nullptr, out_dist + (size_t)si * g.n, back);
  });
  return 0;
}

// keep_ties SSSP for one source; predecessor lists returned CSR-style through
// caller buffers sized by a first call with back_idx == NULL (returns count).
int64_t orc_sssp_keep_ties(void* gp, uint32_t source, const uint32_t* goals, uint32_t n_goals, float* out_dist,
                           uint64_t* back_ptr, uint32_t* back_idx) {
  const Csr& g = ((GraphHandle*)gp)->g;
  std::set<uint32_t> gs;
  if (goals) gs.insert(goals, goals + n_goals);
  std::vector<std::vector<uint32_t>> back;
  if (dijkstra_keep_ties(g, source, goals ? &gs : nullptr, out_dist, back) != 0) return -1;
  uint64_t tot = 0;
  for (uint32_t i = 0; i < g.n; ++i) {
    if (back_ptr) back_ptr[i] = tot;
    if (back_idx)
      for (uint32_t p : back[i]) back_idx[tot++] = p;
    else
      tot += back[i].size();
  }
  if (back_ptr) back_ptr[g.n] = tot;
  return (int64_t)tot;
}

// a11. ClosenessCentrality — all_pairs_shortest_path.rs:97-143
int orc_closeness(void* gp, float* out, uint32_t n_threads) {
  const Csr& g = ((GraphHandle*)gp)->g;
  const uint32_t n = g.n;
  unsigned T = std::max(1u, n_threads);
  std::vector<std::vector<float>> buf(T, std::vector<float>(n));
  parallel_for(n, T, [&](uint32_t start, unsigned t) {
    float* d = buf[t].data();
    dijkstra_cost_only(g, start, d);
    float total = 0.f, nc = 0.f;  // f32 sums in node order, :118-119
    for (uint32_t i = 0; i < n; ++i)
      if (std::isfinite(d[i])) total += d[i];
    size_t cnt = 0;
    for (uint32_t i = 0; i < n; ++i)
      if (std::isfinite(d[i])) cnt++;
    nc = (float)cnt;
    out[start] = nc * nc / total / (float)(n - 1);  // :120
  });
  return 0;
}

// a11. BetweennessCentrality — all_pairs_shortest_path.rs:29-95
// path_cap bounds tied-path enumeration per (source,target) (reference: unbounded).
int orc_betweenness(void* gp, float* out, uint32_t n_threads, uint64_t path_cap) {
  const Csr& g = ((GraphHandle*)gp)->g;
  const uint32_t n = g.n;
  std::vector<std::map<uint32_t, float>> segs(n);
  std::atomic<int> bad{0};
  unsigned T = std::max(1u, n_threads);
  std::vector<std::vector<float>> dbuf(T, std::vector<float>(n));
  parallel_for(n, T, [&](uint32_t start, unsigned t) {
    std::vector<std::vector<uint32_t>> back;
    float* dist = dbuf[t].data();
    if (dijkstra_keep_ties(g, start, nullptr, dist, back) != 0) {
      bad = 1;
      return;
    }
    std::map<uint32_t, float>& ret = segs[start];
    for (uint32_t target = 0; target < n; ++target) {  // Goal=() iterates 0..n, :233-235
      if (!std::isfinite(dist[target])) continue;       // one (target, inf, []) row: len<3
      std::vector<std::vector<uint32_t>> paths;
      std::vector<uint32_t> chain{target};
      collect_paths(chain, start, back, paths, path_cap);
      float l = (float)paths.size();  // :58
      for (auto& p : paths) {
        if (p.size() < 3) continue;
        for (size_t i = 1; i + 1 < p.size(); ++i) ret[p[i]] += 1.f / l;  // :63-66
      }
    }
  });
  if (bad) return -1;
  for (uint32_t i = 0; i < n; ++i) out[i] = 0.f;
  for (uint32_t s = 0; s < n; ++s)  // serial merge in source order, :72-77
    for (auto& kv : segs[s]) out[kv.first] += kv.second;
  return 0;
}

// ClusteringCoefficients — fixed_rule/algos/triangles.rs:59-98 over the graph of
// as_directed_graph(undirected = true) (triangles.rs:35).  `edges` is the out-neighbour list WITH
// duplicates; a pair of positions (e_src, e_dst) counts when e_src > e_dst by value and e_dst
// occurs among the out-neighbours of e_src.  The reference scans that list linearly; a binary
// search over the sorted adjacency answers the same membership question.
int orc_clustering(void* gp, double* cc, uint64_t* n_triangles, uint64_t* degree, uint32_t n_threads) {
  const Csr& g = ((GraphHandle*)gp)->g;
  parallel_for(g.n, n_threads, [&](uint32_t u, unsigned) {
    const uint32_t* e = g.out_idx.data() + g.out_ptr[u];
    const uint64_t deg = g.out_ptr[u + 1] - g.out_ptr[u];
    degree[u] = deg;
    if (deg < 2) {  // triangles.rs:72-73
      cc[u] = 0.0;
      n_triangles[u] = 0;
      return;
    }
    uint64_t t = 0;
    for (uint64_t i = 0; i < deg; ++i) {
      const uint32_t a = e[i];
      const uint32_t* ab = g.out_idx.data() + g.out_ptr[a];
      const uint32_t* ae = g.out_idx.data() + g.out_ptr[a + 1];
      for (uint64_t j = 0; j < deg; ++j) {
        const uint32_t b = e[j];
        if (a <= b) continue;  // triangles.rs:80-82
        if (std::binary_search(ab, ae, b)) ++t;
      }
    }
    n_triangles[u] = t;
    cc[u] = 2. * (double)t / ((double)deg * ((double)deg - 1.));  // triangles.rs:93
  });
  return 0;
}

// KShortestPathYen for one (start, goal) pair.  out_cost [k], path_ptr [k+1], path_buf sized by a
// first call with path_buf == NULL (returns total path length via *n_path_elems).
int orc_yen(void* gp, uint32_t start, uint32_t goal, uint32_t k, float* out_cost, uint64_t* path_ptr,
            uint32_t* path_buf, uint64_t* n_path_elems) {
  const Csr& g = ((GraphHandle*)gp)->g;
  auto res = k_shortest_path_yen(g, k, start, goal);
  uint64_t tot = 0;
  for (size_t i = 0; i < res.size(); ++i) {
    if (out_cost) out_cost[i] = res[i].first;
    if (path_ptr) path_ptr[i] = tot;
    for (uint32_t u : res[i].second) {
      if (path_buf) path_buf[tot] = u;
      ++tot;
    }
  }
  if (path_ptr) path_ptr[res.size()] = tot;
  if (n_path_elems) *n_path_elems = tot;
  return (int)res.size();
}

// seeded level law shared with tests (hnsw.rs:46-52 with a SplitMix64 uniform)
int64_t orc_random_level(uint64_t* state, uint32_t m) {
  SplitMix64 r{*state};
  double u = r.uniform();
  *state = r.s;
  double x = -std::log(u) * (1.0 / std::log((double)m));
  if (!(x < 1e6)) x = 1e6;
  return -(int64_t)std::floor(x);
}

}  // extern "C"
