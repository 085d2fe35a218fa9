// hnsw.hpp — host side of the HNSW operator: staging the index *relation* into the
// device layout, SessionTx::hnsw_knn's row assembly, and the HnswSearchRA operator that
// collects parent tuples, launches one batched search and scatters the results.
//
// Mirrors (same names / argument meaning / error behaviour):
//   HnswIndexManifest                    runtime/hnsw.rs:27-43, runtime/relation.rs:1136-1151
//   index relation schema                runtime/relation.rs:1064-1126 (SURVEY.md appendix A)
//   hnsw_get_neighbours reading rules    runtime/hnsw.rs:588-629
//   SessionTx::hnsw_knn                  runtime/hnsw.rs:869-1012
//   HnswSearch / all_bindings            data/program.rs:976-991, 1016-1025
//   HnswSearchRA::iter                   query/ra.rs:1085-1121
#pragma once
#include <algorithm>
#include <climits>
#include <functional>
#include <map>
#include <optional>
#include <thread>

#include "fixed_rule.hpp"
#include "memcmp.hpp"
#include "msgpack.hpp"

namespace cozo_host {

enum class HnswDistance { L2 = COZO_GPU_L2, Cosine = COZO_GPU_COSINE, InnerProduct = COZO_GPU_IP };  // sys.rs:94-98

struct HnswIndexManifest {  // hnsw.rs:27-43
  std::string base_relation, index_name;
  size_t vec_dim = 0;
  bool dtype_f64 = false;          // VecElementType::F64 is outside the device envelope
  std::vector<size_t> vec_fields;  // column indices of the base relation holding vectors
  HnswDistance distance = HnswDistance::L2;
  size_t ef_construction = 0, m_neighbours = 0, m_max = 0, m_max0 = 0;
  double level_multiplier = 0;
  bool extend_candidates = false, keep_pruned_connections = false;
  // relation.rs:1145-1147
  void derive() {
    m_max = m_neighbours;
    m_max0 = m_neighbours * 2;
    level_multiplier = 1.0 / std::log((double)m_neighbours);
  }
};

// A stored relation as the operator sees it: key columns then value columns, rows in key order.
struct RelationHandle {
  std::string name;
  std::vector<std::string> keys, non_keys;  // column names
  std::map<Tuple, Tuple, TupleLess> rows;   // key tuple -> full row (keys ++ values)
  void put(const Tuple& full) {
    Tuple k(full.begin(), full.begin() + keys.size());
    rows[k] = full;
  }
  const Tuple* get(const Tuple& key) const {
    auto it = rows.find(key);
    return it == rows.end() ? nullptr : &it->second;
  }
  bool erase(const Tuple& key) { return rows.erase(key) > 0; }
};

// The same relation as the storage layer holds it: (key bytes, value bytes) pairs in memcmp order —
// what StoreTx::range_scan yields for one relation id (storage/mod.rs; runtime/relation.rs:247-296).
struct KvRelation {
  uint64_t id = 0;
  size_t n_keys = 0;
  std::vector<std::pair<std::string, std::string>> kv;  // ascending key bytes

  // encode_key_for_store / encode_val_for_store over every row of a RelationHandle
  static KvRelation encode(const RelationHandle& rel, uint64_t id) {
    KvRelation r;
    r.id = id;
    r.n_keys = rel.keys.size();
    r.kv.reserve(rel.rows.size());
    for (auto& row : rel.rows)
      r.kv.emplace_back(memcmp_codec::encode_as_key(row.first, id), msgpack_codec::encode_vals(row.second, r.n_keys, id));
    // storage order = byte order of the memcmp keys.  For Null/Bool/Num/Str/Bytes/List keys it equals DataValue
    // order; for Vec keys it does not (VEC_TAG 0x04 sorts before numbers, elements are raw BE bits) — the byte-level
    // planner (plan_kv_bytes) follows storage order like the reference's scans do (hnsw.rs:891-899)
    std::sort(r.kv.begin(), r.kv.end());
    return r;
  }
  const std::string* get_val_bytes(const std::string& k) const {
    auto it = std::lower_bound(kv.begin(), kv.end(), k,
                               [](const std::pair<std::string, std::string>& a, const std::string& b) { return a.first < b; });
    return (it != kv.end() && it->first == k) ? &it->second : nullptr;
  }
  // point read: RelationHandle::get (relation.rs:398-417)
  const std::string* get_val(const Tuple& key) const {
    const std::string k = memcmp_codec::encode_as_key(key, id);
    auto it = std::lower_bound(kv.begin(), kv.end(), k,
                               [](const std::pair<std::string, std::string>& a, const std::string& b) { return a.first < b; });
    return (it != kv.end() && it->first == k) ? &it->second : nullptr;
  }
};

// decode_tuple_from_kv (relation.rs:520-524)
inline Tuple decode_tuple_from_kv(const std::string& key, const std::string& val) {
  Tuple t = memcmp_codec::decode_tuple_from_key(key);
  msgpack_codec::extend_tuple_from_v(t, val);
  return t;
}

using CompoundKey = std::tuple<Tuple, size_t, int32_t>;  // hnsw.rs:55
struct CompoundKeyLess {
  bool operator()(const CompoundKey& a, const CompoundKey& b) const {
    int c = cmp_tuple(std::get<0>(a), std::get<0>(b));
    if (c) return c < 0;
    if (std::get<1>(a) != std::get<1>(b)) return std::get<1>(a) < std::get<1>(b);
    return std::get<2>(a) < std::get<2>(b);
  }
};

// SHA-256 (FIPS 180-4) of a vector's little-endian element bytes: Vector::get_hash (data/value.rs:333-348),
// the `hash` column of the self-loop rows (hnsw.rs:168, 237-241).
inline std::string sha256_le_f32(const std::vector<float>& v) {
  static const uint32_t K[64] = {
      0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98,
      0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786,
      0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8,
      0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13,
      0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819,
      0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a,
      0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7,
      0xc67178f2};
  std::string msg(reinterpret_cast<const char*>(v.data()), v.size() * 4);  // x86-64: already little endian
  const uint64_t bitlen = (uint64_t)msg.size() * 8;
  msg.push_back((char)0x80);
  while (msg.size() % 64 != 56) msg.push_back(0);
  for (int i = 7; i >= 0; --i) msg.push_back((char)((bitlen >> (8 * i)) & 0xff));
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  auto rotr = [](uint32_t x, int n) { return (x >> n) | (x << (32 - n)); };
  for (size_t off = 0; off < msg.size(); off += 64) {
    uint32_t w[64];
    for (int i = 0; i < 16; ++i)
      w[i] = ((uint32_t)(uint8_t)msg[off + 4 * i] << 24) | ((uint32_t)(uint8_t)msg[off + 4 * i + 1] << 16) |
             ((uint32_t)(uint8_t)msg[off + 4 * i + 2] << 8) | (uint32_t)(uint8_t)msg[off + 4 * i + 3];
    for (int i = 16; i < 64; ++i) {
      uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
      uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
      w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int i = 0; i < 64; ++i) {
      uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
      uint32_t ch = (e & f) ^ (~e & g);
      uint32_t t1 = hh + S1 + ch + K[i] + w[i];
      uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
      uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
      uint32_t t2 = S0 + mj;
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  }
  std::string out(32, 0);
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 4; ++j) out[4 * i + j] = (char)((h[i] >> (24 - 8 * j)) & 0xff);
  return out;
}

// Everything cozo_gpu_hnsw_stage needs, as plain host arrays: the product of reading `rel:idx` (+ the
// vectors of `rel`).  Two producers — from decoded tuples (plan_with) and straight from KV bytes
// (plan_kv_bytes) — must agree element for element; tests/test_stage_plan_cpu.py holds them to that.
struct StagePlan {
  std::vector<CompoundKey> keys;  // dense id -> compound key (key order)
  uint32_t entry = COZO_GPU_NONE, n_levels = 1;
  std::vector<std::vector<uint32_t>> node_ids, col_idx;  // per level (node_ids[0] stays empty: all nodes)
  std::vector<std::vector<uint64_t>> row_ptr;
  std::vector<float> vectors;
  uint64_t n_edges_kept = 0, n_rows_dropped_same_key = 0, n_rows_dropped_ignored = 0;
};

// The device-resident copy of one index: a cache of the index relation.
struct StagedHnswIndex {
  cozo_gpu_hnsw_t* h = nullptr;
  std::vector<CompoundKey> keys;  // dense id -> compound key (key order)
  HnswIndexManifest manifest;
  uint64_t n_edges_kept = 0, n_rows_dropped_same_key = 0, n_rows_dropped_ignored = 0;
  StagedHnswIndex() = default;
  StagedHnswIndex(const StagedHnswIndex&) = delete;
  StagedHnswIndex& operator=(const StagedHnswIndex&) = delete;
  ~StagedHnswIndex() {
    if (h) cozo_gpu_hnsw_free(h);
  }

  // idx_rows: scan_all of the index relation, i.e. tuples
  //   (layer, fr_k.., fr__field, fr__sub_idx, to_k.., to__field, to__sub_idx, dist, hash, ignore_link)
  // in key order (relation.rs:1064-1126).  K = number of key columns of the base relation.
  void stage(const RelationHandle& base, std::vector<Tuple> idx_rows, const HnswIndexManifest& mf) {
    stage_with(base.keys.size(), std::move(idx_rows), mf, [&](const CompoundKey& ck, float* out) {
      const Tuple* row = base.get(std::get<0>(ck));
      if (!row) throw CozoError("", "Cannot find compound key for HNSW");
      const DataValue* field = &(*row)[std::get<1>(ck)];
      if (std::get<2>(ck) >= 0) {
        if (field->kind != DataValue::List) throw CozoError("", "Cannot interpret " + field->repr() + " as list");
        field = &field->list[(size_t)std::get<2>(ck)];
      }
      if (field->kind != DataValue::Vec || field->v->size() != mf.vec_dim)
        throw CozoError("", "Cannot interpret " + field->repr() + " as vector");
      std::copy(field->v->begin(), field->v->end(), out);
    });
  }

  // The same from the KV bytes of both relations (SURVEY §8f rank 1), without decoding a single index row
  // into DataValues: see plan_kv_bytes.
  void stage_kv(const KvRelation& base, const KvRelation& idx, const HnswIndexManifest& mf) {
    upload(plan_kv_bytes(base, idx, mf), mf);
  }

  // Reference implementation of stage_kv: decode every KV pair into a tuple first (decode_tuple_from_kv),
  // then plan as `stage` does.  Kept as the cross-check of the byte-level planner.
  static StagePlan plan_kv_tuples(const KvRelation& base, const KvRelation& idx, const HnswIndexManifest& mf) {
    std::vector<Tuple> idx_rows;
    idx_rows.reserve(idx.kv.size());
    for (auto& kv : idx.kv) idx_rows.push_back(decode_tuple_from_kv(kv.first, kv.second));
    const size_t K = base.n_keys;
    return plan_with(K, std::move(idx_rows), mf, [&](const CompoundKey& ck, float* out) {
      const std::string* val = base.get_val(std::get<0>(ck));
      if (!val) throw CozoError("", "Cannot find compound key for HNSW");
      const size_t fld = std::get<1>(ck);
      if (fld < K) {  // a vector stored in a key column: it is part of the compound key itself
        const DataValue& f = std::get<0>(ck)[fld];
        if (f.kind != DataValue::Vec || f.v->size() != mf.vec_dim)
          throw CozoError("", "Cannot interpret " + f.repr() + " as vector");
        std::copy(f.v->begin(), f.v->end(), out);
        return;
      }
      msgpack_codec::extract_vector(*val, fld - K, std::get<2>(ck), out, mf.vec_dim);
    });
  }

  // Byte-level planner.  An index key is  relid(8) | layer | FROM | TO  where FROM and TO are the memcmp
  // encodings of (k.., field, sub_idx): self-delimiting, order-preserving and canonical, so
  //   * the scan order of the relation IS (layer, FROM, TO) order: per level, rows arrive grouped by FROM,
  //   * dense ids are the ranks of the distinct FROM byte strings of the layer-0 block,
  //   * a TO is resolved by binary search over those byte strings,
  //   * "same base row" (hnsw.rs:609) is byte equality of the k.. prefixes,
  //   * the base row of a vector is found under  base relid | k.. bytes  with no re-encoding.
  // Only `layer`, `field`, `sub_idx` (integers), `ignore_link` (one msgpack bool) and the n compound keys
  // handed back for result assembly are ever decoded.
  static StagePlan plan_kv_bytes(const KvRelation& base, const KvRelation& idx, const HnswIndexManifest& mf) {
    if (mf.dtype_f64)
      throw CozoError("gpu::unsupported", "F64 vector indexes are outside the device envelope (f32 only)");
    using memcmp_codec::skip_datavalue;
    const size_t K = base.n_keys;
    struct Row {
      int64_t layer;
      const uint8_t *from, *to;  // start of FROM / TO
      uint32_t from_len, from_klen, to_len, to_klen;
      bool canary, ignored;
      const std::string* val;
    };
    std::vector<Row> rows(idx.kv.size());
    auto parse_range = [&](size_t lo, size_t hi) {
      for (size_t ri = lo; ri < hi; ++ri) {
        auto& kv = idx.kv[ri];
        const uint8_t* p = reinterpret_cast<const uint8_t*>(kv.first.data());
        const uint8_t* end = p + kv.first.size();
        if (kv.first.size() < memcmp_codec::ENCODED_KEY_MIN_LEN) throw CozoError("", "key shorter than the relation id prefix");
        p += memcmp_codec::ENCODED_KEY_MIN_LEN;
        DataValue layer;
        p += memcmp_codec::decode_datavalue(p, (size_t)(end - p), layer);
        Row r{};
        if (!layer.get_int(r.layer)) throw CozoError("", "corrupted index: layer is not an integer");
        r.val = &kv.second;
        auto part = [&](const uint8_t*& start, uint32_t& len, uint32_t& klen, bool& null_field) {
          start = p;
          for (size_t i = 0; i < K; ++i) p += skip_datavalue(p, (size_t)(end - p));
          klen = (uint32_t)(p - start);
          null_field = p < end && *p == memcmp_codec::NULL_TAG;
          p += skip_datavalue(p, (size_t)(end - p));  // field
          p += skip_datavalue(p, (size_t)(end - p));  // sub_idx
          len = (uint32_t)(p - start);
        };
        bool to_null = false;
        part(r.from, r.from_len, r.from_klen, r.canary);  // canary row: fr__field is Null (hnsw.rs:903-909)
        part(r.to, r.to_len, r.to_klen, to_null);
        if (p != end) throw CozoError("", "corrupted index: bad row width");
        // ignore_link is read here, next to the key, while the pair is in cache (hnsw.rs:618-620)
        r.ignored = r.layer <= 0 && !r.canary && msgpack_codec::read_bool_column(kv.second, 2);
        rows[ri] = r;
      }
    };
    {  // rows are independent: parse them on a few threads (exceptions are carried back to the caller)
      const size_t nt = std::max<size_t>(1, std::min<size_t>({(size_t)std::thread::hardware_concurrency(), (size_t)16,
                                                              rows.size() / 65536 + 1}));
      std::vector<std::thread> th;
      std::vector<std::exception_ptr> errs(nt);
      for (size_t t = 0; t < nt; ++t)
        th.emplace_back([&, t] {
          try {
            parse_range(rows.size() * t / nt, rows.size() * (t + 1) / nt);
          } catch (...) {
            errs[t] = std::current_exception();
          }
        });
      for (auto& t : th) t.join();
      for (auto& e : errs)
        if (e) std::rethrow_exception(e);
    }
    auto key_less = [](const Row& a, const Row& b) {  // (layer, FROM, TO): the storage order
      if (a.layer != b.layer) return a.layer < b.layer;
      int c = std::memcmp(a.from, b.from, std::min(a.from_len, b.from_len));
      if (c || a.from_len != b.from_len) return c ? c < 0 : a.from_len < b.from_len;
      c = std::memcmp(a.to, b.to, std::min(a.to_len, b.to_len));
      return c ? c < 0 : a.to_len < b.to_len;
    };
    if (!std::is_sorted(rows.begin(), rows.end(), key_less)) std::sort(rows.begin(), rows.end(), key_less);
    StagePlan pl;
    // dense ids: distinct FROMs of the layer-0 block, which is contiguous and sorted
    std::vector<std::pair<const uint8_t*, uint32_t>> froms;
    for (const Row& r : rows) {
      if (r.layer != 0 || r.canary) continue;
      if (froms.empty() || froms.back().second != r.from_len || std::memcmp(froms.back().first, r.from, r.from_len) != 0)
        froms.emplace_back(r.from, r.from_len);
    }
    const uint32_t n = (uint32_t)froms.size();
    // FROM / TO bytes -> dense id: open addressing over the byte strings (FNV-1a), ids = ranks in `froms`
    std::vector<uint32_t> table(n ? (size_t)1 << (64 - __builtin_clzll((uint64_t)n * 2)) : 1, COZO_GPU_NONE);
    const size_t tmask = table.size() - 1;
    auto hash_of = [](const uint8_t* b, uint32_t len) {
      uint64_t hsh = 1469598103934665603ull;
      for (uint32_t i = 0; i < len; ++i) hsh = (hsh ^ b[i]) * 1099511628211ull;
      return (size_t)(hsh ^ (hsh >> 29));
    };
    for (uint32_t i = 0; i < n; ++i) {
      size_t slot = hash_of(froms[i].first, froms[i].second) & tmask;
      while (table[slot] != COZO_GPU_NONE) slot = (slot + 1) & tmask;
      table[slot] = i;
    }
    auto id_of = [&](const uint8_t* b, uint32_t len) -> uint32_t {
      if (n == 0) return COZO_GPU_NONE;
      for (size_t slot = hash_of(b, len) & tmask;; slot = (slot + 1) & tmask) {
        const uint32_t i = table[slot];
        if (i == COZO_GPU_NONE) return COZO_GPU_NONE;
        if (froms[i].second == len && std::memcmp(froms[i].first, b, len) == 0) return i;
      }
    };
    // the compound keys handed back for result assembly (n decodes, not one per row)
    pl.keys.reserve(n);
    for (auto& f : froms) {
      Tuple t;
      size_t off = 0;
      while (off < f.second) {
        DataValue v;
        off += memcmp_codec::decode_datavalue(f.first + off, f.second - off, v);
        t.push_back(std::move(v));
      }
      if (t.size() != K + 2) throw CozoError("", "corrupted index: bad row width");
      int64_t fld = 0, sub = 0;
      if (!t[K].get_int(fld) || !t[K + 1].get_int(sub)) throw CozoError("", "corrupted index: field / sub index");
      t.resize(K);
      pl.keys.emplace_back(std::move(t), (size_t)fld, (int32_t)sub);
    }
    // entry point: the first row in key order with layer in [i64::MIN, 1] (hnsw.rs:891-899)
    int64_t bottom_level = 0;
    for (const Row& r : rows) {
      if (r.layer > 1) continue;
      if (!r.canary) {
        bottom_level = r.layer;
        pl.entry = id_of(r.from, r.from_len);
        if (pl.entry == COZO_GPU_NONE) throw CozoError("", "corrupted index");
      }
      break;
    }
    pl.n_levels = pl.entry == COZO_GPU_NONE ? 1 : (uint32_t)(-bottom_level) + 1;
    pl.node_ids.assign(pl.n_levels, {});
    pl.col_idx.assign(pl.n_levels, {});
    pl.row_ptr.assign(pl.n_levels, std::vector<uint64_t>(1, 0));
    // adjacency with the reading rules of hnsw_get_neighbours(include_deleted=false); per level the rows
    // arrive grouped by FROM in ascending id order, so the CSR is appended to directly
    std::vector<uint32_t> cur(pl.n_levels, COZO_GPU_NONE);  // the FROM whose row is open, per level
    uint32_t next0 = 0;                                     // level 0 lists every id: rows closed so far
    const uint8_t* last_from = nullptr;
    uint32_t last_len = 0, last_fi = COZO_GPU_NONE;
    for (const Row& r : rows) {
      if (r.layer > 0 || r.canary) continue;
      const uint32_t L = (uint32_t)(-r.layer);
      if (L >= pl.n_levels) continue;
      // rows of one FROM are consecutive: resolve it once
      if (!(last_from && last_len == r.from_len && std::memcmp(last_from, r.from, r.from_len) == 0)) {
        last_from = r.from;
        last_len = r.from_len;
        last_fi = id_of(r.from, r.from_len);
        if (last_fi == COZO_GPU_NONE) throw CozoError("", "corrupted index");
      }
      const uint32_t fi = last_fi;
      if (cur[L] != fi) {  // open a new row (self-loop rows create the, possibly empty, row)
        if (L == 0) {
          for (; next0 < fi; ++next0) pl.row_ptr[0].push_back(pl.col_idx[0].size());  // ids without rows
          next0 = fi + 1;
        } else {
          pl.node_ids[L].push_back(fi);
        }
        pl.row_ptr[L].push_back(pl.col_idx[L].size());
        cur[L] = fi;
      }
      if (r.to_klen == r.from_klen && std::memcmp(r.to, r.from, r.from_klen) == 0) {  // hnsw.rs:609: tuple key only
        pl.n_rows_dropped_same_key++;
        continue;
      }
      if (r.ignored) {  // hnsw.rs:618-620
        pl.n_rows_dropped_ignored++;
        continue;
      }
      const uint32_t ti = id_of(r.to, r.to_len);
      if (ti == COZO_GPU_NONE) throw CozoError("", "corrupted index: edge to an unknown vector");
      pl.col_idx[L].push_back(ti);
      pl.row_ptr[L].back() = pl.col_idx[L].size();
      pl.n_edges_kept++;
    }
    for (; next0 < n; ++next0) pl.row_ptr[0].push_back(pl.col_idx[0].size());
    // vectors: VectorCache::ensure_key (hnsw.rs:122-151) against the base relation's KV bytes
    pl.vectors.resize((size_t)n * mf.vec_dim);
    std::string bkey;
    for (uint32_t i = 0; i < n; ++i) {
      float* out = pl.vectors.data() + (size_t)i * mf.vec_dim;
      const size_t fld = std::get<1>(pl.keys[i]);
      if (fld < K) {
        const DataValue& f = std::get<0>(pl.keys[i])[fld];
        if (f.kind != DataValue::Vec || f.v->size() != mf.vec_dim)
          throw CozoError("", "Cannot interpret " + f.repr() + " as vector");
        std::copy(f.v->begin(), f.v->end(), out);
        continue;
      }
      bkey.clear();
      memcmp_codec::put_u64_be(bkey, base.id);
      // the k.. bytes of FROM are the base relation's key bytes: klen = length of the first K values
      {
        size_t klen = 0;
        for (size_t c = 0; c < K; ++c) klen += skip_datavalue(froms[i].first + klen, froms[i].second - klen);
        bkey.append(reinterpret_cast<const char*>(froms[i].first), klen);
      }
      const std::string* val = base.get_val_bytes(bkey);
      if (!val) throw CozoError("", "Cannot find compound key for HNSW");
      msgpack_codec::extract_vector(*val, fld - K, std::get<2>(pl.keys[i]), out, mf.vec_dim);
    }
    return pl;
  }

  // fetch(compound key, out[vec_dim]) = VectorCache::ensure_key (hnsw.rs:122-151)
  template <class Fetch>
  void stage_with(size_t K, std::vector<Tuple> idx_rows, const HnswIndexManifest& mf, Fetch fetch) {
    upload(plan_with(K, std::move(idx_rows), mf, fetch), mf);
  }

  template <class Fetch>
  static StagePlan plan_with(size_t K, std::vector<Tuple> idx_rows, const HnswIndexManifest& mf, Fetch fetch) {
    StagePlan pl;
    std::vector<CompoundKey>& keys = pl.keys;
    uint64_t &n_edges_kept = pl.n_edges_kept, &n_rows_dropped_same_key = pl.n_rows_dropped_same_key,
             &n_rows_dropped_ignored = pl.n_rows_dropped_ignored;
    if (mf.dtype_f64)
      throw CozoError("gpu::unsupported", "F64 vector indexes are outside the device envelope (f32 only)");
    // This planner orders rows and compound keys by DataValue order.  Storage (and the reference's entry-point
    // scan, hnsw.rs:891-899) orders them by memcmp bytes; the two agree for every key type except Vec, whose tag
    // sorts before numbers and whose elements are raw big-endian bits.  Relations keyed by vectors go through
    // stage_kv / plan_kv_bytes, which works on the stored bytes; refuse them here instead of mis-ordering.
    for (const Tuple& t : idx_rows)
      for (size_t c = 1; c < t.size() && c < 2 * K + 5; ++c)
        if (t[c].kind == DataValue::Vec)
          throw CozoError("gpu::unsupported", "vector-typed key columns: stage this index from KV bytes (stage_kv)");
    std::sort(idx_rows.begin(), idx_rows.end(), TupleLess());
    // dense ids = compound keys of the layer-0 self-loop rows, in key order
    std::map<CompoundKey, uint32_t, CompoundKeyLess> ids;
    auto fr_key = [&](const Tuple& t, bool& canary) -> CompoundKey {
      int64_t fld = 0, sub = 0;
      canary = !t[K + 1].get_int(fld);  // canary row: fr__field is Null (hnsw.rs:903-909)
      if (!canary) t[K + 2].get_int(sub);
      return CompoundKey(Tuple(t.begin() + 1, t.begin() + 1 + K), (size_t)fld, (int32_t)sub);
    };
    auto to_key = [&](const Tuple& t) -> CompoundKey {
      int64_t fld = 0, sub = 0;
      t[2 * K + 3].get_int(fld);
      t[2 * K + 4].get_int(sub);
      return CompoundKey(Tuple(t.begin() + K + 3, t.begin() + 2 * K + 3), (size_t)fld, (int32_t)sub);
    };
    for (const Tuple& t : idx_rows) {
      if (t.size() != 2 * K + 8) throw CozoError("", "corrupted index: bad row width");
      int64_t layer;
      if (!t[0].get_int(layer) || layer != 0) continue;
      bool canary;
      CompoundKey f = fr_key(t, canary);
      if (canary) continue;
      ids.emplace(f, 0u);
    }
    keys.clear();
    for (auto& kv : ids) {
      kv.second = (uint32_t)keys.size();
      keys.push_back(kv.first);
    }
    const uint32_t n = (uint32_t)keys.size();
    // entry point: the first row in key order with layer in [i64::MIN, 1] (hnsw.rs:891-899)
    uint32_t& entry = pl.entry;
    int64_t bottom_level = 0;
    for (const Tuple& t : idx_rows) {
      int64_t layer;
      if (!t[0].get_int(layer) || layer > 1) continue;
      bool canary;
      CompoundKey f = fr_key(t, canary);
      if (!canary) {
        bottom_level = layer;
        auto it = ids.find(f);
        if (it == ids.end()) throw CozoError("", "corrupted index");
        entry = it->second;
      }
      break;
    }
    const uint32_t n_levels = pl.n_levels = entry == COZO_GPU_NONE ? 1 : (uint32_t)(-bottom_level) + 1;
    // adjacency with the reading rules of hnsw_get_neighbours(include_deleted=false)
    pl.node_ids.assign(n_levels, {});
    std::vector<std::vector<uint32_t>>& node_ids = pl.node_ids;
    std::vector<std::map<uint32_t, std::vector<uint32_t>>> adj(n_levels);
    for (const Tuple& t : idx_rows) {
      int64_t layer;
      if (!t[0].get_int(layer) || layer > 0) continue;
      bool canary;
      CompoundKey f = fr_key(t, canary);
      if (canary) continue;
      const uint32_t L = (uint32_t)(-layer);
      if (L >= n_levels) continue;
      CompoundKey to = to_key(t);
      uint32_t fi = ids.at(f);
      auto& row = adj[L][fi];  // self-loop rows create the (possibly empty) row
      if (cmp_tuple(std::get<0>(to), std::get<0>(f)) == 0) {  // hnsw.rs:609: tuple key only
        n_rows_dropped_same_key++;
        continue;
      }
      bool ignored = false;
      t[2 * K + 7].get_bool(ignored);
      if (ignored) {  // hnsw.rs:618-620
        n_rows_dropped_ignored++;
        continue;
      }
      auto it = ids.find(to);
      if (it == ids.end()) throw CozoError("", "corrupted index: edge to an unknown vector");
      row.push_back(it->second);  // rows arrive in key order => ascending ids
      n_edges_kept++;
    }
    // vectors (VectorCache::ensure_key, hnsw.rs:122-151)
    pl.vectors.resize((size_t)n * mf.vec_dim);
    std::vector<float>& vectors = pl.vectors;
    for (uint32_t i = 0; i < n; ++i) fetch(keys[i], vectors.data() + (size_t)i * mf.vec_dim);
    // flatten
    pl.row_ptr.assign(n_levels, {});
    pl.col_idx.assign(n_levels, {});
    for (uint32_t L = 0; L < n_levels; ++L) {
      pl.row_ptr[L].push_back(0);
      if (L == 0) {
        for (uint32_t i = 0; i < n; ++i) {
          auto it = adj[0].find(i);
          if (it != adj[0].end()) pl.col_idx[0].insert(pl.col_idx[0].end(), it->second.begin(), it->second.end());
          pl.row_ptr[0].push_back(pl.col_idx[0].size());
        }
      } else {
        for (auto& kv : adj[L]) {
          node_ids[L].push_back(kv.first);
          pl.col_idx[L].insert(pl.col_idx[L].end(), kv.second.begin(), kv.second.end());
          pl.row_ptr[L].push_back(pl.col_idx[L].size());
        }
      }
    }
    return pl;
  }

  // hand a plan to the device (cozo_gpu_hnsw_stage) and adopt its dictionary
  void upload(StagePlan pl, const HnswIndexManifest& mf) {
    manifest = mf;
    const uint32_t n = (uint32_t)pl.keys.size();
    std::vector<CozoGpuHnswLevel> levels(pl.n_levels);
    for (uint32_t L = 0; L < pl.n_levels; ++L) {
      levels[L].n_nodes = L == 0 ? n : (uint32_t)pl.node_ids[L].size();
      levels[L].node_ids = L == 0 ? nullptr : pl.node_ids[L].data();
      levels[L].row_ptr = pl.row_ptr[L].data();
      levels[L].col_idx = pl.col_idx[L].data();
    }
    float dummy = 0;
    CozoGpuHnswStageDesc d{};
    d.n_vectors = n;
    d.dim = (uint32_t)mf.vec_dim;
    d.metric = (int32_t)mf.distance;
    d.n_levels = pl.n_levels;
    d.levels = levels.data();
    d.vectors = n ? pl.vectors.data() : &dummy;
    d.vectors_on_device = 0;
    d.entry_point = pl.entry;
    d.m_max0 = (uint32_t)mf.m_max0;
    d.m_max = (uint32_t)mf.m_max;
    if (h) {
      cozo_gpu_hnsw_free(h);
      h = nullptr;
    }
    gpu_check(cozo_gpu_hnsw_stage(&h, &d));
    keys = std::move(pl.keys);
    key_ids.clear();
    live.clear();
    n_edges_kept = pl.n_edges_kept;
    n_rows_dropped_same_key = pl.n_rows_dropped_same_key;
    n_rows_dropped_ignored = pl.n_rows_dropped_ignored;
  }

  // create_hnsw_index (runtime/relation.rs:1010-1201): index every vector of the base relation in key
  // order (single vectors and list-of-vectors columns, hnsw.rs:694-706), on the device.
  void build(const RelationHandle& base, const HnswIndexManifest& mf, uint64_t level_seed = 0x5EED0003ull) {
    manifest = mf;
    if (mf.dtype_f64)
      throw CozoError("gpu::unsupported", "F64 vector indexes are outside the device envelope (f32 only)");
    keys.clear();
    key_ids.clear();
    live.clear();
    std::vector<float> vectors;
    for (auto& kv : base.rows) {
      for (size_t fld : mf.vec_fields) {
        const DataValue& val = kv.second.at(fld);
        auto push = [&](const DataValue& v, int32_t sub) {
          if (v.kind != DataValue::Vec) return;
          if (v.v->size() != mf.vec_dim) throw CozoError("", "vector dimension mismatch for the index");
          keys.emplace_back(kv.first, fld, sub);
          vectors.insert(vectors.end(), v.v->begin(), v.v->end());
        };
        if (val.kind == DataValue::Vec) push(val, -1);
        else if (val.kind == DataValue::List)
          for (size_t i = 0; i < val.list.size(); ++i) push(val.list[i], (int32_t)i);
      }
    }
    // keys are generated row by row, field by field: sort into compound-key order (dense id = key order)
    std::vector<size_t> order(keys.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return CompoundKeyLess()(keys[a], keys[b]); });
    std::vector<CompoundKey> k2(keys.size());
    std::vector<float> v2(vectors.size());
    for (size_t r = 0; r < order.size(); ++r) {
      k2[r] = keys[order[r]];
      std::copy(vectors.begin() + order[r] * mf.vec_dim, vectors.begin() + (order[r] + 1) * mf.vec_dim,
                v2.begin() + r * mf.vec_dim);
    }
    keys.swap(k2);
    if (h) {
      cozo_gpu_hnsw_free(h);
      h = nullptr;
    }
    if (keys.empty()) {  // nothing to index yet: an empty staged index (canary only)
      CozoGpuHnswLevel l0{};
      uint64_t zero = 0;
      l0.row_ptr = &zero;
      CozoGpuHnswStageDesc d{};
      d.dim = (uint32_t)mf.vec_dim;
      d.metric = (int32_t)mf.distance;
      d.n_levels = 1;
      d.levels = &l0;
      d.entry_point = COZO_GPU_NONE;
      d.m_max0 = (uint32_t)mf.m_max0;
      d.m_max = (uint32_t)mf.m_max;
      float dummy = 0;
      d.vectors = &dummy;
      gpu_check(cozo_gpu_hnsw_stage(&h, &d));
      return;
    }
    CozoGpuHnswBuildDesc d{};
    d.n_vectors = (uint32_t)keys.size();
    d.dim = (uint32_t)mf.vec_dim;
    d.metric = (int32_t)mf.distance;
    d.vectors = v2.data();
    d.m_neighbours = (uint32_t)mf.m_neighbours;
    d.ef_construction = (uint32_t)mf.ef_construction;
    d.extend_candidates = mf.extend_candidates;
    d.keep_pruned_connections = mf.keep_pruned_connections;
    d.level_seed = level_seed;
    gpu_check(cozo_gpu_hnsw_build(&h, &d));
  }

  // ---- maintenance: `:put` / `:rm` on an indexed relation (query/stored.rs:332, 995-997) -------------
  // The device copy absorbs a mutation in place when dense ids can stay in compound-key order (the order
  // the entry-point rule reads, hnsw.rs:891-899): changed vectors under existing keys, removals, and new
  // rows whose key sorts after every indexed key (the append case).  A new key inside the indexed range
  // re-indexes from the base relation (`rebuilt` counts those), or, with `insert_inside`, goes to
  // cozo_gpu_hnsw_insert_at, which moves existing ids up so that they stay in key order.
  std::map<CompoundKey, uint32_t, CompoundKeyLess> key_ids;  // compound key -> dense id (lazily rebuilt)
  std::vector<uint8_t> live;                                  // host mirror of the device's live flags
  bool is_live(uint32_t id) const { return live.size() != keys.size() || live[id] != 0; }
  uint64_t n_put_unchanged = 0, n_put_updated = 0, n_put_appended = 0, n_put_inserted = 0, n_removed = 0, n_rebuilt = 0;
  bool insert_inside = false;  // opt-in: keys inside the indexed range are inserted in place instead of re-indexing

  void sync_dictionary() {
    if (key_ids.size() == keys.size() && live.size() == keys.size()) return;
    key_ids.clear();
    for (uint32_t i = 0; i < keys.size(); ++i) key_ids.emplace(keys[i], i);
    live.assign(keys.size(), 1);
    if (!keys.empty()) gpu_check(cozo_gpu_hnsw_export_live(h, live.data()));
  }

  // the (vector, field, sub_idx) triples hnsw_put extracts from a row (hnsw.rs:694-706)
  std::vector<std::tuple<const std::vector<float>*, size_t, int32_t>> extract_vectors(const Tuple& tuple) const {
    std::vector<std::tuple<const std::vector<float>*, size_t, int32_t>> out;
    for (size_t fld : manifest.vec_fields) {
      const DataValue& val = tuple.at(fld);
      if (val.kind == DataValue::Vec) out.emplace_back(val.v.get(), fld, -1);
      else if (val.kind == DataValue::List)
        for (size_t i = 0; i < val.list.size(); ++i)
          if (val.list[i].kind == DataValue::Vec) out.emplace_back(val.list[i].v.get(), fld, (int32_t)i);
    }
    return out;
  }

  // SessionTx::hnsw_remove (hnsw.rs:728-753) for a batch of rows: every indexed vector of each row
  void remove_rows(RelationHandle& base, const std::vector<Tuple>& rows) {
    sync_dictionary();
    const size_t K = base.keys.size();
    std::vector<uint32_t> ids;
    for (const Tuple& row : rows) {
      Tuple key(row.begin(), row.begin() + K);
      for (auto it = key_ids.lower_bound(CompoundKey(key, 0, INT32_MIN));
           it != key_ids.end() && cmp_tuple(std::get<0>(it->first), key) == 0; ++it)
        if (live[it->second]) {
          ids.push_back(it->second);
          live[it->second] = 0;
        }
      base.erase(key);
    }
    if (!ids.empty()) gpu_check(cozo_gpu_hnsw_remove(h, ids.data(), (uint32_t)ids.size()));
    n_removed += ids.size();
  }

  // cozo_gpu_hnsw_compact: the removed ids leave the device copy and their keys leave the dictionary, so that dense ids
  // are again the key ranks of the indexed rows, as a fresh stage gives them
  void compact() {
    sync_dictionary();
    if (keys.empty()) return;
    std::vector<uint32_t> old_to_new(keys.size());
    gpu_check(cozo_gpu_hnsw_compact(h, old_to_new.data()));
    std::vector<CompoundKey> k2;
    for (size_t i = 0; i < keys.size(); ++i)
      if (old_to_new[i] != COZO_GPU_NONE) {
        if (old_to_new[i] != k2.size()) throw CozoError("", "device ids out of step with the key dictionary");
        k2.push_back(std::move(keys[i]));
      }
    keys.swap(k2);
    live.assign(keys.size(), 1);
    key_ids.clear();
    for (uint32_t i = 0; i < keys.size(); ++i) key_ids.emplace(keys[i], i);
  }

  // SessionTx::hnsw_put (hnsw.rs:679-727) for a batch of rows, then the rows go into the base relation.
  // `filter` is the index_filter predicate (rows failing it are un-indexed, hnsw.rs:688-693).
  void put_rows(RelationHandle& base, const std::vector<Tuple>& all_rows,
                const std::function<bool(const Tuple&)>& filter = nullptr) {
    sync_dictionary();
    const size_t K = base.keys.size(), dim = manifest.vec_dim;
    // several rows under one key in a batch: the reference applies them in order, so the last one stands
    std::vector<Tuple> rows;
    {
      std::map<Tuple, size_t, TupleLess> last;
      for (size_t i = 0; i < all_rows.size(); ++i) {
        if (all_rows[i].size() < K) throw CozoError("", "row arity mismatch");
        last[Tuple(all_rows[i].begin(), all_rows[i].begin() + K)] = i;
      }
      for (size_t i = 0; i < all_rows.size(); ++i)
        if (last[Tuple(all_rows[i].begin(), all_rows[i].begin() + K)] == i) rows.push_back(all_rows[i]);
    }
    std::vector<uint32_t> upd_ids, rm_ids;
    std::vector<float> upd_vecs;
    std::vector<std::pair<CompoundKey, const std::vector<float>*>> appended;
    for (const Tuple& row : rows) {
      if (row.size() != base.keys.size() + base.non_keys.size()) throw CozoError("", "row arity mismatch");
      Tuple key(row.begin(), row.begin() + K);
      if (filter && !filter(row)) {  // hnsw.rs:688-693
        for (auto it = key_ids.lower_bound(CompoundKey(key, 0, INT32_MIN));
             it != key_ids.end() && cmp_tuple(std::get<0>(it->first), key) == 0; ++it)
          if (live[it->second]) {
            rm_ids.push_back(it->second);
            live[it->second] = 0;
          }
        continue;
      }
      const Tuple* old_row = base.get(key);
      for (auto& [vec, fld, sub] : extract_vectors(row)) {
        if (vec->size() != dim) throw CozoError("", "vector dimension mismatch for the index");
        CompoundKey ck(key, fld, sub);
        auto it = key_ids.find(ck);
        if (it == key_ids.end()) {
          appended.emplace_back(std::move(ck), vec);
          continue;
        }
        if (live[it->second] && old_row) {  // same bytes under the same key: nothing to do (hnsw.rs:175-179)
          const DataValue* f = &(*old_row)[fld];
          if (sub >= 0 && f->kind == DataValue::List && (size_t)sub < f->list.size()) f = &f->list[(size_t)sub];
          if (f->kind == DataValue::Vec && f->v->size() == dim &&
              std::memcmp(f->v->data(), vec->data(), dim * sizeof(float)) == 0) {
            n_put_unchanged++;
            continue;
          }
        }
        upd_ids.push_back(it->second);  // remove + insert again (hnsw.rs:180-182)
        upd_vecs.insert(upd_vecs.end(), vec->begin(), vec->end());
        live[it->second] = 1;
      }
    }
    std::sort(appended.begin(), appended.end(),
              [](const auto& a, const auto& b) { return CompoundKeyLess()(a.first, b.first); });
    const bool in_order = appended.empty() || key_ids.empty() || CompoundKeyLess()(key_ids.rbegin()->first, appended.front().first);
    for (const Tuple& row : rows) base.put(row);
    // a new key lands inside the indexed key range (ids must stay in key order), or nothing is indexed yet
    // (then this is create_hnsw_index over the rows just stored): re-index from the base relation
    if ((!in_order && !insert_inside) || (keys.empty() && !appended.empty())) {
      n_rebuilt++;
      build(base, manifest);
      if (filter) {
        std::vector<Tuple> drop;
        for (auto& kv : base.rows)
          if (!filter(kv.second)) drop.push_back(kv.second);
        // un-index without deleting the rows
        sync_dictionary();
        std::vector<uint32_t> ids;
        for (const Tuple& row : drop) {
          Tuple key(row.begin(), row.begin() + K);
          for (auto it = key_ids.lower_bound(CompoundKey(key, 0, INT32_MIN));
               it != key_ids.end() && cmp_tuple(std::get<0>(it->first), key) == 0; ++it)
            if (live[it->second]) {
              ids.push_back(it->second);
              live[it->second] = 0;
            }
        }
        if (!ids.empty()) gpu_check(cozo_gpu_hnsw_remove(h, ids.data(), (uint32_t)ids.size()));
      }
      return;
    }
    if (!rm_ids.empty()) gpu_check(cozo_gpu_hnsw_remove(h, rm_ids.data(), (uint32_t)rm_ids.size()));
    n_removed += rm_ids.size();
    if (!upd_ids.empty())
      gpu_check(cozo_gpu_hnsw_update(h, upd_ids.data(), upd_vecs.data(), (uint32_t)upd_ids.size(),
                                     (uint32_t)manifest.ef_construction, manifest.keep_pruned_connections ? 1 : 0));
    n_put_updated += upd_ids.size();
    if (!appended.empty()) {
      std::vector<float> flat;
      flat.reserve(appended.size() * dim);
      for (auto& a : appended) flat.insert(flat.end(), a.second->begin(), a.second->end());
      const uint32_t efc = (uint32_t)manifest.ef_construction, keep = manifest.keep_pruned_connections ? 1 : 0;
      if (in_order) {
        uint32_t first = 0;
        gpu_check(cozo_gpu_hnsw_insert(h, flat.data(), (uint32_t)appended.size(), 0, efc, keep, &first));
        if (first != keys.size()) throw CozoError("", "device ids out of step with the key dictionary");
        for (auto& a : appended) {
          key_ids.emplace(a.first, (uint32_t)keys.size());
          keys.push_back(a.first);
          live.push_back(1);
        }
        n_put_appended += appended.size();
      } else {
        // position = ids (removed ones included) whose key sorts before the new key; `appended` is in key order
        const uint32_t c = (uint32_t)appended.size();
        std::vector<uint32_t> pos(c), ids(c);
        for (uint32_t i = 0; i < c; ++i)
          pos[i] = (uint32_t)(std::lower_bound(keys.begin(), keys.end(), appended[i].first, CompoundKeyLess()) - keys.begin());
        gpu_check(cozo_gpu_hnsw_insert_at(h, pos.data(), flat.data(), c, 0, efc, keep, ids.data()));
        std::vector<CompoundKey> k2;
        std::vector<uint8_t> l2;
        k2.reserve(keys.size() + c);
        l2.reserve(keys.size() + c);
        uint32_t j = 0;
        for (uint32_t i = 0; i <= c; ++i) {
          const uint32_t upto = i < c ? pos[i] : (uint32_t)keys.size();
          for (; j < upto; ++j) {
            k2.push_back(std::move(keys[j]));
            l2.push_back(live[j]);
          }
          if (i == c) break;
          if (ids[i] != k2.size()) throw CozoError("", "device ids out of step with the key dictionary");
          k2.push_back(appended[i].first);
          l2.push_back(1);
        }
        keys.swap(k2);
        live.swap(l2);
        key_ids.clear();
        for (uint32_t i = 0; i < keys.size(); ++i) key_ids.emplace(keys[i], i);
        n_put_inserted += c;
      }
    }
  }

  // The rows of `rel:idx` (runtime/relation.rs:1064-1126; SURVEY.md appendix A) that describe the device
  // copy: the canary, one self-loop row per (node, layer) carrying the degree and the vector's SHA-256,
  // one row per directed edge carrying the stored distance.  Feeding them back to stage() reproduces
  // the same index.
  std::vector<Tuple> to_index_rows(const RelationHandle& base) const {
    const size_t K = base.keys.size();
    uint32_t n = 0, dim = 0, n_levels = 0, entry = COZO_GPU_NONE;
    gpu_check(cozo_gpu_hnsw_info(h, &n, &dim, &n_levels, &entry));
    std::vector<uint8_t> live(std::max<uint32_t>(n, 1), 1);
    if (n) gpu_check(cozo_gpu_hnsw_export_live(h, live.data()));
    auto key_part = [&](Tuple& t, uint32_t id) {
      const CompoundKey& ck = keys[id];
      t.insert(t.end(), std::get<0>(ck).begin(), std::get<0>(ck).end());
      t.push_back(DataValue::from_int((int64_t)std::get<1>(ck)));
      t.push_back(DataValue::from_int((int64_t)std::get<2>(ck)));
    };
    std::vector<Tuple> rows;
    if (entry == COZO_GPU_NONE) return rows;  // the last vector was removed: the canary goes too (hnsw.rs:861-864)
    {  // canary (hnsw.rs:642-669): (1, Null x (2K+4)) => (top layer, key bytes of the entry's self loop, false)
      Tuple t{DataValue::from_int(1)};
      for (size_t i = 0; i < 2 * K + 4; ++i) t.push_back(DataValue::null());
      t.push_back(DataValue::from_int(-(int64_t)(n_levels - 1)));
      t.push_back(DataValue::from_bytes("entry:" + std::to_string(entry)));
      t.push_back(DataValue::from_bool(false));
      rows.push_back(std::move(t));
    }
    for (uint32_t L = 0; L < n_levels; ++L) {
      uint32_t nn = 0;
      uint64_t ne = 0;
      gpu_check(cozo_gpu_hnsw_level_size(h, L, &nn, &ne));
      std::vector<uint32_t> ni(std::max<uint32_t>(nn, 1)), ci(std::max<uint64_t>(ne, 1));
      std::vector<uint64_t> rp((size_t)nn + 1);
      std::vector<float> ds(std::max<uint64_t>(ne, 1));
      gpu_check(cozo_gpu_hnsw_export_level(h, L, ni.data(), rp.data(), ci.data()));
      gpu_check(cozo_gpu_hnsw_export_level_dist(h, L, ds.data()));
      for (uint32_t r = 0; r < nn; ++r) {
        const uint32_t id = ni[r];
        if (!live[id]) continue;
        const CompoundKey& ck = keys[id];
        const Tuple* brow = base.get(std::get<0>(ck));
        const DataValue* field = brow ? &(*brow)[std::get<1>(ck)] : nullptr;
        if (field && std::get<2>(ck) >= 0) field = &field->list[(size_t)std::get<2>(ck)];
        Tuple self{DataValue::from_int(-(int64_t)L)};
        key_part(self, id);
        key_part(self, id);
        self.push_back(DataValue::from_float((double)(rp[r + 1] - rp[r])));  // degree (hnsw.rs:269-277)
        self.push_back(DataValue::from_bytes(field && field->v ? sha256_le_f32(*field->v) : std::string()));
        self.push_back(DataValue::from_bool(false));
        rows.push_back(std::move(self));
        for (uint64_t e = rp[r]; e < rp[r + 1]; ++e) {
          Tuple t{DataValue::from_int(-(int64_t)L)};
          key_part(t, id);
          key_part(t, ci[e]);
          t.push_back(DataValue::from_float((double)ds[e]));  // hnsw.rs:281-298
          t.push_back(DataValue::null());
          t.push_back(DataValue::from_bool(false));
          rows.push_back(std::move(t));
        }
      }
    }
    std::sort(rows.begin(), rows.end(), TupleLess());
    return rows;
  }
};

// HnswSearch (data/program.rs:976-991): the operator's parameter block
struct HnswSearch {
  const RelationHandle* base_handle = nullptr;
  const StagedHnswIndex* index = nullptr;  // stands for idx_handle + manifest
  size_t k = 0, ef = 0;
  bool bind_field = false, bind_field_idx = false, bind_distance = false, bind_vector = false;
  std::optional<double> radius;
  std::function<bool(const Tuple&)> filter;  // compiled filter bytecode stand-in (hnsw.rs:997-1001)
  // whether the filter expression reads the bound distance (the only binding that depends on the query).
  // If it does not, the verdict is a property of the indexed row: the glue evaluates the bytecode once per
  // row, ships a bit mask, and the kernel trims to k after filtering (cozo_gpu_hnsw_search_filtered).
  bool filter_reads_distance = true;

  void validate() const {  // SearchInput::normalize_hnsw (program.rs:1341-1569)
    if (k == 0) throw CozoError("parser::expected_positive_int_for_hnsw_k", "Expected positive integer for `k`");
    if (ef == 0) throw CozoError("parser::expected_positive_int_for_hnsw_ef", "Expected positive integer for `ef`");
    if (radius && !(*radius > 0.))
      throw CozoError("parser::expected_positive_float_for_hnsw_radius", "Expected positive float for `radius`");
  }
};

// SessionTx::hnsw_knn for a whole batch of query vectors (hnsw.rs:869-1012).
// Returns, per query, the rows `base row ++ [field name] ++ [field idx] ++ [distance] ++ [vector]`.
inline std::vector<std::vector<Tuple>> hnsw_knn_batch(const std::vector<const std::vector<float>*>& queries,
                                                      const HnswSearch& config, CozoGpuSearchStats* stats = nullptr) {
  const StagedHnswIndex& ix = *config.index;
  const size_t dim = ix.manifest.vec_dim;
  const uint32_t B = (uint32_t)queries.size();
  std::vector<float> q((size_t)B * dim);
  for (uint32_t i = 0; i < B; ++i) {
    if (queries[i]->size() != dim) throw CozoError("", "query vector dimension mismatch");  // hnsw.rs:876-878
    std::copy(queries[i]->begin(), queries[i]->end(), q.begin() + (size_t)i * dim);
  }
  const RelationHandle& base = *config.base_handle;
  // candidate row of an indexed vector: base row ++ bindings in the order of HnswSearch::all_bindings
  // (hnsw.rs:958-995, program.rs:1016-1025)
  auto assemble = [&](uint32_t id, const DataValue& distance) {
    const CompoundKey& ck = ix.keys[id];
    const Tuple* row = base.get(std::get<0>(ck));
    if (!row) throw CozoError("", "corrupted index");  // hnsw.rs:958-961
    Tuple cand = *row;
    const size_t fld = std::get<1>(ck);
    const int32_t sub = std::get<2>(ck);
    if (config.bind_field)  // hnsw.rs:964-974
      cand.push_back(DataValue::from_str(fld < base.keys.size() ? base.keys[fld] : base.non_keys[fld - base.keys.size()]));
    if (config.bind_field_idx) cand.push_back(sub < 0 ? DataValue::null() : DataValue::from_int(sub));  // 975-981
    if (config.bind_distance) cand.push_back(distance);  // 982-984
    if (config.bind_vector) {  // 985-995
      if (sub < 0) {
        cand.push_back((*row)[fld]);
      } else {
        if ((*row)[fld].kind != DataValue::List) throw CozoError("", "corrupted index value");
        cand.push_back((*row)[fld].list[(size_t)sub]);
      }
    }
    return cand;
  };
  // with a filter the trim to k happens after filtering (hnsw.rs:943-947, 1005-1006): either inside the kernel
  // (per-row verdicts as a bit mask) or, when the filter reads the distance, on the host over all ef candidates
  const bool device_filter = config.filter && !config.filter_reads_distance;
  const uint32_t k_dev = (config.filter && !device_filter) ? (uint32_t)config.ef : (uint32_t)std::min(config.k, config.ef);
  std::vector<uint32_t> ids((size_t)B * k_dev), count(B);
  std::vector<float> dist((size_t)B * k_dev);
  if (device_filter) {
    const size_t n = ix.keys.size();
    std::vector<uint32_t> mask((n + 31) / 32 + 1, 0u);
    for (size_t id = 0; id < n; ++id)
      if (ix.is_live((uint32_t)id) && base.get(std::get<0>(ix.keys[id])) &&  // removed rows never come back from the device
          config.filter(assemble((uint32_t)id, DataValue::null())))
        mask[id >> 5] |= 1u << (id & 31);
    gpu_check(cozo_gpu_hnsw_search_filtered(ix.h, q.data(), B, k_dev, (uint32_t)config.ef,
                                            config.radius ? *config.radius : -1.0, mask.data(), ids.data(), dist.data(),
                                            count.data(), stats));
  } else {
    gpu_check(cozo_gpu_hnsw_search(ix.h, q.data(), B, k_dev, (uint32_t)config.ef, config.radius ? *config.radius : -1.0,
                                   ids.data(), dist.data(), count.data(), stats));
  }
  std::vector<std::vector<Tuple>> out(B);
  for (uint32_t i = 0; i < B; ++i) {
    for (uint32_t j = 0; j < count[i]; ++j) {
      Tuple cand = assemble(ids[(size_t)i * k_dev + j], DataValue::from_float((double)dist[(size_t)i * k_dev + j]));
      if (config.filter && !device_filter && !config.filter(cand)) continue;  // hnsw.rs:997-1001
      out[i].push_back(std::move(cand));
    }
    if (out[i].size() > config.k) out[i].resize(config.k);  // hnsw.rs:1006
  }
  return out;
}

// HnswSearchRA (query/ra.rs:896-901, 1085-1121): for every parent tuple, bind the query
// column, search, emit parent ++ result.  The reference does this lazily one tuple at a
// time; the operator is a pure function of (tuple, index snapshot), so draining the parent
// into ONE batched launch and re-emitting in parent order is equivalent.
struct HnswSearchRA {
  HnswSearch hnsw_search;
  size_t bind_idx = 0;  // position of the `query` variable in the parent bindings (ra.rs:1091-1098)
  CozoGpuSearchStats last_stats{};

  std::vector<Tuple> iter(const std::vector<Tuple>& parent) {
    hnsw_search.validate();
    std::vector<const std::vector<float>*> qs;
    std::vector<std::shared_ptr<std::vector<float>>> keep;
    for (const Tuple& t : parent) {
      const DataValue& d = t.at(bind_idx);
      if (d.kind != DataValue::Vec) throw CozoError("", "Expected vector, got " + d.repr());  // ra.rs:1106-1109
      qs.push_back(d.v.get());
    }
    auto res = hnsw_knn_batch(qs, hnsw_search, &last_stats);
    std::vector<Tuple> out;
    for (size_t i = 0; i < parent.size(); ++i)
      for (auto& r : res[i]) {  // ra.rs:1112-1116
        Tuple row = parent[i];
        row.insert(row.end(), r.begin(), r.end());
        out.push_back(std::move(row));
      }
    return out;
  }
};

}  // namespace cozo_host
