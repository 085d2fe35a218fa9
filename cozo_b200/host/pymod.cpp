// pymod.cpp — pybind11 test harness over the C++ host layer (fixed_rule.hpp, hnsw.hpp).
// It only converts Python objects to DataValues and back; all logic lives in the headers.
#include <pybind11/functional.h>
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <chrono>

#include "hnsw.hpp"
#include "memcmp.hpp"

namespace py = pybind11;
using namespace cozo_host;

static DataValue to_dv(const py::handle& o) {
  if (o.is_none()) return DataValue::null();
  if (py::isinstance<py::bool_>(o)) return DataValue::from_bool(o.cast<bool>());
  if (py::isinstance<py::int_>(o)) return DataValue::from_int(o.cast<int64_t>());
  if (py::isinstance<py::float_>(o)) return DataValue::from_float(o.cast<double>());
  if (py::isinstance<py::str>(o)) return DataValue::from_str(o.cast<std::string>());
  if (py::isinstance<py::bytes>(o)) return DataValue::from_bytes(o.cast<std::string>());
  if (py::isinstance<py::array>(o)) {
    // Vector::F32, or Vector::F64 cast to the index dtype (hnsw.rs:879-884)
    auto a = py::array_t<float, py::array::c_style | py::array::forcecast>::ensure(o);
    if (!a || a.ndim() != 1) throw CozoError("", "only 1-d float arrays convert to vectors");
    return DataValue::from_vec(std::vector<float>(a.data(), a.data() + a.size()));
  }
  if (py::isinstance<py::list>(o) || py::isinstance<py::tuple>(o)) {
    std::vector<DataValue> l;
    for (auto x : o) l.push_back(to_dv(x));
    return DataValue::from_list(std::move(l));
  }
  // numpy scalars
  if (py::hasattr(o, "item")) return to_dv(o.attr("item")());
  throw CozoError("", "unsupported python value");
}

static py::object from_dv(const DataValue& d) {
  switch (d.kind) {
    case DataValue::Null: return py::none();
    case DataValue::Bool: return py::bool_(d.b);
    case DataValue::Num: return d.is_float ? py::object(py::float_(d.f)) : py::object(py::int_(d.i));
    case DataValue::Str: return py::str(d.s);
    case DataValue::Bytes: return py::bytes(d.s);
    case DataValue::List: {
      py::list l;
      for (auto& x : d.list) l.append(from_dv(x));
      return l;
    }
    case DataValue::Vec: {
      py::array_t<float> a(d.v->size());
      std::copy(d.v->begin(), d.v->end(), a.mutable_data());
      return a;
    }
    default: return py::none();
  }
}

static Tuple to_tuple(const py::handle& row) {
  Tuple t;
  for (auto x : row) t.push_back(to_dv(x));
  return t;
}
static py::list from_tuple(const Tuple& t) {
  py::list l;
  for (auto& x : t) l.append(from_dv(x));
  return l;
}
static std::vector<Tuple> to_rows(const py::handle& rows) {
  std::vector<Tuple> r;
  for (auto x : rows) r.push_back(to_tuple(x));
  return r;
}
static py::list from_rows(const std::vector<Tuple>& rows) {
  py::list l;
  for (auto& t : rows) l.append(from_tuple(t));
  return l;
}

struct PyDb {
  FixedRuleRegistry reg;
  py::list run_fixed_rule(const std::string& name, py::list inputs, py::dict options, size_t head_arity,
                          std::vector<size_t> input_arities, std::shared_ptr<Poison> poison) {
    std::vector<std::vector<Tuple>> ins;
    for (auto r : inputs) ins.push_back(to_rows(r));
    Options opts;
    for (auto kv : options) opts[kv.first.cast<std::string>()] = to_dv(kv.second);
    Poison p = poison ? *poison : Poison();
    return from_rows(reg.run(name, ins, input_arities, std::move(opts), head_arity, p));
  }
  void register_fixed_rule(const std::string& name, size_t arity, py::function fn) {
    auto rule = std::make_shared<SimpleFixedRule>(
        arity, [fn](const std::vector<std::vector<Tuple>>& ins, const Options& opts) -> std::vector<Tuple> {
          py::list pins;
          for (auto& r : ins) pins.append(from_rows(r));
          py::dict popts;
          for (auto& kv : opts) popts[py::str(kv.first)] = from_dv(kv.second);
          return to_rows(fn(pins, popts));
        });
    reg.register_fixed_rule(name, rule);
  }
  bool unregister_fixed_rule(const std::string& name) { return reg.unregister_fixed_rule(name); }
};

struct PyRelation {
  RelationHandle rel;
  PyRelation(const std::string& name, std::vector<std::string> keys, std::vector<std::string> non_keys) {
    rel.name = name;
    rel.keys = std::move(keys);
    rel.non_keys = std::move(non_keys);
  }
  void put(py::handle row) { rel.put(to_tuple(row)); }
  size_t size() const { return rel.rows.size(); }
};

static KvRelation load_kv(py::handle h, uint64_t id, size_t nk) {
  KvRelation r;
  r.id = id;
  r.n_keys = nk;
  for (auto item : h) {
    auto t = item.cast<py::tuple>();
    r.kv.emplace_back(t[0].cast<std::string>(), t[1].cast<std::string>());
  }
  std::sort(r.kv.begin(), r.kv.end());
  return r;
}

struct PyHnswIndex {
  StagedHnswIndex ix;
  void stage(const PyRelation& base, py::handle idx_rows, py::dict mf) {
    HnswIndexManifest m;
    m.vec_dim = mf["dim"].cast<size_t>();
    m.m_neighbours = mf["m"].cast<size_t>();
    m.ef_construction = mf["ef_construction"].cast<size_t>();
    m.vec_fields = mf["fields"].cast<std::vector<size_t>>();
    std::string dist = mf.contains("distance") ? mf["distance"].cast<std::string>() : "L2";
    if (dist == "L2") m.distance = HnswDistance::L2;
    else if (dist == "Cosine") m.distance = HnswDistance::Cosine;
    else if (dist == "IP") m.distance = HnswDistance::InnerProduct;
    else throw CozoError("", "Invalid distance: " + dist);  // sys.rs:584-590
    std::string dt = mf.contains("dtype") ? mf["dtype"].cast<std::string>() : "F32";
    if (dt == "F64" || dt == "Double") m.dtype_f64 = true;
    else if (dt != "F32" && dt != "Float") throw CozoError("", "Invalid dtype: " + dt);  // sys.rs:567-573
    m.derive();
    ix.stage(base.rel, to_rows(idx_rows), m);
  }
  // the same from KV bytes: lists of (key bytes, value bytes) as a storage range scan yields them
  void stage_kv(py::handle base_kv, uint64_t base_id, size_t n_keys, py::handle idx_kv, uint64_t idx_id, py::dict mf) {
    KvRelation b = load_kv(base_kv, base_id, n_keys), i = load_kv(idx_kv, idx_id, 0);
    ix.stage_kv(b, i, manifest_of(mf));
  }
  static HnswIndexManifest manifest_of(py::dict mf) {
    HnswIndexManifest m;
    m.vec_dim = mf["dim"].cast<size_t>();
    m.m_neighbours = mf["m"].cast<size_t>();
    m.ef_construction = mf["ef_construction"].cast<size_t>();
    m.vec_fields = mf["fields"].cast<std::vector<size_t>>();
    std::string dist = mf.contains("distance") ? mf["distance"].cast<std::string>() : "L2";
    if (dist == "L2") m.distance = HnswDistance::L2;
    else if (dist == "Cosine") m.distance = HnswDistance::Cosine;
    else if (dist == "IP") m.distance = HnswDistance::InnerProduct;
    else throw CozoError("", "Invalid distance: " + dist);
    if (mf.contains("keep_pruned_connections")) m.keep_pruned_connections = mf["keep_pruned_connections"].cast<bool>();
    m.derive();
    return m;
  }
  void build(const PyRelation& base, py::dict mf) { ix.build(base.rel, manifest_of(mf)); }
  void put_rows(PyRelation& base, py::handle rows, py::object filter) {
    std::function<bool(const Tuple&)> f;
    if (!filter.is_none()) f = [filter](const Tuple& t) { return filter(from_tuple(t)).cast<bool>(); };
    ix.put_rows(base.rel, to_rows(rows), f);
  }
  void remove_rows(PyRelation& base, py::handle rows) { ix.remove_rows(base.rel, to_rows(rows)); }
  void compact() { ix.compact(); }
  py::list to_index_rows(const PyRelation& base) const { return from_rows(ix.to_index_rows(base.rel)); }
  py::dict info() const {
    py::dict d;
    d["n_vectors"] = ix.keys.size();
    d["edges_kept"] = ix.n_edges_kept;
    d["dropped_same_key"] = ix.n_rows_dropped_same_key;
    d["dropped_ignore_link"] = ix.n_rows_dropped_ignored;
    d["put_unchanged"] = ix.n_put_unchanged;
    d["put_updated"] = ix.n_put_updated;
    d["put_appended"] = ix.n_put_appended;
    d["put_inserted"] = ix.n_put_inserted;
    d["removed"] = ix.n_removed;
    d["rebuilt"] = ix.n_rebuilt;
    return d;
  }
};

// a StagePlan as plain Python objects (host-only: no device call), for the planner equivalence tests
static py::dict plan_to_py(const StagePlan& pl) {
  py::dict d;
  py::list keys;
  for (auto& ck : pl.keys) keys.append(py::make_tuple(from_tuple(std::get<0>(ck)), std::get<1>(ck), std::get<2>(ck)));
  d["keys"] = keys;
  d["entry"] = pl.entry;
  d["n_levels"] = pl.n_levels;
  py::list ni, rp, ci;
  for (uint32_t L = 0; L < pl.n_levels; ++L) {
    ni.append(py::array_t<uint32_t>(pl.node_ids[L].size(), pl.node_ids[L].data()));
    rp.append(py::array_t<uint64_t>(pl.row_ptr[L].size(), pl.row_ptr[L].data()));
    ci.append(py::array_t<uint32_t>(pl.col_idx[L].size(), pl.col_idx[L].data()));
  }
  d["node_ids"] = ni;
  d["row_ptr"] = rp;
  d["col_idx"] = ci;
  d["vectors"] = py::array_t<float>(pl.vectors.size(), pl.vectors.data());
  d["edges_kept"] = pl.n_edges_kept;
  d["dropped_same_key"] = pl.n_rows_dropped_same_key;
  d["dropped_ignore_link"] = pl.n_rows_dropped_ignored;
  return d;
}

struct PyHnswSearchRA {
  HnswSearchRA ra;
  std::shared_ptr<PyRelation> base;
  std::shared_ptr<PyHnswIndex> index;
  PyHnswSearchRA(std::shared_ptr<PyRelation> b, std::shared_ptr<PyHnswIndex> ix, size_t k, size_t ef, py::object radius,
                 bool bind_field, bool bind_field_idx, bool bind_distance, bool bind_vector, py::object filter,
                 size_t bind_idx, bool filter_reads_distance)
      : base(std::move(b)), index(std::move(ix)) {
    ra.hnsw_search.base_handle = &base->rel;
    ra.hnsw_search.index = &index->ix;
    ra.hnsw_search.k = k;
    ra.hnsw_search.ef = ef;
    if (!radius.is_none()) ra.hnsw_search.radius = radius.cast<double>();
    ra.hnsw_search.bind_field = bind_field;
    ra.hnsw_search.bind_field_idx = bind_field_idx;
    ra.hnsw_search.bind_distance = bind_distance;
    ra.hnsw_search.bind_vector = bind_vector;
    if (!filter.is_none()) {
      py::function f = filter.cast<py::function>();
      ra.hnsw_search.filter = [f](const Tuple& t) { return f(from_tuple(t)).cast<bool>(); };
    }
    ra.bind_idx = bind_idx;
    ra.hnsw_search.filter_reads_distance = filter_reads_distance;
  }
  py::list iter(py::handle parent) { return from_rows(ra.iter(to_rows(parent))); }
  py::dict stats() const {
    py::dict d;
    d["n_queries"] = ra.last_stats.n_queries;
    d["dist_evals"] = ra.last_stats.dist_evals;
    d["nodes_expanded"] = ra.last_stats.nodes_expanded;
    d["kernel_ms"] = ra.last_stats.kernel_ms;
    return d;
  }
};

PYBIND11_MODULE(_cozo_host, m) {
  m.doc() = "test harness over the C++ host mirror of cozo's FixedRule / HnswSearchRA interfaces";
  static py::exception<CozoError> exc(m, "CozoError");
  py::register_exception_translator([](std::exception_ptr p) {
    try {
      if (p) std::rethrow_exception(p);
    } catch (const CozoError& e) {
      py::object ex = py::handle(exc.ptr())(e.what());
      ex.attr("code") = py::str(e.code);
      PyErr_SetObject(exc.ptr(), ex.ptr());
    }
  });
  m.def("init", [](int dev) { gpu_check(cozo_gpu_init(dev)); });
  py::class_<Poison, std::shared_ptr<Poison>>(m, "Poison").def(py::init<>()).def("kill", &Poison::kill);
  py::class_<PyDb>(m, "Db")
      .def(py::init<>())
      .def("run_fixed_rule", &PyDb::run_fixed_rule, py::arg("name"), py::arg("inputs"), py::arg("options") = py::dict(),
           py::arg("head_arity") = 0, py::arg("input_arities") = std::vector<size_t>(),
           py::arg("poison") = std::shared_ptr<Poison>())
      .def("register_fixed_rule", &PyDb::register_fixed_rule)
      .def("unregister_fixed_rule", &PyDb::unregister_fixed_rule);
  py::class_<PyRelation, std::shared_ptr<PyRelation>>(m, "Relation")
      .def(py::init<const std::string&, std::vector<std::string>, std::vector<std::string>>())
      .def("put", &PyRelation::put)
      .def("__len__", &PyRelation::size);
  py::class_<PyHnswIndex, std::shared_ptr<PyHnswIndex>>(m, "HnswIndex")
      .def(py::init<>())
      .def("stage", &PyHnswIndex::stage)
      .def("stage_kv", &PyHnswIndex::stage_kv)
      .def("build", &PyHnswIndex::build)
      .def("put_rows", &PyHnswIndex::put_rows, py::arg("base"), py::arg("rows"), py::arg("filter") = py::none())
      .def("remove_rows", &PyHnswIndex::remove_rows)
      .def("compact", &PyHnswIndex::compact)
      .def("to_index_rows", &PyHnswIndex::to_index_rows)
      .def("info", &PyHnswIndex::info)
      .def_property(
          "insert_inside", [](const PyHnswIndex& p) { return p.ix.insert_inside; },
          [](PyHnswIndex& p, bool v) { p.ix.insert_inside = v; });
  py::class_<PyHnswSearchRA>(m, "HnswSearchRA")
      .def(py::init<std::shared_ptr<PyRelation>, std::shared_ptr<PyHnswIndex>, size_t, size_t, py::object, bool, bool,
                    bool, bool, py::object, size_t, bool>(),
           py::arg("base"), py::arg("index"), py::arg("k"), py::arg("ef"), py::arg("radius") = py::none(),
           py::arg("bind_field") = false, py::arg("bind_field_idx") = false, py::arg("bind_distance") = false,
           py::arg("bind_vector") = false, py::arg("filter") = py::none(), py::arg("bind_idx") = 0,
           py::arg("filter_reads_distance") = true)
      .def("iter", &PyHnswSearchRA::iter)
      .def("stats", &PyHnswSearchRA::stats);
  m.def("cmp", [](py::handle a, py::handle b) { return cmp(to_dv(a), to_dv(b)); });
  // memcmp key codec (data/memcmp.rs, data/tuple.rs)
  m.def("memcmp_encode_value", [](py::handle v) {
    std::string o;
    memcmp_codec::encode_datavalue(o, to_dv(v));
    return py::bytes(o);
  });
  m.def("memcmp_decode_value", [](py::bytes b) {
    std::string s = b;
    DataValue v;
    size_t used = memcmp_codec::decode_datavalue(reinterpret_cast<const uint8_t*>(s.data()), s.size(), v);
    return py::make_tuple(from_dv(v), used);
  });
  m.def("memcmp_encode_bytes", [](py::bytes b) {
    std::string o;
    memcmp_codec::encode_bytes(o, b);
    return py::bytes(o);
  });
  m.def("memcmp_decode_bytes", [](py::bytes b) {
    std::string s = b, key;
    size_t used = memcmp_codec::decode_bytes(reinterpret_cast<const uint8_t*>(s.data()), s.size(), key);
    return py::make_tuple(py::bytes(key), used);
  });
  m.def("memcmp_encode_key", [](py::handle tuple, uint64_t rel) { return py::bytes(memcmp_codec::encode_as_key(to_tuple(tuple), rel)); });
  m.def("memcmp_decode_key", [](py::bytes b) { return from_tuple(memcmp_codec::decode_tuple_from_key(b)); });
  // msgpack value codec (runtime/relation.rs:275-296, 526-531; rmp-serde 1.2.0 — parity unpinned)
  m.def("msgpack_encode_value", [](py::handle v) {
    std::string o;
    msgpack_codec::encode_datavalue(o, to_dv(v));
    return py::bytes(o);
  });
  m.def("msgpack_decode_value", [](py::bytes b, bool lenient) {
    std::string s = b;
    msgpack_codec::Reader r(reinterpret_cast<const uint8_t*>(s.data()), s.size());
    DataValue v = msgpack_codec::decode_datavalue(r, lenient);
    return py::make_tuple(from_dv(v), (size_t)(r.p - reinterpret_cast<const uint8_t*>(s.data())));
  }, py::arg("data"), py::arg("lenient") = true);
  m.def("msgpack_skip", [](py::bytes b) {
    std::string s = b;
    msgpack_codec::Reader r(reinterpret_cast<const uint8_t*>(s.data()), s.size());
    r.skip();
    return (size_t)(r.p - reinterpret_cast<const uint8_t*>(s.data()));
  });
  m.def("encode_vals", [](py::handle tuple, size_t start, uint64_t rel) {
    return py::bytes(msgpack_codec::encode_vals(to_tuple(tuple), start, rel));
  });
  m.def("decode_tuple_from_kv", [](py::bytes k, py::bytes v) { return from_tuple(decode_tuple_from_kv(k, v)); });
  m.def("extract_vector", [](py::bytes v, size_t col, int32_t sub, size_t dim) {
    py::array_t<float> out(dim);
    msgpack_codec::extract_vector(v, col, sub, out.mutable_data(), dim);
    return out;
  });
  // staging plans (host only): from tuples, from KV bytes via tuples, from KV bytes directly
  m.def("plan_stage", [](const PyRelation& base, py::handle idx_rows, py::dict mf) {
    HnswIndexManifest m = PyHnswIndex::manifest_of(mf);
    const RelationHandle& rel = base.rel;
    return plan_to_py(StagedHnswIndex::plan_with(rel.keys.size(), to_rows(idx_rows), m, [&](const CompoundKey& ck, float* out) {
      const Tuple* row = rel.get(std::get<0>(ck));
      if (!row) throw CozoError("", "Cannot find compound key for HNSW");
      const DataValue* field = &(*row)[std::get<1>(ck)];
      if (std::get<2>(ck) >= 0) field = &field->list.at((size_t)std::get<2>(ck));
      if (field->kind != DataValue::Vec || field->v->size() != m.vec_dim) throw CozoError("", "Cannot interpret value as vector");
      std::copy(field->v->begin(), field->v->end(), out);
    }));
  });
  m.def("plan_stage_kv", [](py::handle base_kv, uint64_t base_id, size_t n_keys, py::handle idx_kv, uint64_t idx_id, py::dict mf,
                            bool bytes_level) {
    KvRelation b = load_kv(base_kv, base_id, n_keys), i = load_kv(idx_kv, idx_id, 0);
    HnswIndexManifest m = PyHnswIndex::manifest_of(mf);
    return plan_to_py(bytes_level ? StagedHnswIndex::plan_kv_bytes(b, i, m) : StagedHnswIndex::plan_kv_tuples(b, i, m));
  }, py::arg("base_kv"), py::arg("base_id"), py::arg("n_keys"), py::arg("idx_kv"), py::arg("idx_id"), py::arg("mf"),
     py::arg("bytes_level") = true);
  // FixedRule output: RegularTempStore::put per row vs the sorted bulk fill (n rows (string key, score))
  m.def("bench_tempstore_fill", [](uint32_t n) {
    std::vector<DataValue> keys;
    keys.reserve(n);
    char buf[32];
    for (uint32_t i = 0; i < n; ++i) {
      snprintf(buf, sizeof buf, "node%010u", (unsigned)((uint64_t)i * 2654435761u % 4000000007u));
      keys.push_back(DataValue::from_str(buf));
    }
    std::map<DataValue, uint32_t, DataValueLess> dict;  // the glue's key -> id dictionary
    for (uint32_t i = 0; i < n; ++i) dict.emplace(keys[i], i);
    auto t0 = std::chrono::steady_clock::now();
    RegularTempStore a;
    for (uint32_t i = 0; i < n; ++i) a.put({keys[i], DataValue::from_float(0.5 * i)});
    auto t1 = std::chrono::steady_clock::now();
    RegularTempStore b;
    std::vector<uint32_t> order;
    order.reserve(n);
    for (auto& kv : dict) order.push_back(kv.second);
    b.put_sorted_bulk(order.size(), [&](size_t i) { return Tuple{keys[order[i]], DataValue::from_float(0.5 * order[i])}; });
    auto t2 = std::chrono::steady_clock::now();
    bool same = a.inner.size() == b.inner.size();
    if (same) {
      auto ia = a.inner.begin();
      auto ib = b.inner.begin();
      for (; ia != a.inner.end(); ++ia, ++ib)
        if (cmp_tuple(ia->first, ib->first) != 0) same = false;
    }
    py::dict d;
    d["rows"] = n;
    d["put_s"] = std::chrono::duration<double>(t1 - t0).count();
    d["bulk_s"] = std::chrono::duration<double>(t2 - t1).count();
    d["identical"] = same;
    return d;
  });
  // throughput of the two KV planners on a synthetic index (n vectors, `deg` neighbours each, int keys)
  m.def("bench_stage_kv", [](uint32_t n, uint32_t dim, uint32_t deg, bool bytes_level) {
    RelationHandle base;
    base.name = "b";
    base.keys = {"k"};
    base.non_keys = {"v"};
    std::vector<Tuple> idx_rows;
    uint64_t x = 88172645463325252ull;
    auto rnd = [&]() { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
    for (uint32_t i = 0; i < n; ++i) {
      std::vector<float> v(dim);
      for (auto& e : v) e = (float)(rnd() % 1000) / 1000.f;
      base.put({DataValue::from_int(i), DataValue::from_vec(std::move(v))});
      auto row = [&](uint32_t to, double d, bool self) {
        return Tuple{DataValue::from_int(0), DataValue::from_int(i), DataValue::from_int(1), DataValue::from_int(-1),
                     DataValue::from_int(to), DataValue::from_int(1), DataValue::from_int(-1), DataValue::from_float(d),
                     self ? DataValue::from_bytes(std::string(32, 'h')) : DataValue::null(), DataValue::from_bool(false)};
      };
      idx_rows.push_back(row(i, (double)deg, true));
      for (uint32_t j = 0; j < deg; ++j) {
        uint32_t to = (uint32_t)(rnd() % n);
        if (to != i) idx_rows.push_back(row(to, 0.5, false));
      }
    }
    Tuple canary{DataValue::from_int(1)};
    for (int c = 0; c < 6; ++c) canary.push_back(DataValue::null());
    canary.push_back(DataValue::from_int(0));
    canary.push_back(DataValue::from_bytes("c"));
    canary.push_back(DataValue::from_bool(false));
    idx_rows.push_back(canary);
    KvRelation bkv = KvRelation::encode(base, 11), ikv;
    ikv.id = 12;
    for (auto& t : idx_rows) {
      Tuple k(t.begin(), t.begin() + 7);
      ikv.kv.emplace_back(memcmp_codec::encode_as_key(k, 12), msgpack_codec::encode_vals(t, 7, 12));
    }
    std::sort(ikv.kv.begin(), ikv.kv.end());
    ikv.kv.erase(std::unique(ikv.kv.begin(), ikv.kv.end(), [](auto& a, auto& b) { return a.first == b.first; }), ikv.kv.end());
    HnswIndexManifest m;
    m.vec_dim = dim;
    m.m_neighbours = deg / 2;
    m.vec_fields = {1};
    m.derive();
    size_t bytes = 0;
    for (auto& kv : ikv.kv) bytes += kv.first.size() + kv.second.size();
    for (auto& kv : bkv.kv) bytes += kv.first.size() + kv.second.size();
    auto t0 = std::chrono::steady_clock::now();
    StagePlan pl = bytes_level ? StagedHnswIndex::plan_kv_bytes(bkv, ikv, m) : StagedHnswIndex::plan_kv_tuples(bkv, ikv, m);
    double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    py::dict d;
    d["index_rows"] = ikv.kv.size();
    d["vectors"] = pl.keys.size();
    d["edges_kept"] = pl.n_edges_kept;
    d["kv_bytes"] = bytes;
    d["seconds"] = s;
    d["index_rows_per_s"] = (double)ikv.kv.size() / s;
    return d;
  });
  // Node id assignment of as_directed_graph on the host, the way it ran before the device took it over: a
  // std::map<DataValue, u32> lookup per endpoint in first-appearance order (fixed_rule/mod.rs:164-179).  Also times the
  // memcmp encoding of the same endpoints that cozo_gpu_graph_stage_keys receives instead, and returns it.
  // `keys`: the 2m endpoint keys, an int64 numpy array (Int values, built on the fly) or any sequence of values.
  m.def("bench_id_assign", [](py::object keys, bool run_map) {
    std::vector<DataValue> vals;
    py::array_t<int64_t> ints;
    const bool is_int = py::isinstance<py::array>(keys) && py::array(keys).dtype().kind() == 'i';
    if (is_int) ints = py::array_t<int64_t, py::array::c_style | py::array::forcecast>::ensure(keys);
    else vals = to_tuple(keys);
    const size_t E = is_int ? (size_t)ints.size() : vals.size();
    const int64_t* ip = is_int ? ints.data() : nullptr;
    auto key = [&](size_t i) { return is_int ? DataValue::from_int(ip[i]) : vals[i]; };
    py::dict d;
    d["endpoints"] = E;
    d["map_s"] = py::none();
    if (run_map) {
      auto t0 = std::chrono::steady_clock::now();
      std::map<DataValue, uint32_t, DataValueLess> inv;
      std::vector<DataValue> indices;
      std::vector<uint32_t> ids(E);
      for (size_t i = 0; i < E; ++i) {
        DataValue k = key(i);
        auto it = inv.find(k);
        if (it != inv.end()) {
          ids[i] = it->second;
          continue;
        }
        ids[i] = (uint32_t)indices.size();
        inv.emplace(k, ids[i]);
        indices.push_back(std::move(k));
      }
      d["map_s"] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      d["distinct"] = indices.size();
    }
    auto t0 = std::chrono::steady_clock::now();
    std::string kb;
    py::array_t<uint64_t> ko(E + 1);
    uint64_t* o = ko.mutable_data();
    o[0] = 0;
    for (size_t i = 0; i < E; ++i) {
      memcmp_codec::encode_datavalue(kb, key(i));
      o[i + 1] = kb.size();
    }
    d["encode_s"] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    py::array_t<uint8_t> kba(std::max<size_t>(kb.size(), 1));
    std::copy(kb.begin(), kb.end(), kba.mutable_data());
    d["key_bytes"] = kba;
    d["key_off"] = ko;
    return d;
  }, py::arg("keys"), py::arg("run_map") = true);
  // a graph rule end to end through the host mirror on Int-keyed edges (rows built here, not timed):
  // as_graph's scan + encoding + device staging + the rule + the RegularTempStore fill
  m.def("bench_rule_int_edges", [](const std::string& name, py::array_t<int64_t, py::array::c_style | py::array::forcecast> src,
                                   py::array_t<int64_t, py::array::c_style | py::array::forcecast> dst, py::dict options) {
    std::vector<std::vector<Tuple>> ins(1);
    ins[0].reserve(src.size());
    for (ssize_t e = 0; e < src.size(); ++e)
      ins[0].push_back({DataValue::from_int(src.data()[e]), DataValue::from_int(dst.data()[e])});
    Options opts;
    for (auto kv : options) opts[kv.first.cast<std::string>()] = to_dv(kv.second);
    FixedRuleRegistry reg;
    auto t0 = std::chrono::steady_clock::now();
    std::vector<Tuple> rows = reg.run(name, ins, {2}, std::move(opts), 0, Poison());
    py::dict d;
    d["seconds"] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    d["rows"] = rows.size();
    return d;
  });
  m.def("relation_to_kv",[](const PyRelation& rel, uint64_t id) {
    KvRelation r = KvRelation::encode(rel.rel, id);
    py::list out;
    for (auto& kv : r.kv) out.append(py::make_tuple(py::bytes(kv.first), py::bytes(kv.second)));
    return out;
  });
  m.def("rows_to_kv", [](py::handle rows, size_t n_keys, uint64_t id) {
    py::list out;
    for (auto& t : to_rows(rows)) {
      Tuple k(t.begin(), t.begin() + n_keys);
      out.append(py::make_tuple(py::bytes(memcmp_codec::encode_as_key(k, id)), py::bytes(msgpack_codec::encode_vals(t, n_keys, id))));
    }
    return out;
  });
  m.def("sha256_le_f32", [](py::array_t<float, py::array::c_style | py::array::forcecast> a) {
    return py::bytes(sha256_le_f32(std::vector<float>(a.data(), a.data() + a.size())));
  });
}
