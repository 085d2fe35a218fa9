"""ctypes binding of libcozo_gpu.so (include/cozo_gpu.h).

This is the Python twin of the Rust `extern "C"` block shown in INTEGRATION.md;
tests, bench.py and smoke() drive the product exclusively through it.  The
library is loaded from cozo_b200/csrc (in-tree) and there is no fallback: if it
is missing or no sm_90 device is usable, calls raise CozoGpuError.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libcozo_gpu.so")

NONE = 0xFFFFFFFF
L2, COSINE, IP = 0, 1, 2
E_INVAL, E_CUDA, E_NODEV, E_NOMEM, E_KILLED, E_UNSUP = -1, -2, -3, -4, -5, -6

# every symbol include/cozo_gpu.h declares
EXPORTS = [
    "cozo_gpu_init", "cozo_gpu_shutdown", "cozo_gpu_last_error", "cozo_gpu_device_count", "cozo_gpu_set_option",
    "cozo_gpu_get_option", "cozo_gpu_hnsw_stage", "cozo_gpu_hnsw_free", "cozo_gpu_hnsw_search",
    "cozo_gpu_hnsw_search_dev", "cozo_gpu_hnsw_search_scatter_dev", "cozo_gpu_hnsw_build", "cozo_gpu_hnsw_insert", "cozo_gpu_hnsw_insert_at", "cozo_gpu_hnsw_remove", "cozo_gpu_hnsw_compact", "cozo_gpu_hnsw_update", "cozo_gpu_hnsw_info", "cozo_gpu_hnsw_level_size",
    "cozo_gpu_hnsw_export_level", "cozo_gpu_hnsw_export_level_dist", "cozo_gpu_hnsw_export_live", "cozo_gpu_hnsw_vectors_dev", "cozo_gpu_topk_merge_dev", "cozo_gpu_graph_stage",
    "cozo_gpu_graph_free", "cozo_gpu_graph_export", "cozo_gpu_pagerank", "cozo_gpu_sssp_multi", "cozo_gpu_closeness",
    "cozo_gpu_betweenness", "cozo_gpu_clustering", "cozo_gpu_sssp_paths", "cozo_gpu_sssp_goals",
    "cozo_gpu_shards_unique_id", "cozo_gpu_shards_init", "cozo_gpu_shards_free", "cozo_gpu_shards_info",
    "cozo_gpu_hnsw_stage_sharded", "cozo_gpu_hnsw_search_sharded", "cozo_gpu_hnsw_search_sharded_dev",
    "cozo_gpu_hnsw_search_filtered", "cozo_gpu_hnsw_search_filtered_dev", "cozo_gpu_hnsw_search_f64",
    "cozo_gpu_graph_stage_keys", "cozo_gpu_graph_node_endpoints", "cozo_gpu_graph_lookup_keys",
    "cozo_gpu_hnsw_search_sharded_filtered", "cozo_gpu_hnsw_search_sharded_filtered_dev",
    "cozo_gpu_hnsw_search_sharded_f64",
]
UID_BYTES = 128


class CozoGpuError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"cozo_gpu error {code}: {msg}")
        self.code = code
        self.msg = msg


class HnswLevel(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("node_ids", C.c_void_p), ("row_ptr", C.c_void_p), ("col_idx", C.c_void_p)]


class HnswStageDesc(C.Structure):
    _fields_ = [("n_vectors", C.c_uint32), ("dim", C.c_uint32), ("metric", C.c_int32), ("n_levels", C.c_uint32),
                ("levels", C.POINTER(HnswLevel)), ("vectors", C.c_void_p), ("vectors_on_device", C.c_int32),
                ("entry_point", C.c_uint32), ("m_max0", C.c_uint32), ("m_max", C.c_uint32), ("vec_dtype", C.c_int32)]


class SearchStats(C.Structure):
    _fields_ = [("n_queries", C.c_uint64), ("dist_evals", C.c_uint64), ("nodes_expanded", C.c_uint64),
                ("nbr_reads", C.c_uint64), ("kernel_ms", C.c_double)]


class HnswBuildDesc(C.Structure):
    _fields_ = [("n_vectors", C.c_uint32), ("dim", C.c_uint32), ("metric", C.c_int32), ("vectors", C.c_void_p),
                ("vectors_on_device", C.c_int32), ("borrow_vectors", C.c_int32), ("m_neighbours", C.c_uint32),
                ("ef_construction", C.c_uint32), ("extend_candidates", C.c_int32),
                ("keep_pruned_connections", C.c_int32), ("level_seed", C.c_uint64), ("max_batch", C.c_uint32)]


_lib = None


def load():
    """Load the shared library (no GPU needed for loading)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CozoGpuError(E_NODEV, f"{LIB_PATH} is missing: run `python -m cozo_b200.build` (no CPU fallback exists)")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i64, f64 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int64, C.c_double
    L.cozo_gpu_init.argtypes = [C.c_int]
    L.cozo_gpu_last_error.restype = C.c_char_p
    L.cozo_gpu_set_option.argtypes = [C.c_char_p, i64]
    L.cozo_gpu_get_option.argtypes = [C.c_char_p]
    L.cozo_gpu_get_option.restype = i64
    L.cozo_gpu_hnsw_stage.argtypes = [C.POINTER(vp), C.POINTER(HnswStageDesc)]
    L.cozo_gpu_hnsw_free.argtypes = [vp]
    L.cozo_gpu_hnsw_free.restype = None
    L.cozo_gpu_hnsw_search.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, C.POINTER(SearchStats)]
    L.cozo_gpu_hnsw_search_dev.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_search_scatter_dev.argtypes = [vp, vp, u32, u32, u32, f64, u32, vp, vp, u32, vp, vp]
    L.cozo_gpu_hnsw_build.argtypes = [C.POINTER(vp), C.POINTER(HnswBuildDesc)]
    L.cozo_gpu_hnsw_insert.argtypes = [vp, vp, u32, C.c_int32, u32, C.c_int32, vp]
    L.cozo_gpu_hnsw_insert_at.argtypes = [vp, vp, vp, u32, C.c_int32, u32, C.c_int32, vp]
    L.cozo_gpu_hnsw_remove.argtypes = [vp, vp, u32]
    L.cozo_gpu_hnsw_compact.argtypes = [vp, vp]
    L.cozo_gpu_hnsw_update.argtypes = [vp, vp, vp, u32, u32, C.c_int32]
    L.cozo_gpu_hnsw_info.argtypes = [vp, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_level_size.argtypes = [vp, u32, vp, vp]
    L.cozo_gpu_hnsw_export_level.argtypes = [vp, u32, vp, vp, vp]
    L.cozo_gpu_hnsw_export_level_dist.argtypes = [vp, u32, vp]
    L.cozo_gpu_hnsw_export_live.argtypes = [vp, vp]
    L.cozo_gpu_hnsw_vectors_dev.argtypes = [vp, vp]
    L.cozo_gpu_hnsw_vectors_dev.restype = vp
    L.cozo_gpu_topk_merge_dev.argtypes = [vp, vp, u32, u32, u32, vp, vp, vp, vp]
    L.cozo_gpu_graph_stage.argtypes = [C.POINTER(vp), u32, u64, vp, vp, vp]
    L.cozo_gpu_graph_stage_keys.argtypes = [C.POINTER(vp), u64, vp, vp, vp, C.c_int32, vp]
    L.cozo_gpu_graph_node_endpoints.argtypes = [vp, vp]
    L.cozo_gpu_graph_lookup_keys.argtypes = [vp, vp, vp, u32, vp]
    L.cozo_gpu_graph_free.argtypes = [vp]
    L.cozo_gpu_graph_free.restype = None
    L.cozo_gpu_graph_export.argtypes = [vp, vp, vp, vp, vp, vp]
    L.cozo_gpu_pagerank.argtypes = [vp, C.c_float, f64, u32, vp, vp, vp, vp, vp]
    L.cozo_gpu_sssp_multi.argtypes = [vp, vp, u32, vp, vp, vp, vp]
    L.cozo_gpu_closeness.argtypes = [vp, vp, vp, vp]
    L.cozo_gpu_betweenness.argtypes = [vp, vp, vp, vp]
    L.cozo_gpu_clustering.argtypes = [vp, vp, vp, vp, vp, vp]
    L.cozo_gpu_sssp_paths.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.cozo_gpu_sssp_goals.argtypes = [vp, vp, u32, vp, u32, C.c_int32, vp, vp, vp, u64, vp, vp, u64, vp, vp]
    L.cozo_gpu_hnsw_search_filtered.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp, C.POINTER(SearchStats)]
    L.cozo_gpu_hnsw_search_filtered_dev.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_search_f64.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp, C.POINTER(SearchStats)]
    L.cozo_gpu_shards_unique_id.argtypes = [vp]
    L.cozo_gpu_shards_init.argtypes = [C.POINTER(vp), vp, C.c_int, C.c_int]
    L.cozo_gpu_shards_free.argtypes = [vp]
    L.cozo_gpu_shards_free.restype = None
    L.cozo_gpu_shards_info.argtypes = [vp, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_stage_sharded.argtypes = [vp, vp, vp, vp]
    L.cozo_gpu_hnsw_search_sharded.argtypes = [vp, vp, u32, u32, u32, f64, C.c_int, vp, vp, vp, C.POINTER(SearchStats)]
    L.cozo_gpu_hnsw_search_sharded_dev.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_search_sharded_filtered.argtypes = [vp, vp, u32, u32, u32, f64, C.c_int, vp, vp, vp, vp,
                                                        C.POINTER(SearchStats)]
    L.cozo_gpu_hnsw_search_sharded_filtered_dev.argtypes = [vp, vp, u32, u32, u32, f64, vp, vp, vp, vp, vp]
    L.cozo_gpu_hnsw_search_sharded_f64.argtypes = [vp, vp, u32, u32, u32, f64, C.c_int, vp, vp, vp, vp,
                                                   C.POINTER(SearchStats)]
    _lib = L
    return L


def _check(rc: int):
    if rc != 0:
        raise CozoGpuError(rc, load().cozo_gpu_last_error().decode("utf-8", "replace"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def init(device: int = 0):
    _check(load().cozo_gpu_init(device))


def device_count() -> int:
    return load().cozo_gpu_device_count()


def set_option(name: str, value: int):
    _check(load().cozo_gpu_set_option(name.encode(), int(value)))


def get_option(name: str) -> int:
    return load().cozo_gpu_get_option(name.encode())


def pack_row_mask(row_pass) -> np.ndarray:
    """bool[n] -> u32 words, bit (id & 31) of word id >> 5"""
    b = np.ascontiguousarray(row_pass, bool)
    words = np.zeros((b.size + 31) // 32 + 1, np.uint32)
    packed = np.packbits(b, bitorder="little")
    words.view(np.uint8)[:packed.size] = packed
    return words


class HnswIndex:
    """Owner of a cozo_gpu_hnsw_t handle."""

    def __init__(self, handle, dim, keep=None):
        self._h = handle
        self.dim = dim
        self._keep = keep

    # -- staging from per-level CSR (levels[0] = layer 0) ---------------------
    @classmethod
    def stage(cls, vectors: np.ndarray, node_ids, row_ptr, col_idx, entry, metric=L2, m_max0=0, m_max=0,
              vectors_dev_ptr: int | None = None, n_vectors: int | None = None, dim: int | None = None):
        L = load()
        nl = len(row_ptr)
        lv = (HnswLevel * nl)()
        keep = []
        for i in range(nl):
            rp = np.ascontiguousarray(row_ptr[i], np.uint64)
            ci = np.ascontiguousarray(col_idx[i], np.uint32)
            keep += [rp, ci]
            lv[i].n_nodes = len(rp) - 1
            lv[i].row_ptr = rp.ctypes.data
            lv[i].col_idx = ci.ctypes.data if ci.size else None
            if i > 0:
                ni = np.ascontiguousarray(node_ids[i], np.uint32)
                keep.append(ni)
                lv[i].node_ids = ni.ctypes.data if ni.size else None
        d = HnswStageDesc()
        if vectors_dev_ptr is None:
            f64 = np.asarray(vectors).dtype == np.float64         # an F64 index (VecElementType::F64)
            vectors = np.ascontiguousarray(vectors, np.float64 if f64 else np.float32)
            keep.append(vectors)
            d.n_vectors, d.dim = vectors.shape
            d.vectors = vectors.ctypes.data
            d.vectors_on_device = 0
            d.vec_dtype = 1 if f64 else 0
        else:
            d.n_vectors, d.dim = n_vectors, dim
            d.vectors = vectors_dev_ptr
            d.vectors_on_device = 1
        d.metric = metric
        d.n_levels = nl
        d.levels = lv
        d.entry_point = NONE if entry is None else int(entry)
        d.m_max0, d.m_max = m_max0, m_max
        h = C.c_void_p()
        _check(L.cozo_gpu_hnsw_stage(C.byref(h), C.byref(d)))
        return cls(h, d.dim)

    # -- construction on the device ---------------------------------------------
    @classmethod
    def build(cls, vectors: np.ndarray | None, metric=L2, m=16, ef_construction=200, keep_pruned_connections=False,
              level_seed=0x5EED0003, max_batch=0, vectors_dev_ptr: int | None = None, n_vectors: int | None = None,
              dim: int | None = None, borrow=False, extend_candidates=False):
        L = load()
        d = HnswBuildDesc()
        keep = None
        if vectors_dev_ptr is None:
            vectors = np.ascontiguousarray(vectors, np.float32)
            keep = vectors
            d.n_vectors, d.dim = vectors.shape
            d.vectors = vectors.ctypes.data
            d.vectors_on_device = 0
        else:
            d.n_vectors, d.dim = n_vectors, dim
            d.vectors = vectors_dev_ptr
            d.vectors_on_device = 1
            d.borrow_vectors = int(borrow)
        d.metric = metric
        d.m_neighbours = m
        d.ef_construction = ef_construction
        d.extend_candidates = int(extend_candidates)
        d.keep_pruned_connections = int(keep_pruned_connections)
        d.level_seed = level_seed
        d.max_batch = max_batch
        h = C.c_void_p()
        _check(L.cozo_gpu_hnsw_build(C.byref(h), C.byref(d)))
        return cls(h, d.dim, keep)

    def insert(self, vectors: np.ndarray, ef_construction: int = 0, keep_pruned_connections: int = -1) -> int:
        """hnsw_put of new rows (ids appended); returns the first new id"""
        vectors = np.ascontiguousarray(vectors, np.float32).reshape(-1, self.dim)
        first = C.c_uint32()
        _check(load().cozo_gpu_hnsw_insert(self._h, _p(vectors), vectors.shape[0], 0, ef_construction,
                                           keep_pruned_connections, C.byref(first)))
        return first.value

    def insert_at(self, positions, vectors: np.ndarray, ef_construction: int = 0,
                  keep_pruned_connections: int = -1) -> np.ndarray:
        """hnsw_put of new rows at any key position: positions[i] = ids whose key sorts before row i (non-decreasing).
        Existing ids move up to keep dense ids in key order; returns the new rows' ids (positions[i] + i)."""
        positions = np.ascontiguousarray(positions, np.uint32)
        vectors = np.ascontiguousarray(vectors, np.float32).reshape(positions.size, self.dim)
        out = np.zeros(positions.size, np.uint32)
        _check(load().cozo_gpu_hnsw_insert_at(self._h, _p(positions), _p(vectors), positions.size, 0, ef_construction,
                                              keep_pruned_connections, _p(out)))
        return out

    def update(self, ids, vectors, ef_construction: int = 0, keep_pruned_connections: int = -1):
        """hnsw_put of changed vectors under existing ids (remove + insert again, hnsw.rs:175-182)"""
        ids = np.ascontiguousarray(ids, np.uint32)
        vectors = np.ascontiguousarray(vectors, np.float32).reshape(ids.size, self.dim)
        _check(load().cozo_gpu_hnsw_update(self._h, _p(ids), _p(vectors), ids.size, ef_construction,
                                           keep_pruned_connections))

    def remove(self, ids):
        ids = np.ascontiguousarray(ids, np.uint32)
        _check(load().cozo_gpu_hnsw_remove(self._h, _p(ids), ids.size))

    def compact(self) -> np.ndarray:
        """drop every removed id; live ids move down in key order.  Returns old_to_new (NONE for a removed id)."""
        out = np.zeros(self.info()[0], np.uint32)
        _check(load().cozo_gpu_hnsw_compact(self._h, _p(out)))
        return out

    def info(self):
        n, dim, nl, ep = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        _check(load().cozo_gpu_hnsw_info(self._h, C.byref(n), C.byref(dim), C.byref(nl), C.byref(ep)))
        return n.value, dim.value, nl.value, (None if ep.value == NONE else ep.value)

    def export_levels(self):
        """-> (node_ids[list], row_ptr[list], col_idx[list], entry) with node_ids[0] = None."""
        L = load()
        _, _, nl, ep = self.info()
        node_ids, row_ptr, col_idx = [], [], []
        for lvl in range(nl):
            nn, ne = C.c_uint32(), C.c_uint64()
            _check(L.cozo_gpu_hnsw_level_size(self._h, lvl, C.byref(nn), C.byref(ne)))
            ni = np.zeros(nn.value, np.uint32)
            rp = np.zeros(nn.value + 1, np.uint64)
            ci = np.zeros(max(ne.value, 1), np.uint32)
            _check(L.cozo_gpu_hnsw_export_level(self._h, lvl, _p(ni), _p(rp), _p(ci)))
            node_ids.append(None if lvl == 0 else ni)
            row_ptr.append(rp)
            col_idx.append(ci[:ne.value])
        return node_ids, row_ptr, col_idx, ep

    def export_dists(self):
        """stored edge distances per layer, aligned with export_levels()' col_idx"""
        ni, rp, ci, ep = self.export_levels()
        out = []
        for lvl in range(len(ci)):
            d = np.zeros(max(ci[lvl].size, 1), np.float32)
            _check(load().cozo_gpu_hnsw_export_level_dist(self._h, lvl, _p(d)))
            out.append(d[:ci[lvl].size])
        return out

    def export_live(self):
        live = np.ones(self.info()[0], np.uint8)
        _check(load().cozo_gpu_hnsw_export_live(self._h, _p(live)))
        return live.astype(bool)

    def vectors_dev(self):
        stride = C.c_uint32()
        p = load().cozo_gpu_hnsw_vectors_dev(self._h, C.byref(stride))
        return p, stride.value

    def search(self, queries: np.ndarray, k: int, ef: int, radius: float | None = None, row_pass: np.ndarray | None = None):
        """Host-buffer call == the FFI the Rust HnswSearchRA glue makes.
        row_pass: optional bool[n] filter verdicts per indexed row (the filtered form, trim to k after the filter).
        -> ids[B,k] u32, dist[B,k] f32, count[B] u32, SearchStats"""
        queries = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        B = queries.shape[0]
        ids = np.empty((B, max(k, 1)), np.uint32)
        dist = np.empty((B, max(k, 1)), np.float32)
        cnt = np.zeros(B, np.uint32)
        st = SearchStats()
        r = -1.0 if radius is None else float(radius)
        if row_pass is None:
            _check(load().cozo_gpu_hnsw_search(self._h, _p(queries), B, k, ef, r, _p(ids), _p(dist), _p(cnt), C.byref(st)))
        else:
            mask = pack_row_mask(row_pass)
            _check(load().cozo_gpu_hnsw_search_filtered(self._h, _p(queries), B, k, ef, r, _p(mask), _p(ids), _p(dist),
                                                        _p(cnt), C.byref(st)))
        return ids, dist, cnt, st

    def search_f64(self, queries: np.ndarray, k: int, ef: int, radius: float | None = None, row_pass: np.ndarray | None = None):
        """hnsw_knn on an F64 index -> ids[B,k] u32, dist[B,k] f64, count[B], SearchStats"""
        queries = np.ascontiguousarray(queries, np.float64).reshape(-1, self.dim)
        B = queries.shape[0]
        ids = np.empty((B, max(k, 1)), np.uint32)
        dist = np.empty((B, max(k, 1)), np.float64)
        cnt = np.zeros(B, np.uint32)
        st = SearchStats()
        mask = None if row_pass is None else pack_row_mask(row_pass)
        _check(load().cozo_gpu_hnsw_search_f64(self._h, _p(queries), B, k, ef, -1.0 if radius is None else float(radius),
                                               _p(mask), _p(ids), _p(dist), _p(cnt), C.byref(st)))
        return ids, dist, cnt, st

    def search_dev(self, q_ptr: int, B: int, k: int, ef: int, ids_ptr: int, dist_ptr: int, count_ptr: int | None = None,
                   qstats_ptr: int | None = None, stream: int | None = None, radius: float | None = None):
        _check(load().cozo_gpu_hnsw_search_dev(self._h, q_ptr, B, k, ef, -1.0 if radius is None else float(radius),
                                               ids_ptr, dist_ptr, count_ptr, qstats_ptr, stream))

    def search_scatter_dev(self, q_ptr: int, B: int, k: int, ef: int, dest_ids_ptrs, dest_dist_ptrs, slot: int,
                           qstats_ptr: int | None = None, stream: int | None = None, radius: float | None = None):
        """fused search + exchange: top-k lists go straight into every destination's [S][B][k] buffers"""
        n = len(dest_ids_ptrs)
        ia = (C.c_uint64 * n)(*[int(x) for x in dest_ids_ptrs])
        da = (C.c_uint64 * n)(*[int(x) for x in dest_dist_ptrs])
        _check(load().cozo_gpu_hnsw_search_scatter_dev(self._h, q_ptr, B, k, ef, -1.0 if radius is None else float(radius),
                                                       n, ia, da, slot, qstats_ptr, stream))

    def close(self):
        if self._h:
            load().cozo_gpu_hnsw_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardGroup:
    """Owner of a cozo_gpu_shards_t: the ranks (one process per GPU) that hold the shards of one corpus.
    `uid` = ShardGroup.unique_id() of ONE rank, handed to the others by any host channel."""

    def __init__(self, uid: bytes, rank: int, world: int):
        assert len(uid) == UID_BYTES
        self._uid = (C.c_uint8 * UID_BYTES).from_buffer_copy(uid)
        h = C.c_void_p()
        _check(load().cozo_gpu_shards_init(C.byref(h), self._uid, rank, world))
        self._h = h
        self.rank, self.world = rank, world
        self.index = None
        self.offset = self.total_rows = 0

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_uint8 * UID_BYTES)()
        _check(load().cozo_gpu_shards_unique_id(buf))
        return bytes(buf)

    def attach(self, index: "HnswIndex"):
        """collective: this rank's shard; -> (global id of its row 0, rows of the whole corpus)"""
        off, tot = C.c_uint64(), C.c_uint64()
        _check(load().cozo_gpu_hnsw_stage_sharded(self._h, index._h, C.byref(off), C.byref(tot)))
        self.index = index
        self.offset, self.total_rows = off.value, tot.value
        return off.value, tot.value

    def info(self):
        r, w, x, t = C.c_int(), C.c_int(), C.c_int(), C.c_uint64()
        _check(load().cozo_gpu_shards_info(self._h, C.byref(r), C.byref(w), C.byref(x), C.byref(t)))
        return {"rank": r.value, "world": w.value, "exchange": "fused" if x.value else "nccl", "total_rows": t.value}

    def _search(self, fn, dtype, queries, k, ef, radius, root, B, row_pass, takes_mask):
        if queries is not None:
            queries = np.ascontiguousarray(queries, dtype).reshape(-1, self.index.dim)
            B = queries.shape[0]
        ids = np.empty((B, max(k, 1)), np.uint64)
        dist = np.empty((B, max(k, 1)), dtype)
        cnt = np.zeros(B, np.uint32)
        st = SearchStats()
        mask = None if row_pass is None else pack_row_mask(row_pass)
        args = (_p(mask),) if takes_mask else ()
        _check(fn(self._h, _p(queries), B, k, ef, -1.0 if radius is None else float(radius), root, *args, _p(ids),
                  _p(dist), _p(cnt), C.byref(st)))
        return ids, dist, cnt, st

    def search(self, queries, k: int, ef: int, radius: float | None = None, root: int = -1, B: int | None = None,
               row_pass=None):
        """collective host-buffer call -> global ids[B,k] u64 (UINT64_MAX padded), dist[B,k], count[B], stats.
        row_pass: optional bool[n_local] filter verdicts over this rank's rows (the filtered form)"""
        L = load()
        if row_pass is None:
            return self._search(L.cozo_gpu_hnsw_search_sharded, np.float32, queries, k, ef, radius, root, B, None,
                                False)
        return self._search(L.cozo_gpu_hnsw_search_sharded_filtered, np.float32, queries, k, ef, radius, root, B,
                            row_pass, True)

    def search_f64(self, queries, k: int, ef: int, radius: float | None = None, root: int = -1, B: int | None = None,
                   row_pass=None):
        """collective host-buffer call on a group of F64 shards -> global ids[B,k] u64, dist[B,k] f64, count[B], stats"""
        return self._search(load().cozo_gpu_hnsw_search_sharded_f64, np.float64, queries, k, ef, radius, root, B,
                            row_pass, True)

    def search_dev(self, q_ptr: int, B: int, k: int, ef: int, out_ids_ptr: int, out_dist_ptr: int,
                   qstats_ptr: int | None = None, stream: int | None = None, radius: float | None = None,
                   row_mask_ptr: int | None = None):
        """row_mask_ptr: device pointer of this rank's packed verdicts (pack_row_mask layout), the filtered form"""
        r = -1.0 if radius is None else float(radius)
        if row_mask_ptr is None:
            _check(load().cozo_gpu_hnsw_search_sharded_dev(self._h, q_ptr, B, k, ef, r, out_ids_ptr, out_dist_ptr,
                                                           qstats_ptr, stream))
        else:
            _check(load().cozo_gpu_hnsw_search_sharded_filtered_dev(self._h, q_ptr, B, k, ef, r, row_mask_ptr,
                                                                    out_ids_ptr, out_dist_ptr, qstats_ptr, stream))

    def close(self):
        if self._h:
            load().cozo_gpu_shards_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def topk_merge_dev(dist_ptr, ids_ptr, n_shards, B, k, offsets_ptr, out_ids_ptr, out_dist_ptr, stream=None):
    _check(load().cozo_gpu_topk_merge_dev(dist_ptr, ids_ptr, n_shards, B, k, offsets_ptr, out_ids_ptr, out_dist_ptr,
                                          stream))


class Graph:
    """Owner of a cozo_gpu_graph_t handle (dense u32 ids, optional f32 weights)."""

    def __init__(self, n: int, src, dst, w=None):
        src = np.ascontiguousarray(src, np.uint32)
        dst = np.ascontiguousarray(dst, np.uint32)
        w = None if w is None else np.ascontiguousarray(w, np.float32)
        self.n, self.m = int(n), int(src.size)
        self.weighted = w is not None
        h = C.c_void_p()
        _check(load().cozo_gpu_graph_stage(C.byref(h), n, src.size, _p(src), _p(dst), _p(w)))
        self._h = h

    @staticmethod
    def pack_keys(keys):
        """byte strings -> (bytes u8[], offsets u64[len+1]), the layout the key calls take"""
        keys = [bytes(k) for k in keys]
        off = np.zeros(len(keys) + 1, np.uint64)
        off[1:] = np.cumsum([len(k) for k in keys], dtype=np.uint64)
        return np.frombuffer(b"".join(keys) or b"\0", np.uint8).copy(), off

    @classmethod
    def from_keys(cls, key_bytes, key_off=None, w=None, undirected=False):
        """Stage from node KEYS: endpoint 2e is edge e's from key, 2e+1 its to key.  `key_bytes` is a list of 2m byte
        strings, or (with `key_off` [2m+1]) one u8 buffer.  Dense ids in first-appearance order; undirected mirrors
        every edge right after itself."""
        if key_off is None:
            key_bytes, key_off = cls.pack_keys(key_bytes)
        key_bytes = np.ascontiguousarray(key_bytes, np.uint8)
        key_off = np.ascontiguousarray(key_off, np.uint64)
        m = (key_off.size - 1) // 2
        w = None if w is None else np.ascontiguousarray(w, np.float32)
        g = cls.__new__(cls)
        h, n = C.c_void_p(), C.c_uint32()
        _check(load().cozo_gpu_graph_stage_keys(C.byref(h), m, _p(key_bytes), _p(key_off), _p(w), int(bool(undirected)),
                                                C.byref(n)))
        g._h = h
        g.n, g.m, g.weighted = n.value, 2 * m if undirected else m, w is not None
        return g

    def node_endpoints(self):
        """per dense id, the endpoint index where its key first appeared (graphs staged from keys)"""
        out = np.zeros(max(self.n, 1), np.uint64)
        _check(load().cozo_gpu_graph_node_endpoints(self._h, _p(out)))
        return out[:self.n]

    def lookup_keys(self, key_bytes, key_off=None):
        """dense id of every key (list of byte strings, or buffer + offsets); NONE where the graph has no such node"""
        if key_off is None:
            key_bytes, key_off = self.pack_keys(key_bytes)
        key_bytes = np.ascontiguousarray(key_bytes, np.uint8)
        key_off = np.ascontiguousarray(key_off, np.uint64)
        out = np.zeros(max(key_off.size - 1, 1), np.uint32)
        _check(load().cozo_gpu_graph_lookup_keys(self._h, _p(key_bytes), _p(key_off), key_off.size - 1, _p(out)))
        return out[:key_off.size - 1]

    def export(self):
        out_ptr = np.zeros(self.n + 1, np.uint32)
        in_ptr = np.zeros(self.n + 1, np.uint32)
        out_idx = np.zeros(self.m, np.uint32)
        in_idx = np.zeros(self.m, np.uint32)
        out_w = np.zeros(self.m, np.float32) if self.weighted else None
        _check(load().cozo_gpu_graph_export(self._h, _p(out_ptr), _p(out_idx), _p(out_w), _p(in_ptr), _p(in_idx)))
        return out_ptr, out_idx, out_w, in_ptr, in_idx

    def pagerank(self, damping=0.85, tol=1e-4, max_iter=10, poison=None):
        scores = np.zeros(self.n, np.float32)
        it, err, ms = C.c_uint32(), C.c_double(), C.c_double()
        _check(load().cozo_gpu_pagerank(self._h, float(np.float32(damping)), float(np.float32(tol)), max_iter,
                                        _p(scores), C.byref(it), C.byref(err), C.byref(ms), _p(poison)))
        return scores, it.value, err.value, ms.value

    def sssp(self, sources, want_pred=True, poison=None):
        sources = np.ascontiguousarray(sources, np.uint32)
        dist = np.zeros((sources.size, self.n), np.float32)
        pred = np.zeros((sources.size, self.n), np.uint32) if want_pred else None
        ms = C.c_double()
        _check(load().cozo_gpu_sssp_multi(self._h, _p(sources), sources.size, _p(dist), _p(pred), C.byref(ms),
                                          _p(poison)))
        return dist, pred, ms.value

    def closeness(self, poison=None):
        out = np.zeros(self.n, np.float32)
        ms = C.c_double()
        _check(load().cozo_gpu_closeness(self._h, _p(out), C.byref(ms), _p(poison)))
        return out, ms.value

    def betweenness(self, poison=None):
        out = np.zeros(self.n, np.float32)
        ms = C.c_double()
        _check(load().cozo_gpu_betweenness(self._h, _p(out), C.byref(ms), _p(poison)))
        return out, ms.value

    def sssp_paths(self, sources, goals, forb_nodes=None, forb_edges=None, max_len=64, poison=None):
        """batch of goal-directed searches; forb_nodes / forb_edges: per-search lists (or None).
        -> list of (cost, path list) ; unreachable = (inf, [])"""
        sources = np.ascontiguousarray(sources, np.uint32)
        goals = np.ascontiguousarray(goals, np.uint32)
        k = sources.size
        fnp = fnn = fep = fes = fed = None
        if forb_nodes is not None or forb_edges is not None:
            forb_nodes = forb_nodes or [[] for _ in range(k)]
            forb_edges = forb_edges or [[] for _ in range(k)]
            fnp = np.zeros(k + 1, np.uint32)
            fep = np.zeros(k + 1, np.uint32)
            fnp[1:] = np.cumsum([len(x) for x in forb_nodes])
            fep[1:] = np.cumsum([len(x) for x in forb_edges])
            fnn = np.array([v for x in forb_nodes for v in x] or [0], np.uint32)
            fes = np.array([e[0] for x in forb_edges for e in x] or [0], np.uint32)
            fed = np.array([e[1] for x in forb_edges for e in x] or [0], np.uint32)
        while True:
            cost = np.zeros(k, np.float32)
            ln = np.zeros(k, np.uint32)
            paths = np.zeros((k, max_len), np.uint32)
            ms = C.c_double()
            _check(load().cozo_gpu_sssp_paths(self._h, _p(sources), _p(goals), k, _p(fnp), _p(fnn), _p(fep), _p(fes),
                                              _p(fed), max_len, _p(cost), _p(ln), _p(paths), C.byref(ms), _p(poison)))
            if k == 0 or ln.max() <= max_len:
                break
            max_len = int(ln.max())
        return [(float(cost[i]), paths[i, :ln[i]].tolist()) for i in range(k)], ms.value

    def sssp_goals(self, sources, goals, keep_ties=False, poison=None, cap=None):
        """shortest paths from every source to the goals only; each search stops once its goals are settled.
        -> (costs f32 [n_src, n_goals], rows, kernel ms).  rows: without keep_ties, per pair (si, gi) the path list
        start..goal ([] when unreachable), as a list of n_src lists; with keep_ties, per source the tied-predecessor
        edges leading back from its goals, a u32 array [k, 2] of (v, p).  The first call has room for `cap` path nodes
        or tie edges (default: 64 per pair) and is repeated with the reported total when that is too small."""
        sources = np.ascontiguousarray(sources, np.uint32)
        goals = np.ascontiguousarray(goals, np.uint32)
        ns, ng = sources.size, goals.size
        cap = 64 * ns * ng if cap is None else int(cap)
        while True:
            cost = np.zeros((ns, ng), np.float32)
            off = np.zeros((ns + 1) if keep_ties else (ns * ng + 1), np.uint64)
            rows = np.zeros(max(cap, 1) * (2 if keep_ties else 1), np.uint32)
            ms = C.c_double()
            args = (None, None, 0, _p(off), _p(rows), cap) if keep_ties else (_p(off), _p(rows), cap, None, None, 0)
            _check(load().cozo_gpu_sssp_goals(self._h, _p(sources), ns, _p(goals), ng, int(bool(keep_ties)), _p(cost),
                                              *args, C.byref(ms), _p(poison)))
            if int(off[-1]) <= cap:
                break
            cap = int(off[-1])
        off = off.astype(np.int64)
        if keep_ties:
            edges = rows[:2 * off[-1]].reshape(-1, 2)
            return cost, [edges[off[i]:off[i + 1]] for i in range(ns)], ms.value
        paths = [rows[off[i]:off[i + 1]].tolist() for i in range(ns * ng)]
        return cost, [paths[i * ng:(i + 1) * ng] for i in range(ns)], ms.value

    def clustering(self, poison=None):
        cc = np.zeros(self.n, np.float64)
        nt = np.zeros(self.n, np.uint64)
        deg = np.zeros(self.n, np.uint64)
        ms = C.c_double()
        _check(load().cozo_gpu_clustering(self._h, _p(cc), _p(nt), _p(deg), C.byref(ms), _p(poison)))
        return cc, nt, deg, ms.value

    def close(self):
        if self._h:
            load().cozo_gpu_graph_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
