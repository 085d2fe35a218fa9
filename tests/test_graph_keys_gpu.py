"""Dense node ids assigned on the device from node keys (cozo_gpu_graph_stage_keys): ids, CSR, lookups and errors
against first-appearance dictionaries (fixed_rule/mod.rs:164-179), and every graph rule of the host mirror on a graph
whose keys mix every value kind, against the oracle run on the dictionary-derived dense graph."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.hostmod import load
from tests.util import rmat_edges

pytestmark = pytest.mark.gpu
EMU = bool(os.environ.get("COZO_EMU_LIB"))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def h(gpu):
    m = load()
    m.init(0)
    return m


def mixed_keys():
    """Null, Bool, 1 vs 1.0, -0.0 vs 0.0, NaN, i64 extremes, neighbouring ints above 2^53, strings sharing
    8/16/24-byte prefixes, embedded NUL, the empty string, bytes, nested lists, 4 KB keys"""
    p = "abcdefghijklmnopqrstuvwx"
    return [None, False, True, 0, 1, 1.0, -0.0, 0.0, float("nan"), float("inf"), -1.5, 2 ** 63 - 1, -2 ** 63,
            2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, -(2 ** 53) - 1, p[:8], p[:8] + "y", p[:16], p[:16] + "y", p, p + "y",
            p[:7], "a\0b", "a\0", "a", "", b"", b"a\0", b"\0" * 9, [], [1], [1.0], [1, "x"], [1, ["x"]], [[]],
            "k" * 4096, "k" * 4095 + "l", b"\x07" * 4096]


def first_appearance(enc):
    """the reference's dictionary over encoded endpoints -> (ids per endpoint, first endpoint per id)"""
    ids, first, out = {}, [], np.empty(len(enc), np.uint32)
    for i, k in enumerate(enc):
        if k not in ids:
            ids[k] = len(first)
            first.append(i)
        out[i] = ids[k]
    return out, np.array(first, np.uint64)


def dense_stream(eid, w, undirected):
    src, dst = eid[0::2], eid[1::2]
    if undirected:
        src, dst = np.stack([src, dst], 1).ravel(), np.stack([dst, src], 1).ravel()
        w = None if w is None else np.repeat(w, 2)
    return src, dst, w


def assert_same_csr(a, b):
    for x, y in zip(a.export(), b.export()):
        if x is None or y is None:
            assert x is None and y is None
        else:
            assert x.dtype == y.dtype and np.array_equal(x.view(np.uint32), y.view(np.uint32))


def check_ids(gpu, enc, w=None, undirected=False, packed=None):
    g = gpu.Graph.from_keys(*(packed or (enc,)), w=w, undirected=undirected)
    eid, first = first_appearance(enc)
    assert g.n == first.size
    assert np.array_equal(g.node_endpoints(), first)
    src, dst, ww = dense_stream(eid, w, undirected)
    assert_same_csr(g, gpu.Graph(first.size, src, dst, ww))
    return g, eid


def mixed_edges(h, seed, m=400):
    keys = mixed_keys()
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, len(keys), (m, 2))
    pick[:5, 1] = pick[:5, 0]                                          # self loops
    pick[5:10] = pick[10:15]                                           # parallel edges
    w = (rng.integers(1, 24, m) / 8.0).astype(np.float32)             # ties on purpose
    enc = [h.memcmp_encode_value(keys[k]) for k in pick.ravel()]
    return keys, pick, w, enc


def test_ids_air_routes(h, gpu):
    d = np.load(os.path.join(GOLDEN, "air_routes.npz"))
    codes = [str(c) for c in d["codes"]]
    enc_code = [h.memcmp_encode_value(c) for c in codes]
    enc = [enc_code[i] for pair in zip(d["fr"], d["to"]) for i in pair]
    for undirected in (False, True):
        g, _ = check_ids(gpu, enc, d["dist"], undirected)
        names = [codes[int((d["fr"], d["to"])[ep % 2][ep // 2])] for ep in g.node_endpoints()]
        seen = list(dict.fromkeys(c for pair in zip(d["fr"], d["to"]) for c in (codes[pair[0]], codes[pair[1]])))
        assert names == seen


@pytest.mark.parametrize("undirected", [False, True])
def test_ids_rmat16_int_keys(h, gpu, undirected):
    n, s, t = rmat_edges(16, 16, 7)
    perm = np.random.default_rng(8).permutation(n).astype(np.int64) * 7919 - (1 << 40)
    keys = np.stack([perm[s], perm[t]], 1).ravel()
    enc = [h.memcmp_encode_value(int(k)) for k in keys]
    g, eid = check_ids(gpu, enc, None, undirected)
    assert np.array_equal(keys[g.node_endpoints().astype(np.int64)], list(dict.fromkeys(keys.tolist())))


def test_ids_mixed_keys(h, gpu):
    keys, pick, w, enc = mixed_edges(h, 1)
    g, _ = check_ids(gpu, enc)
    got = [repr(keys[pick.ravel()[ep]]) for ep in g.node_endpoints()]
    assert got == list(dict.fromkeys(repr(keys[k]) for k in pick.ravel()))
    assert g.n == len({repr(k) for k in keys[:]} & {repr(keys[k]) for k in pick.ravel()})


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("undirected", [False, True])
def test_csr_matches_dense_staging(h, gpu, weighted, undirected):
    """parallel edges with different weights, self loops, every value kind"""
    keys, pick, w, enc = mixed_edges(h, 2, m=3000)
    check_ids(gpu, enc, w if weighted else None, undirected)
    # the same through one packed buffer whose first offset is not 0
    kb, ko = gpu.Graph.pack_keys(enc)
    kb = np.concatenate([np.full(5, 0xAB, np.uint8), kb])
    check_ids(gpu, enc, w if weighted else None, undirected, packed=(kb, ko + np.uint64(5)))


@pytest.mark.skipif(EMU, reason="67 M edges: too large for the emulated library")
def test_scale_rmat22_int64_keys(h, gpu):
    n, s, t = rmat_edges(22, 16, 3)
    perm = np.random.default_rng(4).permutation(n).astype(np.int64) * 1_000_003 + (1 << 50)
    keys = np.stack([perm[s], perm[t]], 1).ravel()
    enc = h.bench_id_assign(keys, False)
    kb, ko = enc["key_bytes"], enc["key_off"]
    uniq, first_idx, inv = np.unique(keys, return_index=True, return_inverse=True)
    rank = np.empty(uniq.size, np.uint32)
    rank[np.argsort(first_idx, kind="stable")] = np.arange(uniq.size, dtype=np.uint32)
    eid = rank[inv]
    g1 = gpu.Graph.from_keys(kb, ko)
    assert g1.n == uniq.size
    assert np.array_equal(g1.node_endpoints(), np.sort(first_idx).astype(np.uint64))
    ref = gpu.Graph(uniq.size, eid[0::2], eid[1::2])
    assert_same_csr(g1, ref)
    del ref
    g2 = gpu.Graph.from_keys(kb, ko)
    assert_same_csr(g1, g2)
    assert np.array_equal(g1.node_endpoints(), g2.node_endpoints())


def test_lookups(h, gpu):
    keys, pick, w, enc = mixed_edges(h, 3)
    g, _ = check_ids(gpu, enc)
    ids, _ = first_appearance(enc)
    present = {e: int(i) for e, i in zip(enc, ids)}
    q = list(present)
    assert g.lookup_keys(q).tolist() == [present[e] for e in q]
    absent = ["k" * 4096 + "m", "k" * 4095, "abcdefghijklmnopqrstuvwxz", "abcdefghijklmnop\0", 2 ** 53 + 3, -0.5,
              [1, "y"], [[1]], b"\0" * 8, "zzz", 3]
    absent = [h.memcmp_encode_value(a) for a in absent]
    absent = [a for a in absent if a not in present]
    assert len(absent) >= 8
    assert g.lookup_keys(absent).tolist() == [gpu.NONE] * len(absent)
    mixed = [x for pair in zip(q, absent) for x in pair]
    assert g.lookup_keys(mixed).tolist() == [present.get(e, gpu.NONE) for e in mixed]
    assert g.lookup_keys([]).size == 0
    with pytest.raises(gpu.CozoGpuError) as e:                          # dense-id graphs keep no keys
        gpu.Graph(3, [0, 1], [1, 2]).lookup_keys(q[:1])
    assert e.value.code == gpu.E_INVAL


def test_errors_and_empty(h, gpu):
    L = gpu.load()
    enc = [h.memcmp_encode_value(k) for k in ("a", "b", "b", "c")]
    kb, ko = gpu.Graph.pack_keys(enc)
    bad = ko.copy()
    bad[2] = bad[1] - 1
    with pytest.raises(gpu.CozoGpuError) as e:
        gpu.Graph.from_keys(kb, bad)
    assert e.value.code == gpu.E_INVAL and "decrease" in e.value.msg
    h_ = C.c_void_p()
    n = C.c_uint32()
    assert L.cozo_gpu_graph_stage_keys(C.byref(h_), 2, None, gpu._p(ko), None, 0, C.byref(n)) == gpu.E_INVAL
    assert L.cozo_gpu_graph_stage_keys(C.byref(h_), 2, gpu._p(kb), None, None, 0, C.byref(n)) == gpu.E_INVAL
    assert L.cozo_gpu_graph_stage_keys(None, 2, gpu._p(kb), gpu._p(ko), None, 0, C.byref(n)) == gpu.E_INVAL
    for badw in ([1.0, float("nan")], [-1.0, 1.0], [float("inf"), 0.0]):
        with pytest.raises(gpu.CozoGpuError) as e1:
            gpu.Graph.from_keys(enc, w=badw)
        with pytest.raises(gpu.CozoGpuError) as e2:
            gpu.Graph(3, [0, 1], [1, 2], badw)
        assert (e1.value.code, e1.value.msg) == (e2.value.code, e2.value.msg)
    for w in (None, np.zeros(0, np.float32)):
        g = gpu.Graph.from_keys([], w=w)
        assert g.n == 0 and g.node_endpoints().size == 0
        assert g.lookup_keys(enc).tolist() == [gpu.NONE] * 4
        out_ptr, out_idx, _, in_ptr, in_idx = g.export()
        assert out_ptr.tolist() == [0] and in_ptr.tolist() == [0] and out_idx.size == 0
        assert g.pagerank()[0].size == 0


# ---- every rule through the host mirror, keys of every kind --------------------------------------------------

def _rule_graph(h, seed, m=260):
    keys, pick, w, enc = mixed_edges(h, seed, m)
    # a stored relation is a set of tuples in key order: one row per (from, to, weight) is enough here
    rows = [[keys[a], keys[b], float(ww)] for (a, b), ww in zip(pick, w)]
    return keys, rows, enc


def _dense(h, rows, undirected=False, weighted=True):
    enc = [h.memcmp_encode_value(r[i]) for r in rows for i in (0, 1)]
    eid, first = first_appearance(enc)
    w = np.array([r[2] for r in rows], np.float32) if weighted else None
    src, dst, ww = dense_stream(eid, w, undirected)
    inv = [rows[int(ep) // 2][int(ep) % 2] for ep in first]
    ids = {e: int(i) for e, i in zip(enc, eid)}
    return ids, inv, O.OracleGraph(first.size, src, dst, ww)


def _k(h, v):
    return h.memcmp_encode_value(v)


def test_rules_on_mixed_keys(h, gpu):
    keys, rows, enc = _rule_graph(h, 5)
    db = h.Db()
    # PageRank (unweighted), both directions
    for undirected in (False, True):
        ids, inv, o = _dense(h, rows, undirected, weighted=False)
        out = db.run_fixed_rule("PageRank", [[r[:2] for r in rows]], {"undirected": undirected, "iterations": 20,
                                                                       "epsilon": 0.0}, head_arity=2)
        exp, _, _ = o.pagerank(0.85, 0.0, 20)
        assert len(out) == len(inv)
        for k, s in out:
            assert abs(s - exp[ids[_k(h, k)]]) <= 1e-5 * exp[ids[_k(h, k)]]
    ids, inv, o = _dense(h, rows)
    # closeness / betweenness
    cl, bt = o.closeness(n_threads=4), o.betweenness(n_threads=4)
    for k, c in db.run_fixed_rule("ClosenessCentrality", [rows], {}, head_arity=2):
        e = cl[ids[_k(h, k)]]
        assert (np.isfinite(c) == np.isfinite(e)) and (not np.isfinite(e) or abs(c - e) <= 1e-5 * abs(e) + 1e-7)
    for k, c in db.run_fixed_rule("BetweennessCentrality", [rows], {}, head_arity=2):
        assert abs(c - bt[ids[_k(h, k)]]) <= 1e-4 * abs(bt[ids[_k(h, k)]]) + 1e-4
    # clustering over the mirrored stream
    idsu, invu, ou = _dense(h, rows, True, weighted=False)
    cc, nt, deg = ou.clustering()
    out = db.run_fixed_rule("ClusteringCoefficients", [[r[:2] for r in rows]], {}, head_arity=4)
    assert len(out) == len(invu)
    for k, c, t, d in out:
        i = idsu[_k(h, k)]
        assert (c, t, d) == (cc[i], nt[i], deg[i])


def _tie_paths(bp, bi, s, t):
    """every path s -> t through the predecessor lists of the oracle's keep_ties search"""
    if t == s:
        return [[s]]
    out = []
    for p in bi[int(bp[t]):int(bp[t + 1])]:
        out += [q + [t] for q in _tie_paths(bp, bi, s, int(p))]
    return out


def test_dijkstra_and_yen_on_mixed_keys(h, gpu):
    keys, rows, enc = _rule_graph(h, 6)
    db = h.Db()
    ids, inv, o = _dense(h, rows)
    starts = [[inv[0]], [inv[3]], ["not-a-node"], [2 ** 53 + 7]]
    goals = [[r[1]] for r in rows[:6]] + [[b"absent"]]
    enck = lambda v: repr(_k(h, v))
    sids = sorted({ids[_k(h, s[0])] for s in starts if _k(h, s[0]) in ids})
    gids = sorted({ids[_k(h, g[0])] for g in goals if _k(h, g[0]) in ids})
    wmin = {}
    for a, b, ww in rows:
        kk = (enck(a), enck(b))
        wmin[kk] = min(wmin.get(kk, 1e30), ww)
    # plain: one shortest path per (start, goal)
    out = db.run_fixed_rule("ShortestPathDijkstra", [rows, starts, goals], {}, head_arity=4)
    assert len(out) == len(sids) * len(gids)
    for s, t, cost, path in out:
        d, _ = o.sssp([ids[_k(h, s)]])
        exp = float(d[0, ids[_k(h, t)]])
        if np.isinf(exp):
            assert np.isinf(cost) and path == []
            continue
        assert cost == exp and enck(path[0]) == enck(s) and enck(path[-1]) == enck(t)
        assert abs(sum(wmin[(enck(a), enck(b))] for a, b in zip(path, path[1:])) - cost) < 1e-4
    # keep_ties: every tied path
    out = db.run_fixed_rule("ShortestPathDijkstra", [rows, starts, goals], {"keep_ties": True}, head_arity=4)
    exp = set()
    for s in sids:
        d, bp, bi = o.sssp_keep_ties(s, gids)
        for t in gids:
            if np.isinf(d[t]):
                exp.add((enck(inv[s]), enck(inv[t]), float("inf"), ()))
            elif t != s:
                for p in _tie_paths(bp, bi, s, t):
                    exp.add((enck(inv[s]), enck(inv[t]), float(d[t]), tuple(enck(inv[u]) for u in p)))
    got = {(enck(s), enck(t), float(c), tuple(enck(u) for u in p)) for s, t, c, p in out}
    assert got == exp
    # Yen, with weights that leave no ties among the k shortest paths (the order of tied candidates is free)
    rng = np.random.default_rng(7)
    rows = [[a, b, float(np.float32(rng.random() * 10 + 0.5))] for a, b, _ in rows]
    ids, inv, o = _dense(h, rows)
    out = db.run_fixed_rule("KShortestPathYen", [rows, starts, goals], {"k": 3}, head_arity=4)
    exp = []
    for s in sids:
        for t in gids:
            for c, p in o.yen(s, t, 3):
                exp.append((enck(inv[s]), enck(inv[t]), float(c), tuple(enck(inv[u]) for u in p)))
    got = [(enck(s), enck(t), float(c), tuple(enck(u) for u in p)) for s, t, c, p in out]
    assert sorted(got) == sorted(exp)
