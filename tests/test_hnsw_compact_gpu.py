"""cozo_gpu_hnsw_compact: removed ids leave the handle.  Live id j becomes j - #{removed ids < j}, the upper-layer rows
of removed ids go too, and the map is monotone, so searches give the same answers through the map, bit for bit, with
the same traversal counters.  Sizes are small enough for the emulated library too."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_hnsw_insert_at_gpu import _edges, _levels_of, _relabel, _search_dev_stats
from tests.util import recall, uniform_vectors

pytestmark = pytest.mark.gpu
EMU = bool(os.environ.get("COZO_EMU_LIB"))
NONE = 0xFFFFFFFF
M, EFC = 8, 60


def _removal_set(g, n, seed):
    """a random tenth plus the entry point, several upper-layer nodes, id 0, the last id and a contiguous run"""
    rng = np.random.default_rng(seed)
    entry = g.info()[3]
    upper = np.flatnonzero(_levels_of(g) > 0)
    ids = set(rng.choice(n, n // 10, replace=False).tolist()) | {0, n - 1, entry}
    ids |= set(rng.choice(upper, min(6, upper.size), replace=False).tolist())
    ids |= set(range(n // 3, n // 3 + 40))
    return np.array(sorted(ids), np.uint32)


def _expected_map(n, dead):
    live = np.ones(n, bool)
    live[dead] = False
    m = np.full(n, NONE, np.int64)
    m[live] = np.arange(live.sum())
    return m, np.flatnonzero(live)


def _search_all(gpu, g, Q, k, ef, row_pass=None):
    out = []
    for mode in (0, 1, 2):
        gpu.set_option("hnsw.mode", mode)
        try:
            out.append(g.search(Q, k, ef, row_pass=row_pass))
        finally:
            gpu.set_option("hnsw.mode", -1)
    return out


def _assert_mapped(before, after, pi):
    """search answers of the compacted handle equal the earlier ones read through pi (old id -> new id)"""
    for (ib, db, cb, sb), (ia, da, ca, sa) in zip(before, after):
        assert np.array_equal(ca, cb)
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
        valid = np.arange(ib.shape[1])[None, :] < cb[:, None]
        assert np.all(pi[ib[valid].astype(np.int64)] != NONE)
        assert np.array_equal(ia[valid].astype(np.int64), pi[ib[valid].astype(np.int64)])
        assert np.all(ia[~valid] == NONE)
        assert (sa.dist_evals, sa.nodes_expanded, sa.nbr_reads) == (sb.dist_evals, sb.nodes_expanded, sb.nbr_reads)


def _assert_exports_mapped(before, after, pi):
    """export_level / export_level_dist after compaction = the earlier exports, removed rows dropped, ids mapped.  No
    kept row may name a removed id: hnsw_remove drops every edge into a removed node."""
    (ni0, rp0, ci0, ep0), d0 = before
    (ni1, rp1, ci1, ep1), d1 = after
    assert len(rp0) == len(rp1)
    assert ep1 == (None if ep0 is None else int(pi[ep0]))
    for L in range(len(rp0)):
        nodes = np.arange(rp0[0].size - 1) if L == 0 else ni0[L].astype(np.int64)
        deg = np.diff(rp0[L].astype(np.int64))
        keep = pi[nodes] != NONE
        assert np.all(deg[~keep] == 0)                      # a removed node's rows are empty
        assert np.all(pi[ci0[L].astype(np.int64)] != NONE)  # no kept row points at a removed id
        if L:
            assert np.array_equal(ni1[L].astype(np.int64), pi[nodes[keep]])
        assert np.array_equal(np.diff(rp1[L].astype(np.int64)), deg[keep])
        assert np.array_equal(ci1[L].astype(np.int64), pi[ci0[L].astype(np.int64)])
        assert np.array_equal(d1[L].view(np.uint32), d0[L].view(np.uint32))


def _compare_oracle(g, X, Q, k, ef, metric=O.L2):
    """the oracle's search on the exported graph: the usual parity"""
    ni, rp, ci, ep = g.export_levels()
    view = O.OracleHnsw.from_levels(X, O.HnswLevels(ni, rp, ci, ep), metric=metric)
    gi, gd, gc, _ = g.search(Q, k, ef)
    oi, od, oc, _ = view.search(Q, k, ef, n_threads=8)
    assert np.array_equal(gc, oc)
    assert recall(gi, oi) >= 0.999
    fin = np.isfinite(od)
    assert np.allclose(gd[fin], od[fin], rtol=1e-5, atol=1e-6)


def _exports(g):
    return g.export_levels(), g.export_dists()


CASES = [(O.L2, 48, 2000), (O.COSINE, 40, 1500), (O.IP, 36, 1500)]
if not EMU:
    CASES += [(O.L2, 768, 2500), (O.L2, 3072, 1200)]     # code rows and the pruned search; wide rows


@pytest.mark.parametrize("metric,dim,n", CASES)
def test_compact_is_exact_under_relabelling(gpu, metric, dim, n):
    X = uniform_vectors(n, dim, 8100 + dim)
    if metric == O.IP:
        X = X / np.linalg.norm(X, axis=1, keepdims=True)
    Q = uniform_vectors(120, dim, 8200 + dim)
    g = gpu.HnswIndex.build(X, metric=metric, m=M, ef_construction=EFC, level_seed=31)
    dead = _removal_set(g, n, dim)
    g.remove(dead)
    row_pass = np.random.default_rng(dim).random(n) < 0.7
    before = _search_all(gpu, g, Q, 10, 64)
    before_f = _search_all(gpu, g, Q, 10, 64, row_pass)
    ex_before, info_before = _exports(g), g.info()
    if not EMU:
        dev_before = _search_dev_stats(gpu, g, Q, 10, 64)
    pi = g.compact().astype(np.int64)
    want, live_ids = _expected_map(n, dead)
    assert np.array_equal(pi, want)
    n1, _, nl, ep = g.info()
    assert (n1, nl) == (live_ids.size, info_before[2]) and ep == pi[info_before[3]]
    assert g.export_live().all()
    _assert_mapped(before, _search_all(gpu, g, Q, 10, 64), pi)
    _assert_mapped(before_f, _search_all(gpu, g, Q, 10, 64, row_pass[live_ids]), pi)
    _assert_exports_mapped(ex_before, _exports(g), pi)
    if not EMU:
        ib, db, sb = dev_before
        ia, da, sa = _search_dev_stats(gpu, g, Q, 10, 64)
        assert np.array_equal(ia.astype(np.int64), np.where(ib == NONE, NONE, pi[np.minimum(ib, n - 1).astype(np.int64)]))
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
        assert np.array_equal(sa, sb)                      # word 3: f32 rows fetched past the moved code rows
    # the same graph staged from the exports and the live vectors searches bit for bit alike
    ni, rp, ci, ep = g.export_levels()
    s = gpu.HnswIndex.stage(X[live_ids], ni, rp, ci, ep, metric=metric, m_max0=2 * M, m_max=M)
    _assert_mapped(_search_all(gpu, g, Q, 10, 64), _search_all(gpu, s, Q, 10, 64), np.arange(live_ids.size))
    _compare_oracle(g, X[live_ids], Q, 10, 64, metric)


def test_small_chunks_give_the_same_handle(gpu):
    n, dim = 700, 20
    X = uniform_vectors(n, dim, 8300)
    handles = []
    for chunk in (1, 7, 0):
        g = gpu.HnswIndex.build(X, m=M, ef_construction=EFC, level_seed=3)
        g.remove(_removal_set(g, n, 1))
        gpu.set_option("hnsw.shift_chunk_rows", chunk)
        try:
            pi = g.compact()
        finally:
            gpu.set_option("hnsw.shift_chunk_rows", 0)
        handles.append((g, pi))
    Q = uniform_vectors(80, dim, 8301)
    g0, p0 = handles[-1]
    e0, ep0 = _edges(g0)
    r0 = _search_all(gpu, g0, Q, 10, 50)
    for g, pi in handles[:-1]:
        assert np.array_equal(pi, p0) and g.info() == g0.info()
        e, ep = _edges(g)
        assert ep == ep0
        for x, y in zip(e0, e):
            assert all(np.array_equal(a, b) for a, b in zip(x[:3], y[:3]))
            assert np.array_equal(x[3].view(np.uint32), y[3].view(np.uint32))
        _assert_mapped(r0, _search_all(gpu, g, Q, 10, 50), np.arange(g0.info()[0]))


def _top1_is_self(g, V, ids):
    i, d, _, _ = g.search(V, 1, 200)
    assert np.array_equal(i[:, 0].astype(np.int64), np.asarray(ids, np.int64))
    assert np.all(d[:, 0] == 0.0)


def test_maintenance_after_compaction(gpu):
    n, dim = 1500, 24
    X = uniform_vectors(n + 600, dim, 8400)
    Xk = X[:n].copy()                                      # vectors in id (= key) order
    g = gpu.HnswIndex.build(Xk, m=M, ef_construction=EFC, level_seed=8)
    dead = _removal_set(g, n, 2)
    g.remove(dead)
    g.compact()
    Xk = np.delete(Xk, dead, axis=0)
    # append
    V = X[n:n + 150]
    first = g.insert(V)
    assert first == Xk.shape[0]
    Xk = np.concatenate([Xk, V])
    _top1_is_self(g, V, first + np.arange(150))
    # inside the key range
    V = X[n + 150:n + 300]
    n0 = Xk.shape[0]
    P = np.sort(np.random.default_rng(4).integers(0, n0 + 1, 150)).astype(np.uint32)
    ids = g.insert_at(P, V)
    pi = _relabel(n0, P)
    assert np.array_equal(ids, pi[n0:])
    Xn = np.empty((n0 + 150, dim), np.float32)
    Xn[pi] = np.concatenate([Xk, V])
    Xk = Xn
    _top1_is_self(g, V, ids)
    # changed vectors, then removals and another compaction
    upd = np.random.default_rng(5).choice(Xk.shape[0], 100, replace=False).astype(np.uint32)
    g.update(upd, X[n + 300:n + 400])
    Xk[upd] = X[n + 300:n + 400]
    _top1_is_self(g, X[n + 300:n + 400], upd)
    dead = np.random.default_rng(6).choice(Xk.shape[0], 300, replace=False).astype(np.uint32)
    g.remove(dead)
    pi = g.compact().astype(np.int64)
    want, live_ids = _expected_map(Xk.shape[0], dead)
    assert np.array_equal(pi, want)
    Xk = Xk[live_ids]
    Q = uniform_vectors(100, dim, 8401)
    _compare_oracle(g, Xk, Q, 10, 64)
    V = X[n + 400:n + 600]
    first = g.insert(V)
    _top1_is_self(g, V, first + np.arange(200))
    _compare_oracle(g, np.concatenate([Xk, V]), Q, 10, 64)


def test_no_removed_ids_is_a_no_op(gpu):
    n, dim = 800, 16
    X = uniform_vectors(n, dim, 8500)
    g = gpu.HnswIndex.build(X, m=M, ef_construction=EFC, level_seed=9)
    before, info, ep = _edges(g)[0], g.info(), _edges(g)[1]
    assert np.array_equal(g.compact(), np.arange(n))
    after, ep_after = _edges(g)
    assert g.info() == info and ep_after == ep
    for x, y in zip(before, after):
        assert all(np.array_equal(a, b) for a, b in zip(x, y))
    # a staged handle has no build state: compacting it without removals leaves it so
    ix = O.OracleHnsw.new(n, dim, m=M, ef_construction=EFC)
    ix.insert_all(X)
    lv = ix.levels()
    s = gpu.HnswIndex.stage(X, lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, m_max0=2 * M, m_max=M)
    assert np.array_equal(s.compact(), np.arange(n))
    assert s.info() == (n, dim, lv.n_levels, lv.entry)


def test_every_id_removed_then_insert(gpu):
    n, dim = 600, 16
    X = uniform_vectors(n + 300, dim, 8600)
    g = gpu.HnswIndex.build(X[:n], m=M, ef_construction=EFC, level_seed=10)
    g.remove(np.arange(n, dtype=np.uint32))
    assert np.all(g.compact() == NONE)
    assert g.info() == (0, dim, 1, None)                  # as staged from the canary row alone
    ni, rp, ci, ep = g.export_levels()
    assert rp[0].size == 1 and ci[0].size == 0 and ep is None
    first = g.insert(X[n:])
    assert first == 0 and g.info()[0] == 300
    _top1_is_self(g, X[n:], np.arange(300))
    _compare_oracle(g, X[n:], uniform_vectors(80, dim, 8601), 10, 64)


def test_staged_handle(gpu):
    n, dim = 1200, 24
    X = uniform_vectors(n, dim, 8700)
    ix = O.OracleHnsw.new(n, dim, m=M, ef_construction=EFC)
    ix.insert_all(X)
    lv = ix.levels()
    g = gpu.HnswIndex.stage(X, lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, m_max0=2 * M, m_max=M)
    dead = _removal_set(g, n, 3)
    g.remove(dead)
    Q = uniform_vectors(100, dim, 8701)
    before, ex_before = _search_all(gpu, g, Q, 10, 64), _exports(g)
    pi = g.compact().astype(np.int64)
    assert np.array_equal(pi, _expected_map(n, dead)[0])
    _assert_mapped(before, _search_all(gpu, g, Q, 10, 64), pi)
    _assert_exports_mapped(ex_before, _exports(g), pi)


def test_borrowed_buffer_is_never_written(gpu):
    n, dim = 1000, 32
    X = uniform_vectors(n, dim, 8800)
    if EMU:
        keep = np.ascontiguousarray(X)
        ptr = keep.ctypes.data
        readback = lambda: keep  # noqa: E731
    else:
        import torch
        keep = torch.from_numpy(X).cuda()
        ptr = keep.data_ptr()
        readback = lambda: keep.cpu().numpy()  # noqa: E731
    g = gpu.HnswIndex.build(None, m=M, ef_construction=EFC, vectors_dev_ptr=ptr, n_vectors=n, dim=dim, borrow=True)
    dead = _removal_set(g, n, 4)
    g.remove(dead)
    Q = uniform_vectors(100, dim, 8801)
    before = _search_all(gpu, g, Q, 10, 64)
    pi = g.compact().astype(np.int64)
    assert np.array_equal(readback(), X)
    _assert_mapped(before, _search_all(gpu, g, Q, 10, 64), pi)
    _compare_oracle(g, X[_expected_map(n, dead)[1]], Q, 10, 64)


def test_errors(gpu):
    n, dim = 500, 16
    X = uniform_vectors(n, dim, 8900)
    assert gpu.load().cozo_gpu_hnsw_compact(None, None) == gpu.E_INVAL
    ix = O.OracleHnsw.new(n, dim, m=M, ef_construction=EFC)
    ix.insert_all(X)
    lv = ix.levels()
    g64 = gpu.HnswIndex.stage(X.astype(np.float64), lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, m_max0=2 * M, m_max=M)
    with pytest.raises(gpu.CozoGpuError) as e:
        g64.compact()
    assert e.value.code == gpu.E_UNSUP
    assert g64.info() == (n, dim, lv.n_levels, lv.entry)


@pytest.mark.skipif(EMU, reason="an asynchronous search on a torch stream needs a device")
def test_search_dev_enqueued_before_compact_sees_the_old_handle(gpu):
    import torch
    n, dim, B, k, ef = 20000, 128, 4096, 10, 200
    X = uniform_vectors(n, dim, 9000)
    Q = uniform_vectors(B, dim, 9001)
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=11)
    g.remove(_removal_set(g, n, 5))
    want_i, want_d, _, _ = g.search(Q, k, ef)
    dq = torch.from_numpy(Q).cuda()
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(10_000_000)                      # keep the search queued while compact starts
        g.search_dev(dq.data_ptr(), B, k, ef, ids.data_ptr(), dist.data_ptr(), stream=stream.cuda_stream)
    g.compact()                                            # no synchronise in between
    torch.cuda.synchronize()
    assert np.array_equal(ids.cpu().numpy().view(np.uint32), want_i)
    assert np.array_equal(dist.cpu().numpy().view(np.uint32), want_d.view(np.uint32))


def test_host_mirror_compact(gpu):
    from tests.hostmod import load
    h = load()
    h.init(0)
    n, dim = 600, 24
    X = uniform_vectors(n + 100, dim, 9100)
    mf = {"dim": dim, "m": M, "ef_construction": EFC, "fields": [1, 2]}
    name = lambda i: f"key{i:05d}"                                   # noqa: E731
    base = h.Relation("a", ["k"], ["v", "chunks"])
    for i in range(n):
        extra = [X[n + i // 50]] if i % 50 == 0 else []              # some rows carry several vectors
        base.put([name(2 * i), X[i], extra])
    index = h.HnswIndex()
    index.build(base, mf)
    index.insert_inside = True
    gone = [name(2 * i) for i in list(range(0, 30)) + list(range(100, n, 9))]
    index.remove_rows(base, [[k] for k in gone])
    n_before = index.info()["n_vectors"]
    index.compact()
    assert index.info()["n_vectors"] < n_before

    Q = uniform_vectors(60, dim, 9101)

    def answers(ix):
        out = h.HnswSearchRA(base, ix, k=5, ef=40, bind_distance=True, bind_idx=0).iter([[q] for q in Q])
        return [(r[1], r[4]) for r in out]

    fresh = h.HnswIndex()
    fresh.stage(base, index.to_index_rows(base), mf)
    assert fresh.info()["n_vectors"] == index.info()["n_vectors"]
    got = answers(index)
    assert got == answers(fresh) and len(got) == 300 and not ({k for k, _ in got} & set(gone))
    # new keys inside the range land at their key positions
    inside = [1, 61, 301, 2 * n - 3]
    index.put_rows(base, [[name(k), X[n + 60 + j], []] for j, k in enumerate(inside)])
    info = index.info()
    assert info["rebuilt"] == 0 and info["put_inserted"] == len(inside)
    hits = h.HnswSearchRA(base, index, k=1, ef=80, bind_distance=True, bind_idx=0).iter(
        [[v] for v in X[n + 60:n + 60 + len(inside)]])
    assert [(r[1], r[4]) for r in hits] == [(name(k), 0.0) for k in inside]
    fresh = h.HnswIndex()
    fresh.stage(base, index.to_index_rows(base), mf)
    assert answers(index) == answers(fresh)
