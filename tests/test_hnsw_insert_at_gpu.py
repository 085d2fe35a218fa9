"""cozo_gpu_hnsw_insert_at: hnsw_put of rows at any key position.  Existing ids move up so that dense ids stay in key
order, then the new ids are linked in one batched run.  The main check: on data without distance ties, insert_at(P, V)
gives the graph, entry, live flags and search results of insert(V) (an append), read through the relabelling
pi (old j -> j + #{P <= j}, appended row i -> P[i] + i).  Sizes are small enough for the emulated library too."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import uniform_vectors, recall

pytestmark = pytest.mark.gpu
EMU = bool(os.environ.get("COZO_EMU_LIB"))


def _relabel(n0, P):
    P = np.asarray(P, np.int64)
    old = np.arange(n0) + np.searchsorted(P, np.arange(n0), side="right")
    new = P + np.arange(P.size)
    return np.concatenate([old, new]).astype(np.int64)      # index: id in the appended handle


def _levels_of(g):
    """top layer of every id, from the export"""
    ni, rp, _, _ = g.export_levels()
    lv = np.zeros(rp[0].size - 1, np.int64)
    for L in range(1, len(rp)):
        lv[ni[L]] = L
    return lv


def _edges(g, pi=None):
    """every layer as sorted (node, neighbour, dist) triples, ids mapped through pi"""
    ni, rp, ci, ep = g.export_levels()
    ds = g.export_dists()
    out = []
    for L in range(len(rp)):
        nodes = np.arange(rp[0].size - 1) if L == 0 else ni[L].astype(np.int64)
        src = np.repeat(nodes, np.diff(rp[L].astype(np.int64)))
        dst = ci[L].astype(np.int64)
        if pi is not None:
            nodes, src, dst = pi[nodes], pi[src], pi[dst]
        o = np.lexsort((dst, src))
        out.append((np.sort(nodes), src[o], dst[o], ds[L][o]))
    return out, (None if ep is None else (ep if pi is None else int(pi[ep])))


def _assert_same_graph(a, b, pi=None):
    ea, epa = _edges(a)
    eb, epb = _edges(b, pi)
    assert epa == epb
    assert len(ea) == len(eb)
    for (na, sa, da, wa), (nb, sb, db, wb) in zip(ea, eb):
        assert np.array_equal(na, nb) and np.array_equal(sa, sb) and np.array_equal(da, db)
        assert np.array_equal(wa.view(np.uint32), wb.view(np.uint32))
    la, lb = a.export_live(), b.export_live()
    if pi is None:
        assert np.array_equal(la, lb)
    else:
        m = np.zeros_like(la)
        m[pi] = lb
        assert np.array_equal(la, m)


def _assert_same_search(a, b, Q, k, ef, pi=None):
    ia, da, ca, sa = a.search(Q, k, ef)
    ib, db, cb, sb = b.search(Q, k, ef)
    assert np.array_equal(ca, cb)
    assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
    valid = np.arange(k)[None, :] < cb[:, None]
    mapped = ib.astype(np.int64) if pi is None else pi[ib.astype(np.int64) * valid]
    assert np.array_equal(ia[valid].astype(np.int64), mapped[valid])
    assert (sa.dist_evals, sa.nodes_expanded, sa.nbr_reads) == (sb.dist_evals, sb.nodes_expanded, sb.nbr_reads)


def _search_dev_stats(gpu, g, Q, k, ef, mode=-1):
    import torch
    B = Q.shape[0]
    dq = torch.from_numpy(Q).cuda()
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    gpu.set_option("hnsw.mode", mode)
    try:
        g.search_dev(dq.data_ptr(), B, k, ef, ids.data_ptr(), dist.data_ptr(), qstats_ptr=qs.data_ptr(),
                     stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    finally:
        gpu.set_option("hnsw.mode", -1)
    return ids.cpu().numpy().view(np.uint32), dist.cpu().numpy(), qs.cpu().numpy().view(np.uint32)


def _assert_no_ties(X, Q, metric):
    """exact distance ties between an old and a new row may break differently in the two handles"""
    X64, Q64 = X.astype(np.float64), Q.astype(np.float64)
    for A, B in ((X64, X64), (Q64, X64)):
        if metric == O.L2:
            d = (A * A).sum(1)[:, None] + (B * B).sum(1)[None, :] - 2 * A @ B.T
        elif metric == O.COSINE:
            d = 1 - (A / np.linalg.norm(A, axis=1, keepdims=True)) @ (B / np.linalg.norm(B, axis=1, keepdims=True)).T
        else:
            d = 1 - A @ B.T
        s = np.sort(d, axis=1)
        assert np.all(np.diff(s[:, 1:], axis=1) > 0)


def _positions(rng, n0, lv_new, top, entry):
    """random non-decreasing positions with duplicates, 0 and n0; rows on the old top layer land after the entry"""
    c = lv_new.size
    P = np.sort(rng.integers(0, n0 + 1, c))
    P[: c // 10] = P[c // 10]                      # a run of duplicates
    P[0], P[-1] = 0, n0
    P[(lv_new == top) & (P <= entry)] = entry + 1
    return np.maximum.accumulate(P).astype(np.uint32)


CASES = [(O.L2, 48, 2500, 400), (O.COSINE, 40, 2000, 300), (O.IP, 36, 2000, 300)]
if not EMU:
    CASES.append((O.L2, 768, 3000, 500))           # code rows: the pruned search reads moved code rows


@pytest.mark.parametrize("metric,dim,n0,c", CASES)
def test_insert_at_equals_append_under_relabelling(gpu, metric, dim, n0, c):
    m, efc = 8, 60
    X = uniform_vectors(n0 + c, dim, 7100 + dim)
    if metric == O.IP:
        X = X / np.linalg.norm(X, axis=1, keepdims=True)
    X0, V = X[:n0], X[n0:]
    Q = uniform_vectors(150, dim, 7200 + dim)
    _assert_no_ties(X, Q, metric)
    a = gpu.HnswIndex.build(X0, metric=metric, m=m, ef_construction=efc, level_seed=21)
    b = gpu.HnswIndex.build(X0, metric=metric, m=m, ef_construction=efc, level_seed=21)
    dead = np.random.default_rng(3).choice(n0, 40, replace=False).astype(np.uint32)
    a.remove(dead)
    b.remove(dead)
    _, _, nl, entry = a.info()
    b.insert(V)
    lv_new = _levels_of(b)[n0:]
    P = _positions(np.random.default_rng(dim), n0, lv_new, nl - 1, entry)
    ids = a.insert_at(P, V)
    pi = _relabel(n0, P)
    assert np.array_equal(ids, pi[n0:])
    assert a.info()[0] == n0 + c
    _assert_same_graph(a, b, pi)
    _assert_same_search(a, b, Q, 10, 64, pi)
    if not EMU:
        ia, da, sa = _search_dev_stats(gpu, a, Q, 10, 64)
        ib, db, sb = _search_dev_stats(gpu, b, Q, 10, 64)
        assert np.array_equal(ia.astype(np.int64), pi[ib.astype(np.int64)])
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
        assert np.array_equal(sa, sb)                 # word 3: f32 rows fetched past the moved code rows
        if metric == O.L2 and dim >= 512:
            i0, d0, _ = _search_dev_stats(gpu, a, Q, 10, 64, mode=0)
            assert np.array_equal(i0, ia) and np.array_equal(d0.view(np.uint32), da.view(np.uint32))


def test_all_positions_at_n_is_insert(gpu):
    n0, c, dim = 2000, 300, 32
    X = uniform_vectors(n0 + c, dim, 7300)
    a = gpu.HnswIndex.build(X[:n0], m=8, ef_construction=60, level_seed=5)
    b = gpu.HnswIndex.build(X[:n0], m=8, ef_construction=60, level_seed=5)
    ids = a.insert_at(np.full(c, n0, np.uint32), X[n0:])
    assert b.insert(X[n0:]) == n0
    assert np.array_equal(ids, np.arange(n0, n0 + c))
    _assert_same_graph(a, b)
    _assert_same_search(a, b, uniform_vectors(100, dim, 7301), 10, 64)


def _compare_oracle(g, X, Q, k, ef):
    ni, rp, ci, ep = g.export_levels()
    view = O.OracleHnsw.from_levels(X, O.HnswLevels(ni, rp, ci, ep))
    gi, gd, gc, _ = g.search(Q, k, ef)
    oi, od, oc, _ = view.search(Q, k, ef, n_threads=8)
    assert np.array_equal(gc, oc)
    assert recall(gi, oi) >= 0.999
    fin = np.isfinite(od)
    assert np.allclose(gd[fin], od[fin], rtol=1e-5, atol=1e-6)


def test_new_node_before_the_entry_on_the_top_layer_becomes_the_entry(gpu):
    dim, n0, c, m = 16, 40, 200, 4
    X = uniform_vectors(n0 + c, dim, 7400)
    for seed in range(1, 200):
        probe = gpu.HnswIndex.build(X[:n0], m=m, ef_construction=40, level_seed=seed)
        top = probe.info()[2] - 1
        probe.insert(X[n0:])
        lv = _levels_of(probe)[n0:]
        if probe.info()[2] - 1 == top and (lv == top).any():
            break
    else:
        pytest.fail("no seed puts a new row on the old top layer")
    g = gpu.HnswIndex.build(X[:n0], m=m, ef_construction=40, level_seed=seed)
    old_entry = g.info()[3]
    ids = g.insert_at(np.zeros(c, np.uint32), X[n0:])          # every new key sorts first
    entry = g.info()[3]
    first_top = int(ids[np.flatnonzero(lv == top)[0]])
    assert entry == first_top and entry != old_entry + c
    ni, _, _, _ = g.export_levels()
    assert entry == ni[top].min()
    Xk = np.concatenate([X[n0:], X[:n0]])                      # vectors in key (= id) order
    _compare_oracle(g, Xk, uniform_vectors(100, dim, 7401), 10, 40)


def test_quality_after_inserting_a_fifth_inside(gpu):
    n, dim, m, efc = 5000, 32, 12, 80
    X = uniform_vectors(n, dim, 7500)                          # X in final key order
    rng = np.random.default_rng(9)
    new = np.sort(rng.choice(n, n // 5, replace=False))
    old = np.setdiff1d(np.arange(n), new)
    g = gpu.HnswIndex.build(X[old], m=m, ef_construction=efc, level_seed=13)
    P = (np.searchsorted(old, new)).astype(np.uint32)
    ids = g.insert_at(P, X[new])
    assert np.array_equal(ids, new)
    Q = uniform_vectors(300, dim, 7501)
    out = g.search(Q, 10, 80)
    bi, _ = O.bruteforce_knn(X, Q, 10, n_threads=8)
    full = gpu.HnswIndex.build(X, m=m, ef_construction=efc, level_seed=13)
    assert recall(out[0], bi) >= recall(full.search(Q, 10, 80)[0], bi) - 0.03
    _compare_oracle(g, X, Q[:100], 10, 80)


def test_small_shift_chunks_give_the_same_index(gpu):
    n0, c, dim = 1500, 200, 24
    X = uniform_vectors(n0 + c, dim, 7600)
    P = np.sort(np.random.default_rng(1).integers(0, n0 + 1, c)).astype(np.uint32)
    a = gpu.HnswIndex.build(X[:n0], m=8, ef_construction=50, level_seed=3)
    b = gpu.HnswIndex.build(X[:n0], m=8, ef_construction=50, level_seed=3)
    a.insert_at(P, X[n0:])
    gpu.set_option("hnsw.shift_chunk_rows", 3)
    try:
        b.insert_at(P, X[n0:])
    finally:
        gpu.set_option("hnsw.shift_chunk_rows", 0)
    _assert_same_graph(a, b)
    _assert_same_search(a, b, uniform_vectors(100, dim, 7601), 10, 50)


def test_insert_at_into_staged_empty_and_borrowed_handles(gpu):
    dim, m, n0, c = 32, 8, 1500, 300
    X = uniform_vectors(n0 + c, dim, 7700)
    P = np.sort(np.random.default_rng(2).integers(0, n0 + 1, c)).astype(np.uint32)
    pi = _relabel(n0, P)
    Xk = np.empty_like(X)
    Xk[pi] = X                                                 # vectors in key order after the insert
    Q = uniform_vectors(100, dim, 7701)
    # staged from the host: no degrees or stored distances on the device yet, no ef_construction
    ix = O.OracleHnsw.new(n0, dim, m=m, ef_construction=50)
    ix.insert_all(X[:n0])
    lv = ix.levels()
    g = gpu.HnswIndex.stage(X[:n0], lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, m_max0=2 * m, m_max=m)
    with pytest.raises(gpu.CozoGpuError):
        g.insert_at(P, X[n0:])
    g.insert_at(P, X[n0:], ef_construction=50, keep_pruned_connections=0)
    _compare_oracle(g, Xk, Q, 10, 50)
    # staged from the canary row alone: positions of 0
    e = O.OracleHnsw.new(4, dim, m=m, ef_construction=50).levels()
    g0 = gpu.HnswIndex.stage(X[:4], e.node_ids, e.row_ptr, e.col_idx, e.entry, m_max0=2 * m, m_max=m)
    ids = g0.insert_at(np.zeros(200, np.uint32), X[:200], ef_construction=50)
    assert np.array_equal(ids, np.arange(200))
    _compare_oracle(g0, X[:200], Q, 10, 50)
    # borrowed vectors are never written: insert_at takes a private copy first
    if EMU:
        buf = np.ascontiguousarray(X[:n0])
        ptr, keep = buf.ctypes.data, buf
        before = buf.copy()
        readback = lambda: keep  # noqa: E731
    else:
        import torch
        keep = torch.from_numpy(X[:n0]).cuda()
        ptr = keep.data_ptr()
        before = X[:n0].copy()
        readback = lambda: keep.cpu().numpy()  # noqa: E731
    gb = gpu.HnswIndex.build(None, m=m, ef_construction=50, vectors_dev_ptr=ptr, n_vectors=n0, dim=dim, borrow=True)
    gb.insert_at(P, X[n0:])
    assert np.array_equal(readback(), before)
    _compare_oracle(gb, Xk, Q, 10, 50)


def test_bad_positions_and_f64_leave_the_handle_unchanged(gpu):
    n0, dim = 1000, 16
    X = uniform_vectors(n0 + 10, dim, 7800)
    g = gpu.HnswIndex.build(X[:n0], m=8, ef_construction=40, level_seed=4)
    before_info, (before_edges, before_ep) = g.info(), _edges(g)
    bad = [np.array([5, 3] + [7] * 8, np.uint32), np.array([0] * 9 + [n0 + 1], np.uint32)]
    for P in bad:
        with pytest.raises(gpu.CozoGpuError) as e:
            g.insert_at(P, X[n0:])
        assert e.value.code == gpu.E_INVAL
        assert g.info() == before_info
        after_edges, after_ep = _edges(g)
        assert after_ep == before_ep
        for x, y in zip(before_edges, after_edges):
            assert all(np.array_equal(p, q) for p, q in zip(x, y))
    ix = O.OracleHnsw.new(n0, dim, m=8, ef_construction=40)
    ix.insert_all(X[:n0])
    lv = ix.levels()
    g64 = gpu.HnswIndex.stage(X[:n0].astype(np.float64), lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, m_max0=16, m_max=8)
    with pytest.raises(gpu.CozoGpuError) as e:
        g64.insert_at(np.zeros(10, np.uint32), X[n0:], ef_construction=40)
    assert e.value.code == gpu.E_UNSUP
    assert g64.info() == (n0, dim, lv.n_levels, lv.entry)


def _graph_sets(levels):
    ni, rp, ci, _ = levels
    out = []
    for L in range(len(rp)):
        nodes = np.arange(rp[L].size - 1) if L == 0 else ni[L]
        out.append({int(v): set(ci[L][int(rp[L][r]):int(rp[L][r + 1])].tolist()) for r, v in enumerate(nodes)})
    return out


@pytest.mark.parametrize("keep", [False, True])
def test_insert_at_matches_the_sequential_oracle_with_extend_candidates(gpu, keep):
    """extend_candidates links one node per batch, in the reference's order: insert_at must then build what the oracle's
    sequential hnsw_put builds when the old rows go in at their relabelled ids and the new rows at theirs, with the
    device's levels.  Criterion of the builder fidelity scenario: same layer memberships, >= 99 % identical rows."""
    dim, m, efc, n0, c = 16, 4, 12, 48, 20
    X = np.random.default_rng(n0 + keep).random((n0 + c, dim), dtype=np.float32)
    g = gpu.HnswIndex.build(X[:n0], m=m, ef_construction=efc, keep_pruned_connections=keep, level_seed=77, max_batch=1,
                            extend_candidates=True)
    P = np.sort(np.random.default_rng(5).integers(0, n0 + 1, c)).astype(np.uint32)
    P[0] = 0
    ids = g.insert_at(P, X[n0:])
    pi = _relabel(n0, P)
    assert np.array_equal(ids, pi[n0:])
    dev = g.export_levels()
    level = _levels_of(g)
    ix = O.OracleHnsw.new(n0 + c, dim, m=m, ef_construction=efc, keep_pruned_connections=keep, extend_candidates=True)
    for j in range(n0 + c):                      # old rows first, then the new rows, each at its id after the insert
        ix.insert(int(pi[j]), X[j], forced_level=-int(level[pi[j]]))
    lv = ix.levels()
    assert lv.entry == dev[3] and lv.n_levels == len(dev[1])
    dsets = _graph_sets(dev)
    osets = _graph_sets((lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry))
    assert all(sorted(a) == sorted(b) for a, b in zip(dsets, osets))
    same = sum(dsets[L][v] == osets[L][v] for L in range(len(dsets)) for v in dsets[L])
    total = sum(len(d) for d in dsets)
    assert same >= total - max(1, total // 100), (same, total)
