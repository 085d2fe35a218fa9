"""insert_at and compact relabel the handle's rows through one routine, in opposite directions.  A seeded interleaved
sequence runs on two handles built alike: A takes insert_at at random positions, removals and compactions; B appends the
same rows with insert, takes the same removals and is never compacted.  After every step A equals B read through the
accumulated id map (B id -> A id, NONE once compacted away): levels, edge distances, live flags, entry and searches.
A last update + compact on A is checked for its invariants only: update re-links contiguous id runs, which A and B
number differently.  Sizes are small enough for the emulated library too."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_hnsw_compact_gpu import _compare_oracle
from tests.test_hnsw_insert_at_gpu import (_assert_no_ties, _assert_same_search, _levels_of, _positions, _relabel,
                                           _search_dev_stats)
from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu
EMU = bool(os.environ.get("COZO_EMU_LIB"))
NONE = 0xFFFFFFFF
M, EFC = 8, 60


def _graph(g, pi=None):
    """every layer as sorted (nodes, src, dst, dist); with pi, ids go through pi and the nodes it drops must be empty"""
    ni, rp, ci, ep = g.export_levels()
    ds = g.export_dists()
    out = []
    for L in range(len(rp)):
        nodes = np.arange(rp[0].size - 1) if L == 0 else ni[L].astype(np.int64)
        deg = np.diff(rp[L].astype(np.int64))
        src, dst = np.repeat(nodes, deg), ci[L].astype(np.int64)
        if pi is not None:
            keep = pi[nodes] != NONE
            assert np.all(deg[~keep] == 0)
            nodes, src, dst = pi[nodes[keep]], pi[src], pi[dst]
        o = np.lexsort((dst, src))
        out.append((np.sort(nodes), src[o], dst[o], ds[L][o]))
    return out, (None if ep is None else (ep if pi is None else int(pi[ep])))


def _assert_no_removed_ids(g):
    live = g.export_live()
    _, rp, ci, _ = g.export_levels()
    for L in range(len(rp)):
        assert live[ci[L].astype(np.int64)].all()


def _assert_equal_through(gpu, a, b, pi, Q):
    """A = B read through pi"""
    _assert_no_removed_ids(a)
    _assert_no_removed_ids(b)
    (ea, epa), (eb, epb) = _graph(a), _graph(b, pi)
    assert epa == epb and len(ea) == len(eb)
    for (na, sa, da, wa), (nb, sb, db, wb) in zip(ea, eb):
        assert np.array_equal(na, nb) and np.array_equal(sa, sb) and np.array_equal(da, db)
        assert np.array_equal(wa.view(np.uint32), wb.view(np.uint32))
    la, lb = a.export_live(), b.export_live()
    kept = pi != NONE
    assert np.all(~lb[~kept])                                # only removed ids leave A
    m = np.zeros_like(la)
    m[pi[kept]] = lb[kept]
    assert kept.sum() == la.size and np.array_equal(la, m)
    _assert_same_search(a, b, Q, 10, 64, pi)
    if not EMU:
        ia, da, sa = _search_dev_stats(gpu, a, Q, 10, 64)
        ib, db, sb = _search_dev_stats(gpu, b, Q, 10, 64)
        assert np.array_equal(ia.astype(np.int64), np.where(ib == NONE, NONE, pi[np.minimum(ib, pi.size - 1)]))
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
        assert np.array_equal(sa, sb)                        # word 3: f32 rows fetched past the moved code rows


CASES = [(O.L2, 48, 0), (O.L2, 48, 1), (O.COSINE, 40, 3)]
if not EMU:
    CASES.append((O.L2, 768, 0))                             # code rows move too


@pytest.mark.parametrize("metric,dim,chunk", CASES)
def test_insert_at_and_compact_equal_append_through_the_map(gpu, metric, dim, chunk):
    n0, c, rounds = 1200, 150, 2
    X = uniform_vectors(n0 + (rounds + 1) * c + 100, dim, 9300 + dim + chunk)
    Q = uniform_vectors(100, dim, 9400 + dim)
    _assert_no_ties(X[:n0 + (rounds + 1) * c], Q, metric)
    a = gpu.HnswIndex.build(X[:n0], metric=metric, m=M, ef_construction=EFC, level_seed=41)
    b = gpu.HnswIndex.build(X[:n0], metric=metric, m=M, ef_construction=EFC, level_seed=41)
    pi = np.arange(n0, dtype=np.int64)                       # B id -> A id
    Xa = X[:n0].copy()                                       # A's vectors in A's id order
    rng = np.random.default_rng(dim + chunk)
    gpu.set_option("hnsw.shift_chunk_rows", chunk)
    try:
        def insert_at(lo):
            nonlocal pi, Xa
            V = X[lo:lo + c]
            nb = b.insert(V)
            na, _, nl, entry = a.info()
            P = _positions(rng, na, _levels_of(b)[nb:], nl - 1, entry)
            ids = a.insert_at(P, V)
            gap = _relabel(na, P)
            assert np.array_equal(ids, gap[na:])
            pi = np.concatenate([np.where(pi == NONE, NONE, gap[np.minimum(pi, na - 1)]), gap[na:]])
            Xn = np.empty((na + c, dim), np.float32)
            Xn[gap] = np.concatenate([Xa, V])
            Xa = Xn
            _assert_equal_through(gpu, a, b, pi, Q)

        def remove_and_compact():
            nonlocal pi, Xa
            live_b = np.flatnonzero(b.export_live())
            entry_b = b.info()[3]
            upper = np.intersect1d(np.flatnonzero(_levels_of(b) > 0), live_b)
            dead = set(rng.choice(live_b, live_b.size // 8, replace=False).tolist())
            dead |= set(rng.choice(upper, min(5, upper.size), replace=False).tolist())
            dead |= {int(live_b[0]), int(live_b[-1])}
            dead.discard(entry_b)                            # B and A would re-point a removed entry in different id orders
            dead = np.array(sorted(dead), np.uint32)
            b.remove(dead)
            a.remove(pi[dead].astype(np.uint32))
            _assert_equal_through(gpu, a, b, pi, Q)
            m = a.compact().astype(np.int64)
            kept = m != NONE
            pi = np.where(pi == NONE, NONE, m[np.minimum(pi, m.size - 1)])
            Xa = Xa[kept]
            _assert_equal_through(gpu, a, b, pi, Q)

        lo = n0
        for _ in range(rounds):
            insert_at(lo)
            lo += c
            remove_and_compact()
        insert_at(lo)
        lo += c
        # update (live and removed ids), then compact: invariants only
        na = a.info()[0]
        gone = rng.choice(na, na // 10, replace=False).astype(np.uint32)
        a.remove(gone)
        upd = np.unique(np.concatenate([gone[:20], rng.choice(na, 60, replace=False)])).astype(np.uint32)
        W = X[lo:lo + upd.size]
        a.update(upd, W)
        Xa[upd] = W
        _assert_no_removed_ids(a)
        live = a.export_live()
        m = a.compact().astype(np.int64)
        assert np.array_equal(m != NONE, live)
        assert np.array_equal(m[live], np.arange(live.sum()))
        Xa = Xa[live]
        assert a.info()[0] == Xa.shape[0] and a.export_live().all()
        _assert_no_removed_ids(a)
        _compare_oracle(a, Xa, Q, 10, 64, metric)
    finally:
        gpu.set_option("hnsw.shift_chunk_rows", 0)
