"""ShortestPathDijkstra with a termination relation: `Graph.sssp_goals` (cozo_gpu_sssp_goals), where each search stops
once its goals are settled and only the goal answers leave the device.

Judged against the exact oracle (oracle/cozo_oracle.cpp: the reference's dijkstra with its goal stop) and against the
full run of the same library (`Graph.sssp`), in both state forms and across source chunks (`sssp.smem`,
`sssp.max_chunk_sources`, as in test_graph_exact_gpu.py).  Weights are k/8 with 1 <= k < 64, so every path sum is
exact in f32 and costs must agree bit for bit.
- paths: start..goal, every hop a tight edge of the full run's distances; equal to the oracle's back-pointer path
  wherever the oracle has a single shortest path;
- keep_ties: the tied edges equal, as a multiset, the closure from the goals over tight edges of the full distances
  (edges into the source not followed), and the paths walked over them equal, as a set, the paths through the
  oracle's keep_ties predecessor lists.
"""
import contextlib
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import rmat_edges

pytestmark = pytest.mark.gpu
NATURAL = pytest.mark.skipif(bool(os.environ.get("COZO_EMU_LIB")), reason="natural-size graphs: too large for the emulated library")
DEFAULTS = {"sssp.smem": 1, "sssp.max_chunk_sources": 0, "sssp.frontier": 0, "sssp.wide": 0}
COMBOS = [{"sssp.smem": smem, "sssp.max_chunk_sources": k} for smem in (1, 0) for k in (0, 1, 7, 97)]
CIDS = [f"smem{c['sssp.smem']}-chunk{c['sssp.max_chunk_sources']}" for c in COMBOS]


@contextlib.contextmanager
def options(capi, opts):
    try:
        for k, v in opts.items():
            capi.set_option(k, v)
        yield
    finally:
        for k, v in DEFAULTS.items():
            capi.set_option(k, v)


@pytest.fixture(scope="module")
def capi(gpu):
    return gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def random_graph(n, m, seed, kmax=64):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m).astype(np.uint32)
    dst = rng.integers(0, n, m).astype(np.uint32)
    w = (rng.integers(1, kmax, m) / 8.0).astype(np.float32)
    return src, dst, w


def grid(side):
    """unit-weight grid, both directions: many tied shortest paths"""
    idx = np.arange(side * side).reshape(side, side)
    a = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    b = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    return np.concatenate([a, b]).astype(np.uint32), np.concatenate([b, a]).astype(np.uint32)


def walk(preds, s, t, cap=20000):
    """every path s..t over a {v: [p, ...]} predecessor map, edges into s not followed (the reference's collect)"""
    out, chain = [], [t]

    def rec():
        for p in preds.get(chain[-1], ()):
            chain.append(p)
            if p == s:
                out.append(tuple(reversed(chain)))
            else:
                rec()
            chain.pop()
            assert len(out) <= cap, "too many tied paths for a test"
    rec()
    return out


def oracle_preds(bp, bi):
    return {v: bi[bp[v]:bp[v + 1]].tolist() for v in range(bp.size - 1) if bp[v + 1] > bp[v]}


def tie_truth(src, dst, w, s, d, goals):
    """the tied-edge multiset of one source from its full f32 distances d, sorted (v, p) rows"""
    w = np.ones(src.size, np.float32) if w is None else w
    with np.errstate(over="ignore", invalid="ignore"):
        tight = np.isfinite(d[src]) & (d[src] + w == d[dst]) & (dst != s)
    mark = np.zeros(d.size, bool)
    g = np.asarray(goals, np.int64)
    mark[g[(g != s) & np.isfinite(d[g])]] = True
    while True:
        e = tight & mark[dst]
        new = mark.copy()
        new[src[e]] = True
        if np.array_equal(new, mark):
            break
        mark = new
    rows = np.stack([dst[e], src[e]], 1).astype(np.uint32)
    return rows[np.lexsort((rows[:, 1], rows[:, 0]))]


def sort_rows(r):
    r = np.asarray(r, np.uint32).reshape(-1, 2)
    return r[np.lexsort((r[:, 1], r[:, 0]))]


def check_paths(src, dst, w, sources, goals, dist, cost, paths):
    """every path: start..goal, tight hops w.r.t. the full distances; [] exactly when unreachable"""
    w = np.ones(src.size, np.float32) if w is None else w
    n = dist.shape[1]
    key = src.astype(np.int64) * n + dst
    order = np.argsort(key, kind="stable")
    key, ws = key[order], w[order]
    for si, s in enumerate(sources):
        d = dist[si]
        for gi, t in enumerate(goals):
            p = paths[si][gi]
            if not np.isfinite(cost[si, gi]):
                assert p == []
                continue
            assert p[0] == s and p[-1] == t and len(set(p)) == len(p)
            for a, b in zip(p, p[1:]):
                lo, hi = np.searchsorted(key, [a * n + b, a * n + b + 1])
                assert np.any(d[a] + ws[lo:hi] == d[b]), (s, t, a, b)


def run_case(capi, n, src, dst, w, sources, goals, exact_paths=True):
    sources = np.asarray(sources, np.uint32)
    goals = np.asarray(goals, np.uint32)
    g = capi.Graph(n, src, dst, w)
    cost, paths, _ = g.sssp_goals(sources, goals)
    full, _, _ = g.sssp(sources, want_pred=False)
    o = O.OracleGraph(n, src, dst, np.ones(src.size, np.float32) if w is None else w)
    od, back = o.sssp(sources, goals)
    assert np.array_equal(bits(cost), bits(od[:, goals]))
    assert np.array_equal(bits(cost), bits(full[:, goals]))
    check_paths(src, dst, w, sources, goals, full, cost, paths)
    if exact_paths:  # where the oracle has one shortest path (keep_ties enumerates one), the device found it
        for si, s in enumerate(sources.tolist()):
            _, bp, bi = o.sssp_keep_ties(s, goals)
            preds = oracle_preds(bp, bi)
            for gi, t in enumerate(goals.tolist()):
                if t == s or not np.isfinite(cost[si, gi]):
                    continue
                ways = set(walk(preds, s, t))
                if len(ways) == 1:
                    assert tuple(paths[si][gi]) == next(iter(ways))
                    path, cur = [t], t
                    while cur != s:
                        cur = int(back[si, cur])
                        path.append(cur)
                    assert path[::-1] == paths[si][gi]
    return g, cost, paths


@pytest.mark.parametrize("opts", COMBOS, ids=CIDS)
def test_costs_and_paths(capi, opts):
    n = 300
    src, dst, w = random_graph(n, 1500, 11)
    rng = np.random.default_rng(3)
    goals = rng.choice(n, 12, replace=False)
    sources = np.unique(np.concatenate([rng.choice(n, 30, replace=False), goals[:3]]))
    with options(capi, opts):
        run_case(capi, n, src, dst, w, sources, goals)
        run_case(capi, n, src, dst, None, sources, goals)


def long_tail(tail, unreachable_goal):
    """goals one to three hops from node 0; a chain of `tail` nodes hangs off node 1 and keeps the frontier alive"""
    src, dst, w = [], [], []
    for v in range(1, 11):
        src.append(0), dst.append(v), w.append(1.0)
    for v in range(1, 10):
        src.append(v), dst.append(v + 1), w.append(0.125)
    for k in range(tail):
        src.append(1 if k == 0 else 10 + k), dst.append(11 + k), w.append(0.5)
    n = 11 + tail + (1 if unreachable_goal else 0)
    goals = [2, 5, 9] + ([n - 1] if unreachable_goal else [])
    return n, np.array(src, np.uint32), np.array(dst, np.uint32), np.array(w, np.float32), goals


@pytest.mark.parametrize("unreachable", [False, True], ids=["settled", "unreachable-goal"])
@pytest.mark.parametrize("opts", [COMBOS[0], COMBOS[4]], ids=[CIDS[0], CIDS[4]])
def test_early_stop_equals_full_run(capi, opts, unreachable):
    n, src, dst, w, goals = long_tail(3000, unreachable)
    with options(capi, opts):
        g, cost, paths = run_case(capi, n, src, dst, w, [0, 1, 3], goals)
        assert cost[0, 0] == 1.0 and cost[0, 1] == 1.0 and cost[0, 2] == 1.0
        assert np.isinf(cost[0, -1]) == unreachable and (paths[0][-1] == []) == unreachable
        _, ties, _ = g.sssp_goals([0, 1, 3], goals, keep_ties=True)
        full, _, _ = g.sssp([0, 1, 3], want_pred=False)
        for si, s in enumerate([0, 1, 3]):
            assert np.array_equal(sort_rows(ties[si]), tie_truth(src, dst, w, s, full[si], goals))


def check_ties(capi, n, src, dst, w, sources, goals):
    g = capi.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, np.ones(src.size, np.float32) if w is None else w)
    cost, ties, _ = g.sssp_goals(sources, goals, keep_ties=True)
    full, _, _ = g.sssp(sources, want_pred=False)
    assert np.array_equal(bits(cost), bits(full[:, goals]))
    for si, s in enumerate(sources):
        assert np.array_equal(sort_rows(ties[si]), tie_truth(src, dst, w, s, full[si], goals))
        preds = {}
        for v, p in ties[si].tolist():
            preds.setdefault(v, []).append(p)
        _, bp, bi = o.sssp_keep_ties(s, goals)
        opreds = oracle_preds(bp, bi)
        for gi, t in enumerate(goals):
            if t == s:
                continue
            assert set(walk(preds, s, t)) == set(walk(opreds, s, t)), (s, t)


@pytest.mark.parametrize("opts", [COMBOS[0], COMBOS[2], COMBOS[4], COMBOS[6]], ids=[CIDS[i] for i in (0, 2, 4, 6)])
def test_keep_ties(capi, opts):
    with options(capi, opts):
        side = 9
        src, dst = grid(side)
        n = side * side
        check_ties(capi, n, src, dst, None, [0, 4, 40, 80], [80, 44, 8, 72, 0, 40])
        src, dst, w = random_graph(200, 1200, 5, kmax=3)  # weights 1/8 and 2/8: many ties
        check_ties(capi, 200, src, dst, w, list(range(0, 200, 9)), [1, 17, 33, 99, 150, 151, 199])


def test_edge_cases(capi):
    src, dst, w = random_graph(50, 200, 1)
    g = capi.Graph(50, src, dst, w)
    cost, paths, _ = g.sssp_goals([7, 8], [7])                  # goal == source
    assert cost[0, 0] == 0.0 and paths[0][0] == [7]
    _, ties, _ = g.sssp_goals([7], [7], keep_ties=True)
    assert ties[0].shape == (0, 2)
    cost, paths, _ = g.sssp_goals([1, 2], [])                   # no goals
    assert cost.shape == (2, 0) and paths == [[], []]
    cost, ties, _ = g.sssp_goals([1, 2], [], keep_ties=True)
    assert [t.shape for t in ties] == [(0, 2), (0, 2)]
    for goals in ([3, 4, 3], [3, 50]):                          # duplicate, out of range
        with pytest.raises(capi.CozoGpuError) as e:
            g.sssp_goals([1], goals)
        assert e.value.code == capi.E_INVAL
    with pytest.raises(capi.CozoGpuError) as e:
        g.sssp_goals([50], [1])
    assert e.value.code == capi.E_INVAL
    poison = np.ones(1, np.int32)
    for kt in (False, True):
        with pytest.raises(capi.CozoGpuError) as e:
            g.sssp_goals([1], [2], keep_ties=kt, poison=poison)
        assert e.value.code == capi.E_KILLED
    # a capacity too small reports the total; the retry gives the same answer
    sources, goals = list(range(20)), [5, 9, 13, 40]
    cost, paths, _ = g.sssp_goals(sources, goals)
    cost1, paths1, _ = g.sssp_goals(sources, goals, cap=1)
    assert np.array_equal(bits(cost), bits(cost1)) and paths == paths1
    _, ties, _ = g.sssp_goals(sources, goals, keep_ties=True)
    _, ties1, _ = g.sssp_goals(sources, goals, keep_ties=True, cap=1)
    assert all(np.array_equal(sort_rows(a), sort_rows(b)) for a, b in zip(ties, ties1))
    assert sum(t.shape[0] for t in ties) > 1
    e = capi.Graph(0, [], [])                                    # empty graph
    cost, paths, _ = e.sssp_goals([], [])
    assert cost.shape == (0, 0) and paths == []


@NATURAL
def test_natural_size_rmat20(capi):
    """4 096 sources x 16 goals on weighted R-MAT-20: sssp_multi would need 34 GB of host buffers for this call"""
    n, src, dst = rmat_edges(20, 16, 7)
    rng = np.random.default_rng(9)
    w = (rng.integers(1, 64, src.size) / 8.0).astype(np.float32)
    g = capi.Graph(n, src, dst, w)
    sources = rng.choice(n, 4096, replace=False).astype(np.uint32)
    goals = rng.choice(n, 16, replace=False).astype(np.uint32)
    cost, paths, _ = g.sssp_goals(sources, goals)
    assert np.isfinite(cost).any()
    for b0 in range(0, sources.size, 64):
        full, _, _ = g.sssp(sources[b0:b0 + 64], want_pred=False)
        assert np.array_equal(bits(cost[b0:b0 + 64]), bits(full[:, goals]))
    for si in range(0, sources.size, 512):  # a sample of the paths against the distances of their source
        full, _, _ = g.sssp(sources[si:si + 1], want_pred=False)
        check_paths(src, dst, w, sources[si:si + 1].tolist(), goals.tolist(), full, cost[si:si + 1], paths[si:si + 1])


# ---- the rule through the host mirror (cozo_b200/host/fixed_rule.hpp) ---------------------------------------------
@pytest.fixture(scope="module")
def h(capi):
    from tests.hostmod import load
    m = load()
    m.init(0)
    return m


@pytest.mark.parametrize("undirected", [False, True], ids=["directed", "undirected"])
@pytest.mark.parametrize("keep_ties", [False, True], ids=["paths", "keep_ties"])
def test_rule_many_starts_and_goals(h, keep_ties, undirected):
    rng = np.random.default_rng(21)
    n, m = 120, 500
    names = [f"v{i:03d}" for i in range(n)]
    s, d = rng.integers(0, n, m), rng.integers(0, n, m)
    w = rng.integers(1, 4, m) / 8.0
    rows = sorted({(names[a], names[b], float(x)) for a, b, x in zip(s, d, w)})
    rows = [list(r) for r in rows]
    starts = [[names[i]] for i in range(0, n, 7)] + [["not-a-node"]]
    goal_names = [names[i] for i in range(3, n, 11)]
    out = h.Db().run_fixed_rule("ShortestPathDijkstra", [rows, starts, [[x] for x in goal_names]],
                                {"keep_ties": keep_ties, "undirected": undirected}, head_arity=4)
    # the oracle over the same dense ids (first appearance, mirrored edges right after their originals)
    ids, src, dst, ww = {}, [], [], []
    for a, b, x in rows:
        for k in (a, b):
            ids.setdefault(k, len(ids))
        src.append(ids[a]), dst.append(ids[b]), ww.append(x)
        if undirected:
            src.append(ids[b]), dst.append(ids[a]), ww.append(x)
    key = {v: k for k, v in ids.items()}
    o = O.OracleGraph(len(ids), np.array(src, np.uint32), np.array(dst, np.uint32), np.array(ww, np.float32))
    starts_id = sorted(ids[x[0]] for x in starts if x[0] in ids)
    goals_id = sorted(ids[x] for x in goal_names if x in ids)
    want = set()
    for s0 in starts_id:
        dist, bp, bi = o.sssp_keep_ties(s0, goals_id)
        preds = oracle_preds(bp, bi)
        for t in goals_id:
            c = float(dist[t])
            if not np.isfinite(c):
                want.add((key[s0], key[t], c, ()))
            elif keep_ties:
                want |= {(key[s0], key[t], c, tuple(key[u] for u in p)) for p in walk(preds, s0, t)}
            else:
                want.add((key[s0], key[t], c, None))
    got = {(a, b, c, tuple(p) if keep_ties or not p else None) for a, b, c, p in out}
    assert got == want
    if not keep_ties:
        wmin = {}
        for a, b, x in zip(src, dst, ww):
            wmin[(key[a], key[b])] = min(wmin.get((key[a], key[b]), 1e30), x)
        for a, b, c, p in out:
            if p:
                assert p[0] == a and p[-1] == b and sum(wmin[e] for e in zip(p, p[1:])) == c
