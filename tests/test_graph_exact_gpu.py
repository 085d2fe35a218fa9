"""The SSSP family judged by exact f64 references, in both state forms and across source chunks.

ShortestPathDijkstra (`Graph.sssp`), KShortestPathYen's constrained searches (`Graph.sssp_paths`), ClosenessCentrality
and BetweennessCentrality all run through one driver: `sssp_chunks` -> `launch_sssp` in graph.cu.  Two of its paths
are otherwise reached only by large graphs: the state in HBM (`sssp_kernel<FORB, false>`, taken above ~23 k nodes) and
more than one chunk of sources (an 8 GB budget per chunk).  The options `sssp.smem=0` and `sssp.max_chunk_sources=k`
force both on small graphs, where exact references are cheap; the tests marked natural-size take them with the
options at their defaults.

References (numpy / scipy only):
- distances: scipy's f64 Dijkstra on the lightest weight per (u, v), self-loops dropped.  Weights are k/8 with
  1 <= k < 64, so every path sum is exact in f32 and the device must equal it bit for bit;
- predecessor trees: every reached t != s has (pred[t], t) as an edge with fl32(d[pred] + w) == d[t], and pointer
  jumping brings every reached node to s;
- closeness: nc^2 / sum(d) / (n - 1) in f64 (nc counts the source); the device rounds nc^2, the total and two
  quotients to f32, so it may differ by 3e-7 relative;
- betweenness: Brandes in f64 over the tie DAG {(u, v) : fl32(d[u] + w) == d[v]}, counted per edge (parallel tied
  edges count twice), edges into the source skipped, processed level by level in order of distance.  The device
  rounds an f64 sum to f32 once: 2^-23 relative, and exactly 0 where the truth is 0.
"""
import contextlib
import math
import os

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

from oracle import oracle as O
from tests.util import rmat_edges

NONE = 0xFFFFFFFF
UNVERIFIED = [pytest.mark.gpu_unverified,
              pytest.mark.skipif(os.environ.get("COZO_RUN_UNVERIFIED") != "1",
                                 reason="not yet run on a GPU; opt in with COZO_RUN_UNVERIFIED=1")]
NATURAL = pytest.mark.skipif(bool(os.environ.get("COZO_EMU_LIB")), reason="natural-size graphs: too large for the emulated library")
# the flag-scan form is the default; the compacted-frontier and wide forms have not run on a GPU yet
FORMS = [pytest.param({}, id="flags", marks=pytest.mark.gpu),
         pytest.param({"sssp.frontier": 1}, id="frontier", marks=UNVERIFIED),
         pytest.param({"sssp.wide": 1}, id="wide", marks=UNVERIFIED)]
DEFAULTS = {"sssp.smem": 1, "sssp.max_chunk_sources": 0, "sssp.frontier": 0, "sssp.wide": 0}
# shared-memory / HBM state x one chunk, one source per chunk, and chunks that do not divide n
COMBOS = [{"sssp.smem": smem, "sssp.max_chunk_sources": k} for smem in (1, 0) for k in (0, 1, 7, 97)]


@contextlib.contextmanager
def options(capi, opts):
    try:
        for k, v in opts.items():
            capi.set_option(k, v)
        yield
    finally:
        for k, v in DEFAULTS.items():
            capi.set_option(k, v)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def to_f32(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float32)


# ---- references --------------------------------------------------------------------------------------------------
def lightest(n, src, dst, w):
    """(u, v, w) with the lightest weight per pair and no self-loops (csr_matrix would sum duplicates)"""
    w = np.ones(src.size, np.float32) if w is None else np.asarray(w, np.float32)
    k = src != dst
    key = src[k].astype(np.int64) * n + dst[k]
    ww = w[k]
    order = np.lexsort((ww, key))
    key, ww = key[order], ww[order]
    first = np.ones(key.size, bool)
    first[1:] = key[1:] != key[:-1]
    return key[first] // n, key[first] % n, ww[first]


def _dijkstra(n, u, v, ww, sources):
    assert np.all(ww > 0), "explicit zeros: scipy cannot judge this graph"
    a = csr_matrix((ww.astype(np.float64), (u, v)), shape=(n, n))
    return dijkstra(a, directed=True, indices=np.asarray(sources, np.int64)).reshape(len(sources), n)


def exact_dist(n, src, dst, w, sources):
    """f64 Dijkstra from `sources` -> (len(sources), n) f64"""
    return _dijkstra(n, *lightest(n, src, dst, w), sources)


def check_tree(n, src, dst, w, sources, dist, pred):
    """vectorised predecessor-tree check: tied edges, NONE at sources and unreached nodes, paths reach the source"""
    sources = np.asarray(sources, np.int64)
    w = np.ones(src.size, np.float32) if w is None else np.asarray(w, np.float32)
    rows = np.arange(sources.size)
    reached = np.isfinite(dist)
    assert np.all(reached[rows, sources])
    assert np.all(pred[rows, sources] == NONE) and np.all(pred[~reached] == NONE)
    inner = reached.copy()
    inner[rows, sources] = False
    r, t = np.nonzero(inner)
    p = pred[r, t].astype(np.int64)
    assert np.all(p < n)
    # (row, u, v) of every edge that ties, for each row: the set the pair (pred[t], t) must fall in
    ok = []
    for r0 in range(0, sources.size, 16):
        d = dist[r0:r0 + 16]
        with np.errstate(over="ignore"):
            tie = np.isfinite(d[:, src]) & (d[:, src] + w == d[:, dst])
        rr, e = np.nonzero(tie)
        ok.append(((rr + r0) * n + src[e].astype(np.int64)) * n + dst[e])
    ok = np.unique(np.concatenate(ok))
    want = (r.astype(np.int64) * n + p) * n + t
    hit = np.searchsorted(ok, want)
    hit = np.minimum(hit, ok.size - 1)
    assert np.all(ok[hit] == want), "a predecessor is not a tied edge"
    # pointer jumping: every reached node arrives at its source within ceil(log2 n) + 1 doublings
    jump = np.where(reached, pred.astype(np.int64), np.arange(n)[None, :])
    jump[rows, sources] = sources
    for _ in range(math.ceil(math.log2(max(n, 2))) + 1):
        jump = np.take_along_axis(jump, jump, axis=1)
    assert np.all(jump[reached] == np.broadcast_to(sources[:, None], jump.shape)[reached]), "predecessors form a cycle"


def closeness_truth(d64):
    """(n, n) all-pairs distances -> f64 closeness.  A distance past FLT_MAX is unreachable in f32, and a total past
    it is inf in f32 (closeness 0)."""
    n = d64.shape[0]
    reached = np.isfinite(to_f32(d64))
    nc = reached.sum(1).astype(np.float64)
    tot = np.where(reached, d64, 0.0).sum(1)
    tot[np.isinf(to_f32(tot))] = np.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        return nc * nc / tot / (n - 1)


def check_closeness(gc, truth):
    t32 = to_f32(truth)
    assert np.array_equal(np.isnan(gc), np.isnan(t32)) and np.array_equal(np.isinf(gc), np.isinf(t32))
    assert np.array_equal(gc == 0, truth == 0)
    fin = np.isfinite(t32) & (truth != 0)
    rel = np.abs(gc[fin].astype(np.float64) - truth[fin]) / truth[fin]
    assert rel.max(initial=0.0) <= 3e-7, rel.max()


def _levels(d):
    """rank of each distance among its row's distinct values"""
    order = np.argsort(d, axis=1, kind="stable")
    ds = np.take_along_axis(d, order, axis=1)
    step = np.zeros(d.shape, np.int64)
    step[:, 1:] = ds[:, 1:] != ds[:, :-1]
    lvl = np.empty(d.shape, np.int64)
    np.put_along_axis(lvl, order, np.cumsum(step, axis=1), axis=1)
    return lvl


def betweenness_truth(n, src, dst, w, d32, block=128):
    """Brandes in f64 over the tie DAG, per edge, level-synchronous by distance; d32 = (n, n) f32 distances"""
    w = np.ones(src.size, np.float32) if w is None else np.asarray(w, np.float32)
    s64, t64 = src.astype(np.int64), dst.astype(np.int64)
    bc = np.zeros(n)
    for b0 in range(0, n, block):
        d = d32[b0:b0 + block]
        b = d.shape[0]
        srcs = np.arange(b0, b0 + b)
        du, dv = d[:, src], d[:, dst]
        tie = np.isfinite(du) & np.isfinite(dv) & (du + w == dv) & (t64[None, :] != srcs[:, None])
        r, e = np.nonzero(tie)
        lvl = _levels(d)
        lu, lv = lvl[r, s64[e]], lvl[r, t64[e]]
        assert np.all(lv > lu), "a tied edge that does not increase the distance"
        fu, fv = r * n + s64[e], r * n + t64[e]
        sigma = np.zeros(b * n)
        sigma[np.arange(b) * n + srcs] = 1.0
        order = np.argsort(lv, kind="stable")
        cuts = np.searchsorted(lv[order], np.arange(lv.max(initial=0) + 2))
        for k in range(1, cuts.size - 1):          # nodes at level k: every predecessor sits at a lower level
            sl = order[cuts[k]:cuts[k + 1]]
            np.add.at(sigma, fv[sl], sigma[fu[sl]])
        assert sigma.max() < 2.0 ** 53          # path counts exact in f64, so any summation order gives the same bits
        delta = np.zeros(b * n)
        order = np.argsort(lu, kind="stable")
        cuts = np.searchsorted(lu[order], np.arange(lu.max(initial=0) + 2))
        for k in range(cuts.size - 2, -1, -1):     # nodes at level k: every successor's dependency is final
            sl = order[cuts[k]:cuts[k + 1]]
            np.add.at(delta, fu[sl], sigma[fu[sl]] / sigma[fv[sl]] * (1.0 + delta[fv[sl]]))
        delta = delta.reshape(b, n)
        delta[np.arange(b), srcs] = 0.0
        bc += delta.sum(0)
    return bc


def check_betweenness(gb, truth):
    z = truth == 0
    assert np.all(gb[z] == 0), np.nonzero(gb[z])
    rel = np.abs(gb[~z].astype(np.float64) - truth[~z]) / truth[~z]
    assert rel.max(initial=0.0) <= 2.0 ** -23, rel.max()


def check_paths(n, src, dst, w, sources, goals, fn, fe, res):
    """costs == scipy on the graph without the forbidden nodes / edges; paths walk allowed edges and sum to the cost"""
    lu, lv, lw = lightest(n, src, dst, w)                  # forbidding a pair forbids all its parallel edges
    key = lu * n + lv
    for i, (s, t) in enumerate(zip(sources.tolist(), goals.tolist())):
        bad = np.array([a * n + b for a, b in fe[i]], np.int64)
        keep = ~np.isin(lv, fn[i]) & ~np.isin(key, bad)
        exp = to_f32(_dijkstra(n, lu[keep], lv[keep], lw[keep], [s])[0, t])
        cost, path = res[i]
        assert bits(cost) == bits(exp), (i, cost, exp)
        if np.isinf(exp):
            assert path == []
            continue
        assert path[0] == s and path[-1] == t
        hop = np.array(path[:-1], np.int64) * n + np.array(path[1:], np.int64)
        at = np.minimum(np.searchsorted(key, hop), key.size - 1)
        assert np.all(key[at] == hop) and not np.isin(hop, bad).any() and not np.isin(path[1:], fn[i]).any(), i
        acc = np.float32(0)
        for x in lw[at]:                                   # f32 sum along the path over the lightest parallel edge
            acc = np.float32(acc + x)
        assert acc == np.float32(cost), (i, acc, cost)


# ---- graphs ------------------------------------------------------------------------------------------------------
def dyadic(rng, m):
    return (rng.integers(1, 64, m) / 8.0).astype(np.float32)


def random_dyadic():
    rng = np.random.default_rng(0x55D1)
    n, m = 1000, 6000
    src = rng.integers(0, n - 24, m).astype(np.uint32)            # the last 24 ids have no edges
    dst = rng.integers(0, n - 24, m).astype(np.uint32)
    return n, src, dst, dyadic(rng, m)


def rmat_dyadic():
    n, src, dst = rmat_edges(10, 8, 0x55D2)                       # duplicate edges and self-loops kept
    return n + 16, src, dst, dyadic(np.random.default_rng(0x55D2), src.size)


def rmat_unweighted():
    n, src, dst = rmat_edges(10, 8, 0x55D3)                       # every weight 1.0: many tied paths
    return n + 16, src, dst, None


SMALL = {"random_dyadic": random_dyadic, "rmat_dyadic": rmat_dyadic, "rmat_unweighted": rmat_unweighted}


def sources_for(n, src, dst, count, seed):
    """0, n - 1, a node with no edges at all, random others, and 0 again"""
    deg = np.bincount(src, minlength=n) + np.bincount(dst, minlength=n)
    iso = int(np.nonzero(deg == 0)[0][0])
    rng = np.random.default_rng(seed)
    s = np.concatenate([[0, n - 1, iso], rng.integers(0, n, count - 4), [0]])
    return s.astype(np.uint32)


# ---- the references themselves, on the CPU ------------------------------------------------------------------------
def test_references_agree_with_the_oracle():
    """the f64 judges against the oracle (a restatement of the reference): equal distances, closeness and betweenness
    within the oracle's own f32 drift"""
    rng = np.random.default_rng(0x55D0)
    n, m = 300, 1800
    src, dst, w = rng.integers(0, n, m).astype(np.uint32), rng.integers(0, n, m).astype(np.uint32), dyadic(rng, m)
    o = O.OracleGraph(n, src, dst, w)
    d64 = exact_dist(n, src, dst, w, np.arange(n))
    od, _ = o.sssp(np.arange(n, dtype=np.uint32), n_threads=4)
    assert np.array_equal(to_f32(d64), od)
    oc = o.closeness(n_threads=4)
    truth = closeness_truth(d64)
    fin = np.isfinite(truth)
    assert np.array_equal(np.isfinite(oc), fin) and np.allclose(oc[fin], truth[fin], rtol=1e-5)
    bt = betweenness_truth(n, src, dst, w, od)
    assert np.allclose(o.betweenness(n_threads=4), bt, rtol=1e-4, atol=1e-4) and bt.max() > 10
    # parallel tied edges count once each, as the reference's back pointers do: 0 -> 1 twice and 0 -> 2 lead to 3, so
    # two of the three shortest paths 0 -> 3 pass 1
    s, d = np.array([0, 0, 0, 1, 2], np.uint32), np.array([1, 1, 2, 3, 3], np.uint32)
    bt = betweenness_truth(4, s, d, None, to_f32(exact_dist(4, s, d, None, range(4))))
    ob = O.OracleGraph(4, s, d, np.ones(5, np.float32)).betweenness()
    assert np.allclose(bt, [0, 2 / 3, 1 / 3, 0], rtol=1e-15, atol=0) and np.allclose(ob, bt, rtol=1e-6, atol=0)
    # the tree check rejects a predecessor over a longer edge and one over no edge at all
    pred = np.array([[NONE, 0, 0, 1]], np.uint32)
    dist = np.array([[0, 1, 1, 2]], np.float32)
    check_tree(4, s, d, None, [0], dist, pred)
    for bad in ([NONE, 0, 0, 0], [NONE, 0, 3, 2]):
        with pytest.raises(AssertionError):
            check_tree(4, s, d, None, [0], dist, np.array([bad], np.uint32))


# ---- small graphs: every state form and chunking, bitwise identical ----------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", list(SMALL))
def test_sssp_family_exact_in_every_state_form_and_chunking(gpu, kind, form):
    n, src, dst, w = SMALL[kind]()
    g = gpu.Graph(n, src, dst, w)
    d64 = exact_dist(n, src, dst, w, np.arange(n))
    d32 = to_f32(d64)
    sources = sources_for(n, src, dst, 150, 1)
    c_truth = closeness_truth(d64)
    b_truth = betweenness_truth(n, src, dst, w, d32)
    assert (c_truth == np.inf).sum() >= 16 and b_truth.max() > 100
    first = None
    for combo in COMBOS:
        with options(gpu, {**form, **combo}):
            gd, gp, _ = g.sssp(sources)
            gc, _ = g.closeness()
            gb, _ = g.betweenness()
        assert np.array_equal(bits(gd), bits(d32[sources])), combo
        check_tree(n, src, dst, w, sources, gd, gp)
        check_closeness(gc, c_truth)
        check_betweenness(gb, b_truth)
        if first is None:
            first = (gd, gc, gb)
        for a, b in zip(first, (gd, gc, gb)):
            assert np.array_equal(bits(a), bits(b)), combo


@pytest.mark.parametrize("form", FORMS)
def test_sssp_paths_with_forbidden_sets_in_hbm_state(gpu, form):
    """constrained searches (KShortestPathYen's spur searches) with the state in HBM: sssp_kernel<true, false>"""
    n, src, dst, w = rmat_dyadic()
    rng = np.random.default_rng(0x55D4)
    k = 64
    sources = rng.integers(0, n - 16, k).astype(np.uint32)
    goals = rng.integers(0, n - 16, k).astype(np.uint32)
    goals[:2] = sources[:2]                                    # source == goal
    goals[2] = n - 1                                           # an isolated goal
    # forbidden nodes (never the source, sometimes the goal) and forbidden edges drawn from the graph
    fn = [[int(x) for x in rng.integers(0, n, rng.integers(0, 6)) if x != sources[i]] for i in range(k)]
    if goals[3] != sources[3]:
        fn[3].append(int(goals[3]))
    fe = [[(int(src[j]), int(dst[j])) for j in rng.integers(0, src.size, rng.integers(0, 8))] for i in range(k)]
    g = gpu.Graph(n, src, dst, w)
    for smem in (0, 1):
        with options(gpu, {**form, "sssp.smem": smem}):
            res, _ = g.sssp_paths(sources, goals, fn, fe, max_len=4)
        check_paths(n, src, dst, w, sources, goals, fn, fe, res)
    assert sum(np.isinf(c) for c, _ in res) >= 2 and max(len(p) for _, p in res) > 4


# ---- edge values -------------------------------------------------------------------------------------------------
def _run_combos(gpu, g, sources):
    """sssp / closeness / betweenness in every combination, checked bitwise identical across them"""
    first = None
    for combo in COMBOS:
        with options(gpu, combo):
            out = (*g.sssp(sources)[:2], g.closeness()[0], g.betweenness()[0])
        if first is None:
            first = out
        for a, b in zip(first[:1] + first[2:], out[:1] + out[2:]):
            assert np.array_equal(bits(a), bits(b)), combo
        yield out


@pytest.mark.gpu
def test_subnormal_weights(gpu):
    """weights k * 2^-149: every sum is exact (no flush to zero), the tie structure is that of k/8"""
    n, src, dst, w8 = random_dyadic()
    n, keep = 400, (src < 400) & (dst < 400)
    src, dst = src[keep], dst[keep]
    k = (w8[keep] * 8).astype(np.uint32)
    w = k.view(np.float32)
    assert w.max() < 1e-43 and w.min() > 0
    g = gpu.Graph(n, src, dst, w)
    d64 = exact_dist(n, src, dst, w, np.arange(n))
    d32 = to_f32(d64)
    c_truth = closeness_truth(d64)
    b_truth = betweenness_truth(n, src, dst, w, d32)
    sources = np.arange(n, dtype=np.uint32)
    for gd, gp, gc, gb in _run_combos(gpu, g, sources):
        assert np.array_equal(bits(gd), bits(d32))
        check_tree(n, src, dst, w, sources, gd, gp)
        check_closeness(gc, c_truth)                     # nc^2 / (a subnormal total) overflows f32: inf, as in the truth
        check_betweenness(gb, b_truth)
    assert np.isinf(gc).all() and b_truth.max() > 10


@pytest.mark.gpu
def test_weights_near_flt_max_overflow_to_unreachable(gpu):
    """a path whose f32 sum overflows does not reach its target: distance inf, not counted by closeness"""
    big = np.float32(2.0 ** 126)
    src = np.array([0, 1, 2, 3, 4, 0, 5, 6, 6], np.uint32)
    dst = np.array([1, 2, 3, 4, 0, 5, 6, 7, 7], np.uint32)
    w = np.array([big, 1.5 * big, 2 * big, big, 1, 1.25 * big, 1.5 * big, 3.0, 2 * big], np.float32)
    n = 9                                                     # node 8: no edges
    g = gpu.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, w)
    d64 = exact_dist(n, src, dst, w, np.arange(n))
    od, _ = o.sssp(np.arange(n, dtype=np.uint32))
    assert np.array_equal(bits(to_f32(d64)), bits(od))
    assert np.isinf(od[0, 3]) and od[0, 2] == 2.5 * big and od[0, 7] == 2.75 * big      # + 3.0 is absorbed
    c_truth = closeness_truth(d64)
    oc = o.closeness()
    assert (c_truth == 0).any() and np.isinf(c_truth).any()
    for gd, gp, gc, _ in _run_combos(gpu, g, np.arange(n, dtype=np.uint32)):
        assert np.array_equal(bits(gd), bits(od))
        check_tree(n, src, dst, w, np.arange(n), gd, gp)
        # closeness is subnormal or 0 at this scale: judged bitwise by the oracle, whose f32 totals of a few multiples
        # of 2^124 are exact too, and against the truth where it is inf (no other node reached) or 0 (total past FLT_MAX)
        assert np.array_equal(bits(gc), bits(oc))
        assert np.array_equal(np.isinf(gc), np.isinf(c_truth)) and np.array_equal(gc == 0, c_truth == 0)


@pytest.mark.gpu
def test_negative_zero_weight(gpu):
    """-0.0 passes the weight check; 0 + -0.0 = +0.0, so no distance is ever -0.0 (judged bitwise by the oracle)"""
    src = np.array([0, 1, 1, 2, 3, 0, 4], np.uint32)
    dst = np.array([1, 2, 3, 4, 4, 3, 5], np.uint32)
    w = np.array([-0.0, 0.5, 0.5, -0.0, 0.0, 0.5, 1.0], np.float32)
    n = 7
    g = gpu.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, w)
    od, _ = o.sssp(np.arange(n, dtype=np.uint32))
    oc, ob = o.closeness(), o.betweenness()
    assert not np.any(bits(od) == 0x80000000)
    for gd, gp, gc, gb in _run_combos(gpu, g, np.arange(n, dtype=np.uint32)):
        assert np.array_equal(bits(gd), bits(od))
        check_tree(n, src, dst, w, np.arange(n), gd, gp)
        assert np.array_equal(np.isinf(gc), np.isinf(oc)) and np.allclose(gc[np.isfinite(oc)], oc[np.isfinite(oc)], rtol=1e-6)
        assert np.allclose(gb, ob, rtol=1e-6) and ob.max() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 5])
def test_graphs_without_edges(gpu, n):
    e = np.zeros(0, np.uint32)
    g = gpu.Graph(n, e, e, np.zeros(0, np.float32))
    sources = np.array([n - 1, 0, n - 1], np.uint32)
    for gd, gp, gc, gb in _run_combos(gpu, g, sources):
        exp = np.full((3, n), np.inf, np.float32)
        exp[np.arange(3), sources] = 0
        assert np.array_equal(bits(gd), bits(exp)) and np.all(gp == NONE)
        check_closeness(gc, closeness_truth(exact_dist(n, e, e, None, np.arange(n))))
        assert np.isinf(gc).all() and np.all(gb == 0)


@pytest.mark.gpu
def test_two_nodes(gpu):
    g = gpu.Graph(2, [0], [1], [0.375])
    for gd, gp, gc, gb in _run_combos(gpu, g, np.array([1, 0], np.uint32)):
        assert gd.tolist() == [[np.inf, 0.0], [0.0, 0.375]] and gp.tolist() == [[NONE, NONE], [NONE, 0]]
        check_closeness(gc, np.array([4 / 0.375, np.inf]))
        assert gb.tolist() == [0.0, 0.0]


# ---- natural size on the H100: the real shared-memory threshold and memory budget, options at their defaults -----
def rmat16():
    n, src, dst = rmat_edges(16, 16, 0x55D5)
    return n, src, dst, dyadic(np.random.default_rng(0x55D5), src.size)


@pytest.mark.gpu
@NATURAL
def test_sssp_rmat16_state_in_hbm(gpu):
    """65 536 nodes: 10 bytes per node are past shared memory, so the state lives in HBM without any option"""
    n, src, dst, w = rmat16()
    assert 10 * n + 1024 > 227 * 1024
    g = gpu.Graph(n, src, dst, w)
    sources = sources_for(n, src, dst, 64, 2)
    gd, gp, _ = g.sssp(sources)
    assert np.array_equal(bits(gd), bits(to_f32(exact_dist(n, src, dst, w, sources))))
    check_tree(n, src, dst, w, sources, gd, gp)
    assert np.isfinite(gd).sum(1).max() > n // 4


@pytest.mark.gpu
@NATURAL
def test_sssp_paths_rmat16_state_in_hbm(gpu):
    n, src, dst, w = rmat16()
    rng = np.random.default_rng(0x55D6)
    k = 48
    out_deg = np.bincount(src, minlength=n)
    sources = rng.choice(np.nonzero(out_deg > 0)[0], k).astype(np.uint32)
    goals = rng.choice(np.nonzero(out_deg > 0)[0], k).astype(np.uint32)
    fn = [[int(x) for x in rng.integers(0, n, rng.integers(0, 6)) if x != sources[i]] for i in range(k)]
    fe = [[(int(src[j]), int(dst[j])) for j in rng.integers(0, src.size, rng.integers(0, 8))] for i in range(k)]
    for i in range(0, k, 4):                   # some searches lose the first hop of an unconstrained shortest path
        fe[i].append((int(sources[i]), int(dst[src == sources[i]][0])))
    res, _ = gpu.Graph(n, src, dst, w).sssp_paths(sources, goals, fn, fe, max_len=8)
    check_paths(n, src, dst, w, sources, goals, fn, fe, res)
    assert sum(np.isfinite(c) for c, _ in res) > k // 2


@pytest.mark.gpu
@NATURAL
def test_closeness_grid_200x200_several_chunks(gpu):
    """a mirrored 200 x 200 grid, horizontal weight a, vertical b: sum of d from (i, j) is
    a R sum_l |j - l| + b C sum_k |i - k|.  40 000 nodes keep the state in HBM, and at 17 bytes per node and source
    the 8 GB chunk budget needs several chunks"""
    R = C = 200
    a, b = 0.375, 1.25
    idx = np.arange(R * C).reshape(R, C)
    h_s, h_d = idx[:, :-1].ravel(), idx[:, 1:].ravel()
    v_s, v_d = idx[:-1, :].ravel(), idx[1:, :].ravel()
    src = np.concatenate([h_s, h_d, v_s, v_d]).astype(np.uint32)
    dst = np.concatenate([h_d, h_s, v_d, v_s]).astype(np.uint32)
    w = np.concatenate([np.full(2 * h_s.size, a), np.full(2 * v_s.size, b)]).astype(np.float32)
    n = R * C
    assert 17 * n * n > 8 << 30
    gc, _ = gpu.Graph(n, src, dst, w).closeness()
    col = np.abs(np.arange(C)[:, None] - np.arange(C)[None, :]).sum(1).astype(np.float64)
    row = np.abs(np.arange(R)[:, None] - np.arange(R)[None, :]).sum(1).astype(np.float64)
    tot = a * R * col[None, :] + b * C * row[:, None]
    check_closeness(gc, (float(n) * n / tot / (n - 1)).ravel())


@pytest.mark.gpu
@NATURAL
def test_betweenness_star_30000_several_chunks(gpu):
    """a mirrored star: every ordered pair of leaves has one shortest path, through the hub"""
    n = 30000
    leaves = np.arange(1, n, dtype=np.uint32)
    src = np.concatenate([np.zeros(n - 1, np.uint32), leaves])
    dst = np.concatenate([leaves, np.zeros(n - 1, np.uint32)])
    w = np.full(src.size, 0.5, np.float32)
    assert (8 + 9 + 32) * n * n > 8 << 30
    gb, _ = gpu.Graph(n, src, dst, w).betweenness()
    truth = np.zeros(n)
    truth[0] = (n - 1) * (n - 2)
    check_betweenness(gb, truth)
