"""GPU parity tests for the FixedRule graph algorithms vs the CPU oracle."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.test_pagerank_exact_gpu import Truth, chain_lengths, options
from tests.util import rmat_edges

pytestmark = pytest.mark.gpu


def _random_graph(n, m, seed, weighted=True, dyadic=True):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m).astype(np.uint32)
    dst = rng.integers(0, n, m).astype(np.uint32)
    if not weighted:
        return src, dst, None
    w = (rng.integers(1, 64, m) / 8.0).astype(np.float32) if dyadic else (rng.random(m) * 10 + 0.01).astype(np.float32)
    return src, dst, w


def test_csr_staging_matches_oracle(gpu):
    src, dst, w = _random_graph(500, 6000, 1)
    g = gpu.Graph(500, src, dst, w)
    o = O.OracleGraph(500, src, dst, w)
    gop, goi, gow, gip, gii = g.export()
    oop, ooi, oow, oip, oii = o.export()
    assert np.array_equal(gop, oop) and np.array_equal(goi, ooi) and np.array_equal(gow, oow)
    assert np.array_equal(gip, oip) and np.array_equal(gii, oii)


def test_stage_rejects_bad_edges(gpu):
    with pytest.raises(gpu.CozoGpuError):
        gpu.Graph(3, [0, 5], [1, 2])
    with pytest.raises(gpu.CozoGpuError):
        gpu.Graph(3, [0, 1], [1, 2], [1.0, -2.0])       # negative weight (mod.rs:273-286)
    with pytest.raises(gpu.CozoGpuError):
        gpu.Graph(3, [0, 1], [1, 2], [1.0, np.inf])     # non finite (mod.rs:258-271)


@pytest.mark.parametrize("scale,iters,tol", [(10, 10, 1e-4), (14, 10, 1e-4), (14, 50, 0.0), (12, 3, 0.0), (17, 5, 0.0)])
def test_pagerank_rmat_parity(gpu, scale, iters, tol):
    n, src, dst = rmat_edges(scale, 16, 0x5EED0004)
    g = gpu.Graph(n, src, dst)
    o = O.OracleGraph(n, src, dst)
    gs, git, gerr, _ = g.pagerank(0.85, tol, iters)
    if scale == 17:
        gs2, _, _, _ = g.pagerank(0.85, tol, iters)         # work is drawn dynamically, sums are not: bit-identical reruns
        assert np.array_equal(gs, gs2)
    os_, oit, oerr = o.pagerank(0.85, tol, iters, variant="jacobi", n_threads=8)
    assert git == oit
    rel = np.abs(gs - os_) / os_
    assert rel.max() <= 1e-5, rel.max()                    # north-star tolerance: 1e-5 relative
    # scores, iteration count and err against the f64 iteration and its rounding bound
    Truth(n, src, dst, 0.85, tol, iters, chain_lengths(n, src, dst, {})).check(gs, git, gerr)


def test_pagerank_fixed_point_matches_gs_variant(gpu):
    """graph 0.3.1 may update contributions in place (Gauss-Seidel); both schedules share the
    fixed point, so converged GPU scores must match the GS oracle too (DESIGN.md)."""
    n, src, dst = rmat_edges(11, 16, 7)
    g = gpu.Graph(n, src, dst)
    o = O.OracleGraph(n, src, dst)
    gs, git, _, _ = g.pagerank(0.85, 1e-9, 500)
    os_, oit, _ = o.pagerank(0.85, 1e-9, 500, variant="gs")
    assert np.max(np.abs(gs - os_) / os_) <= 1e-5


def test_pagerank_edge_cases(gpu):
    g = gpu.Graph(0, np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    s, it, err, _ = g.pagerank()
    assert s.size == 0 and it == 0                          # pagerank.rs:43-45
    src = np.array([0, 1], np.uint32)
    dst = np.array([1, 2], np.uint32)                       # node 2 dangling
    g = gpu.Graph(3, src, dst)
    o = O.OracleGraph(3, src, dst)
    gs, git, _, _ = g.pagerank(0.85, 0.0, 3)
    os_, oit, _ = o.pagerank(0.85, 0.0, 3)
    assert git == oit == 3 and np.allclose(gs, os_, rtol=1e-6)
    # a hub row (in-degree > 2048) goes through the CTA-per-row kernel
    n = 5000
    src = np.concatenate([np.arange(1, n), np.zeros(n - 1)]).astype(np.uint32)
    dst = np.concatenate([np.zeros(n - 1), np.arange(1, n)]).astype(np.uint32)
    g = gpu.Graph(n, src, dst)
    o = O.OracleGraph(n, src, dst)
    gs, _, _, _ = g.pagerank(0.85, 0.0, 5)
    os_, _, _ = o.pagerank(0.85, 0.0, 5)
    # 4999 equal contributions summed one by one in f32 (what `.sum::<f32>()` does) drift from the
    # exact value by ~3e-5; the device's tree sum does not.  Judge both against f64 arithmetic.
    s64 = np.full(n, 1.0 / n)
    outdeg = np.bincount(src, minlength=n).astype(np.float64)
    for _ in range(5):
        c = s64 / outdeg
        nxt = np.full(n, 0.15 / n)
        np.add.at(nxt, dst, 0.85 * c[src])
        s64 = nxt
    assert np.max(np.abs(gs - s64) / s64) <= 4e-6
    assert np.max(np.abs(gs - os_) / os_) <= np.max(np.abs(os_ - s64) / s64) + 4e-6
    # poison set before the call -> killed
    flag = np.ones(1, np.int32)
    with pytest.raises(gpu.CozoGpuError) as e:
        g.pagerank(poison=flag)
    assert e.value.code == gpu.E_KILLED


PR_ENGINES = [
    {"pagerank.mode": 0},                                                      # round-1 gather pull
    {"pagerank.mode": 1},                                                      # propagation blocking, defaults
    {"pagerank.mode": 1, "pagerank.hub_slots": 64, "pagerank.group_slots": 256, "pagerank.window": 512, "pagerank.chunk": 1024},
    {"pagerank.mode": 1, "pagerank.hub_slots": 0, "pagerank.group_slots": 64, "pagerank.window": 64},   # no hub table
    {"pagerank.mode": 1, "pagerank.hub_slots": 1024, "pagerank.group_slots": 4096, "pagerank.window": 3001},  # odd window
]


@pytest.mark.parametrize("engine", range(len(PR_ENGINES)))
def test_pagerank_engines_and_blockings(gpu, engine):
    """every engine / blocking geometry computes the same iteration: <= 1e-5 of the oracle on R-MAT (all code paths of
    the blocking: several groups, many bins, rows that straddle windows, empty rows), bit-identical reruns"""
    opts = PR_ENGINES[engine]
    with options(gpu, opts):
        for scale, iters in ((13, 6), (9, 4)):
            n, src, dst = rmat_edges(scale, 16, 0x5EED0004 + scale)
            g = gpu.Graph(n, src, dst)
            os_, oit, oerr = O.OracleGraph(n, src, dst).pagerank(0.85, 0.0, iters, variant="jacobi", n_threads=8)
            gs, git, gerr, _ = g.pagerank(0.85, 0.0, iters)
            assert git == oit and np.max(np.abs(gs - os_) / os_) <= 1e-5
            Truth(n, src, dst, 0.85, 0.0, iters, chain_lengths(n, src, dst, opts)).check(gs, git, gerr)
            assert np.array_equal(gs, g.pagerank(0.85, 0.0, iters)[0])
        # a star: one row with 4999 in-edges (many windows long at the small geometries) + reverse edges
        n = 5000
        src = np.concatenate([np.arange(1, n), np.zeros(n - 1)]).astype(np.uint32)
        dst = np.concatenate([np.zeros(n - 1), np.arange(1, n)]).astype(np.uint32)
        gs = gpu.Graph(n, src, dst).pagerank(0.85, 0.0, 5)[0]
        s64 = np.full(n, 1.0 / n)
        outdeg = np.bincount(src, minlength=n).astype(np.float64)
        for _ in range(5):
            nxt = np.full(n, 0.15 / n)
            np.add.at(nxt, dst, 0.85 * (s64 / outdeg)[src])
            s64 = nxt
        assert np.max(np.abs(gs - s64) / s64) <= 4e-6
        # a path graph and a graph whose last ids have no edges at all
        src = np.arange(0, 300, dtype=np.uint32)
        dst = src + 1
        g = gpu.Graph(1000, src, dst)
        os_, _, _ = O.OracleGraph(1000, src, dst).pagerank(0.85, 0.0, 7)
        assert np.allclose(g.pagerank(0.85, 0.0, 7)[0], os_, rtol=1e-6)


def _check_tree(src, dst, w, sources, dist, pred, n):
    best = {}
    for s, t, ww in zip(src, dst, w):
        best.setdefault((int(s), int(t)), []).append(np.float32(ww))
    for si, s in enumerate(sources):
        assert pred[si, s] == 0xFFFFFFFF
        for t in range(n):
            if t == s or not np.isfinite(dist[si, t]):
                continue
            p = int(pred[si, t])
            assert (p, t) in best
            assert any(np.float32(dist[si, p] + ww) == dist[si, t] for ww in best[(p, t)])
            # walking up terminates at the source
            cur, hops = t, 0
            while cur != s:
                cur = int(pred[si, cur])
                hops += 1
                assert hops <= n


@pytest.mark.parametrize("dyadic", [True, False])
def test_sssp_parity(gpu, dyadic):
    n = 600
    src, dst, w = _random_graph(n, 4000, 3, dyadic=dyadic)
    g = gpu.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, w)
    sources = np.arange(0, n, 7, dtype=np.uint32)
    gd, gp, _ = g.sssp(sources)
    od, ob = o.sssp(sources, n_threads=8)
    assert np.array_equal(gd, od)           # f32 path sums are bit-identical (costs exact)
    _check_tree(src, dst, w, sources, gd, gp, n)


def test_sssp_zero_weights_and_unreachable(gpu):
    src = np.array([0, 1, 2, 1, 4], np.uint32)
    dst = np.array([1, 2, 1, 3, 0], np.uint32)
    w = np.array([0, 0, 0, 2, 1], np.float32)
    g = gpu.Graph(6, src, dst, w)
    o = O.OracleGraph(6, src, dst, w)
    gd, gp, _ = g.sssp([0, 4, 5])
    od, _ = o.sssp([0, 4, 5])
    assert np.array_equal(gd, od)
    assert np.isinf(gd[0, 4]) and np.isinf(gd[0, 5]) and gd[2, 5] == 0
    _check_tree(src, dst, w, [0, 4, 5], gd, gp, 6)
    # unweighted graph: weight defaults to 1.0 (mod.rs:254-255)
    g2 = gpu.Graph(6, src, dst)
    gd2, _, _ = g2.sssp([0])
    assert gd2[0].tolist()[:4] == [0, 1, 2, 2]


def test_closeness_parity(gpu):
    n = 400
    src, dst, w = _random_graph(n, 2400, 11, dyadic=False)
    g = gpu.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, w)
    gc, _ = g.closeness()
    oc = o.closeness(n_threads=8)
    fin = np.isfinite(oc)
    assert np.array_equal(np.isfinite(gc), fin)
    assert np.allclose(gc[fin], oc[fin], rtol=1e-5)


def test_betweenness_parity(gpu):
    n = 300
    src, dst, w = _random_graph(n, 1800, 13, dyadic=True)      # dyadic weights => many exact ties
    g = gpu.Graph(n, src, dst, w)
    o = O.OracleGraph(n, src, dst, w)
    gb, _ = g.betweenness()
    ob = o.betweenness(n_threads=8)
    assert np.allclose(gb, ob, rtol=1e-4, atol=1e-4)
    assert ob.max() > 10


# ---- the reference's air-routes fixture as input ----------------------------------------
def test_air_routes_all_rules(gpu):
    from tests.test_air_routes_cpu import load_routes
    n, src, dst, dist, id_of, _ = load_routes()
    g = gpu.Graph(n, src, dst, dist)
    o = O.OracleGraph(n, src, dst, dist)
    starts = np.array([id_of[c] for c in ("JFK", "LHR", "SYD", "AUS", "KUL")], np.uint32)
    gd, gp, _ = g.sssp(starts)
    od, _ = o.sssp(starts, n_threads=8)
    assert np.array_equal(gd, od)
    _check_tree(src, dst, dist, starts, gd, gp, n)
    gc, _ = g.closeness()
    oc = o.closeness(n_threads=16)
    fin = np.isfinite(oc)
    assert np.array_equal(np.isfinite(gc), fin) and np.allclose(gc[fin], oc[fin], rtol=1e-5)
    gb, _ = g.betweenness()
    ob = o.betweenness(n_threads=16)
    assert np.allclose(gb, ob, rtol=2e-4, atol=1e-3)
    g2 = gpu.Graph(n, src, dst)
    o2 = O.OracleGraph(n, src, dst)
    gs, git, _, _ = g2.pagerank(0.85, 1e-4, 10)
    os_, oit, _ = o2.pagerank(0.85, 1e-4, 10)
    assert git == oit and np.max(np.abs(gs - os_) / os_) <= 1e-5


def test_clustering_exact(gpu):
    """ClusteringCoefficients: integer counts and the f64 coefficient are bit-identical to the oracle,
    on a multigraph with duplicate edges and self loops (RMAT) and on the air-routes graph."""
    from tests.test_air_routes_cpu import load_routes
    n, src, dst = rmat_edges(12, 8, 99)
    ms = np.concatenate([src, dst])       # mirrored stream, as as_directed_graph(true) emits it (per edge: f->t, t->f)
    md = np.concatenate([dst, src])
    g = gpu.Graph(n, ms, md)
    o = O.OracleGraph(n, ms, md)
    gc, gt, gd, _ = g.clustering()
    oc, ot, od = o.clustering(n_threads=16)
    assert np.array_equal(gt, ot) and np.array_equal(gd, od) and np.array_equal(gc, oc)
    assert ot.max() > 100
    n, src, dst, dist, _, _ = load_routes()
    ms, md = np.concatenate([src, dst]), np.concatenate([dst, src])
    g = gpu.Graph(n, ms, md)
    o = O.OracleGraph(n, ms, md)
    gc, gt, gd, ms_k = g.clustering()
    oc, ot, od = o.clustering(n_threads=16)
    assert np.array_equal(gt, ot) and np.array_equal(gd, od) and np.array_equal(gc, oc)


def test_sssp_paths_with_forbidden_sets(gpu):
    """goal-directed searches with ForbiddenEdge / ForbiddenNode sets == the oracle's dijkstra run on
    the graph with those nodes / edges deleted (distinct weights: paths are forced)."""
    rng = np.random.default_rng(8)
    n = 200
    pairs = sorted({(int(a), int(b)) for a, b in zip(rng.integers(0, n, 1600), rng.integers(0, n, 1600)) if a != b})
    src = np.array([p[0] for p in pairs], np.uint32)
    dst = np.array([p[1] for p in pairs], np.uint32)
    w = (rng.random(src.size) * 10 + 0.5).astype(np.float32)
    g = gpu.Graph(n, src, dst, w)
    sources = rng.integers(0, n, 40).astype(np.uint32)
    goals = rng.integers(0, n, 40).astype(np.uint32)
    fn = [[int(x) for x in rng.integers(0, n, rng.integers(0, 4)) if x != sources[i]] for i in range(40)]
    fe = [[pairs[int(j)] for j in rng.integers(0, len(pairs), rng.integers(0, 5))] for i in range(40)]
    res, _ = g.sssp_paths(sources, goals, fn, fe, max_len=4)        # small buffer: exercises the retry
    for i in range(40):
        keep = np.array([(a, b) not in set(fe[i]) and b not in set(fn[i]) for a, b in pairs])
        o = O.OracleGraph(n, src[keep], dst[keep], w[keep])
        od, ob = o.sssp([int(sources[i])])
        cost, path = res[i]
        exp = float(od[0, goals[i]])
        if np.isinf(exp):
            assert np.isinf(cost) and path == []
            continue
        assert cost == exp
        p, cur = [], int(goals[i])
        while cur != int(sources[i]):
            p.append(cur)
            cur = int(ob[0, cur])
        p.append(int(sources[i]))
        assert path == p[::-1]
    plain, _ = g.sssp_paths(sources, goals)
    od, _ = O.OracleGraph(n, src, dst, w).sssp(sources)
    assert [c for c, _ in plain] == [float(od[i, goals[i]]) for i in range(40)]
