"""The source-sharded graph calls (cozo_gpu_graph_attach_sharded, cozo_gpu_closeness_sharded,
cozo_gpu_betweenness_sharded, cozo_gpu_sssp_goals_sharded) on the emulated library (tests/emu/build_emu_lib.py), with
the ranks of a communicator as threads of this process (tests/emu/fake_nccl.cpp).  Usage: graph_sharded_emu.py <path to
libcozo_gpu_emu.so>.  Prints EMU_OK at the end.  TEST INFRASTRUCTURE ONLY.

At world sizes 1, 2, 3 and 8 (8 where 8 cores exist) on two random multigraphs (one with unique shortest paths), weighted R-MAT-10 and R-MAT-12 and the
air-routes graph, on every rank:
- closeness equals the single-GPU call bit for bit; sssp_goals has the single-GPU costs bit for bit and, with keep_ties,
  its offsets and per-source tie-edge multisets (the single-GPU call lists them in no particular order within a source).
  Among tied shortest paths the single-GPU call itself may return any one, so paths equal it (offsets and rows
  array_equal) on a graph whose shortest paths are unique, and elsewhere each path walks tie edges from its start to
  its goal;
- betweenness is equal across ranks and reruns and within 2^-23 relative of the exact f64 Brandes judge of
  tests/test_graph_exact_gpu.py;
- graphs that differ between ranks, different calls or arguments on different ranks (two rules run concurrently in
  different orders) and an argument check that fails on one rank give EINVAL, a poisoned rank (with an empty slice
  too) EKILLED and a zero-weight cycle in one rank's slice EUNSUP, on every rank and without a rank left waiting; a row capacity too small reports the same total and offsets
  as on one GPU, and more ranks than sources work.
"""
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from cozo_b200 import capi  # noqa: E402

capi.LIB_PATH = os.path.abspath(sys.argv[1])
assert capi._lib is None
os.environ["COZO_GPU_NCCL_LIB"] = os.path.join(os.path.dirname(capi.LIB_PATH), "libfake_nccl.so")
from tests.test_air_routes_cpu import load_routes  # noqa: E402
from tests.test_graph_exact_gpu import betweenness_truth, check_betweenness, exact_dist, to_f32  # noqa: E402
from tests.util import rmat_edges  # noqa: E402

T0 = time.time()
WORLDS = (1, 2, 3, 8) if (os.cpu_count() or 1) >= 8 else (1, 2, 3)


def step(msg):
    print(f"[{time.time() - T0:7.1f}s] {msg}", flush=True)


def run_ranks(world, fn):
    """fn(rank) on `world` threads -> list of results; every exception is collected, a rank that never returns fails"""
    errors, results = [], [None] * world

    def main(r):
        try:
            results[r] = fn(r)
        except BaseException as e:  # noqa: BLE001
            import traceback
            errors.append(f"rank {r}: {e!r}\n{traceback.format_exc()}")
    th = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(1200)
    assert not any(t.is_alive() for t in th), "a rank hangs"
    assert not errors, "\n".join(errors)
    return results


def expect_code(code, fn):
    try:
        fn()
    except capi.CozoGpuError as e:
        assert e.code == code, e
        return
    raise AssertionError(f"expected code {code}")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def sort_rows(r):
    r = np.asarray(r, np.uint32).reshape(-1, 2)
    return r[np.lexsort((r[:, 1], r[:, 0]))]


def dyadic(rng, m):
    return (rng.integers(1, 64, m) / 8.0).astype(np.float32)


def unique(rng, m):
    """weights k/1024 with 1 <= k < 2^20: path sums exact in f32 and practically never tied"""
    return (rng.integers(1, 1 << 20, m) / 1024.0).astype(np.float32)


def graphs():
    rng = np.random.default_rng(0x5A4C)
    n, m = 150, 900
    src, dst = rng.integers(0, n, m).astype(np.uint32), rng.integers(0, n, m).astype(np.uint32)
    yield "random-unique-paths", n, src, dst, unique(rng, m), True
    rng = np.random.default_rng(0x5A4D)
    n, m = 150, 900                                     # parallel edges and self-loops; the last ids have no edges
    src, dst = rng.integers(0, n - 6, m).astype(np.uint32), rng.integers(0, n - 6, m).astype(np.uint32)
    yield "random-multigraph", n, src, dst, dyadic(rng, m), True
    n, src, dst = rmat_edges(10, 8, 0x5A4E)
    yield "rmat10", n, src, dst, dyadic(np.random.default_rng(1), src.size), True
    n, src, dst = rmat_edges(12, 8, 0x5A4F)
    yield "rmat12", n, src, dst, dyadic(np.random.default_rng(2), src.size), False
    n, src, dst, dist, _, _ = load_routes()
    yield "air-routes", n, src, dst, dist, False


def group_call(world, n, src, dst, w, call, poison_rank=None):
    """every rank stages its own copy of the graph, attaches it and runs call(grp, poison) -> per-rank results"""
    uid = capi.ShardGroup.unique_id()

    def rank_main(r):
        g = capi.Graph(n, src, dst, w)
        grp = capi.ShardGroup(uid, r, world)
        try:
            grp.attach_graph(g)
            return call(grp, np.ones(1, np.int32) if r == poison_rank else None)
        finally:
            grp.close()
            g.close()
    return run_ranks(world, rank_main)


def check_paths_on_ties(sources, goals, cost, off, rows, toff, trows):
    """every path: [start] for goal == start, [] when unreachable, else start..goal over tie edges of its source"""
    ng = goals.size
    off, toff = off.astype(np.int64), toff.astype(np.int64)
    for si, s in enumerate(sources.tolist()):
        ties = {tuple(e) for e in trows[2 * toff[si]:2 * toff[si + 1]].reshape(-1, 2).tolist()}
        for gi, t in enumerate(goals.tolist()):
            p = rows[off[si * ng + gi]:off[si * ng + gi + 1]].tolist()
            if not np.isfinite(cost[si, gi]):
                assert p == []
            elif t == s:
                assert p == [s]
            else:
                assert p[0] == s and p[-1] == t and all((b, a) in ties for a, b in zip(p, p[1:])), (s, t, p)


def check_graph(name, n, src, dst, w, centrality):
    g = capi.Graph(n, src, dst, w)
    rng = np.random.default_rng(n)
    sources = np.unique(rng.choice(n, min(n, 40), replace=False)).astype(np.uint32)
    goals = rng.choice(n, 9, replace=False).astype(np.uint32)
    want_goals = {kt: capi.sssp_goals_once(capi.load().cozo_gpu_sssp_goals, g._h, sources, goals, kt, 1 << 20)
                  for kt in (False, True)}
    if centrality:
        want_c, _ = g.closeness()
        want_b1, _ = g.betweenness()
        truth = betweenness_truth(n, src, dst, w, to_f32(exact_dist(n, src, dst, w, np.arange(n))))
        check_betweenness(want_b1, truth)
    else:
        want_c = want_b1 = truth = None
    entry = capi.load().cozo_gpu_sssp_goals_sharded
    for world in WORLDS:
        def call(grp, _):
            out = {kt: capi.sssp_goals_once(entry, grp._h, sources, goals, kt, 1 << 20) for kt in (False, True)}
            if centrality:
                out["c"] = grp.closeness()[0]
                out["b"] = [grp.betweenness()[0] for _ in range(2)]
            return out
        for r, got in enumerate(call_all := group_call(world, n, src, dst, w, call)):
            gc, go, gr, _ = got[False]
            tc, to, tr, _ = got[True]
            wc, wo, wr, _ = want_goals[False]
            assert np.array_equal(bits(gc), bits(wc)) and np.array_equal(bits(tc), bits(wc)), (name, world, r)
            assert np.array_equal(to, want_goals[True][1]), (name, world, r)
            o = to.astype(np.int64)
            for si in range(sources.size):
                a, b = 2 * o[si], 2 * o[si + 1]
                assert np.array_equal(sort_rows(tr[a:b]), sort_rows(want_goals[True][2][a:b])), (name, world, r, si)
            check_paths_on_ties(sources, goals, gc, go, gr, to, tr)
            if name == "random-unique-paths":
                assert np.array_equal(go, wo) and np.array_equal(gr[:int(wo[-1])], wr[:int(wo[-1])]), (name, world, r)
            if centrality:
                assert np.array_equal(bits(got["c"]), bits(want_c)), (name, world, r)
                b0 = call_all[0]["b"][0]
                assert all(np.array_equal(bits(x), bits(b0)) for x in got["b"]), (name, world, r)
                if world == 1:
                    assert np.array_equal(bits(got["b"][0]), bits(want_b1))
        if centrality:
            check_betweenness(call_all[0]["b"][0], truth)
        step(f"{name} (n {n}, m {src.size}) world {world}: sssp_goals costs and tie edges == single GPU, paths "
             + ("== single GPU" if name == "random-unique-paths" else "over tie edges")
             + (", closeness == single GPU, betweenness equal across ranks and reruns, within 2^-23 of the exact judge"
                if centrality else "") + " on every rank")


def check_chunks_and_forms():
    """source chunks of one source and of 7, HBM state: still equal to the single-GPU calls"""
    rng = np.random.default_rng(77)
    n, m = 90, 500
    src, dst, w = rng.integers(0, n, m).astype(np.uint32), rng.integers(0, n, m).astype(np.uint32), unique(rng, m)
    g = capi.Graph(n, src, dst, w)
    goals = np.array([3, 50, 80], np.uint32)
    for opts in ({"sssp.max_chunk_sources": 1}, {"sssp.max_chunk_sources": 7, "sssp.smem": 0}):
        for k, v in opts.items():
            capi.set_option(k, v)
        want = (g.closeness()[0], g.betweenness()[0], g.sssp_goals(np.arange(n), goals))
        for world in (2, 3):
            for got in group_call(world, n, src, dst, w,
                                  lambda grp, _: (grp.closeness()[0], grp.betweenness()[0],
                                                  grp.sssp_goals(np.arange(n), goals))):
                assert np.array_equal(bits(got[0]), bits(want[0]))
                assert np.allclose(got[1], want[1], rtol=2.0 ** -22, atol=0)
                assert np.array_equal(bits(got[2][0]), bits(want[2][0])) and got[2][1] == want[2][1]
        capi.set_option("sssp.max_chunk_sources", 0)
        capi.set_option("sssp.smem", 1)
    step("source chunks of 1 and 7 sources, HBM state: closeness and sssp_goals == single GPU at world 2 and 3")


def check_errors():
    rng = np.random.default_rng(5)
    n, m = 60, 300
    src, dst, w = rng.integers(0, n, m).astype(np.uint32), rng.integers(0, n, m).astype(np.uint32), dyadic(rng, m)
    # graphs that differ: one weight on rank 1; then a different node count on rank 1
    def bump(x):
        x = x.copy()
        x[17] += np.float32(0.125)
        return x
    for world in (2, 3):
        uid = capi.ShardGroup.unique_id()

        def rank_main(r):
            g = capi.Graph(n + (1 if r == 1 else 0), src, dst, bump(w) if r == 2 else w)
            grp = capi.ShardGroup(uid, r, world)
            expect_code(capi.E_INVAL, lambda: grp.attach_graph(g))
            grp.graph = g
            expect_code(capi.E_INVAL, lambda: grp.closeness())       # no graph attached
            expect_code(capi.E_INVAL, lambda: grp.sssp_goals([0], [1]))
            grp.close()
        run_ranks(world, rank_main)
        uid = capi.ShardGroup.unique_id()

        def rank_main_w(r):
            g = capi.Graph(n, src, dst, bump(w) if r == world - 1 else w)
            grp = capi.ShardGroup(uid, r, world)
            expect_code(capi.E_INVAL, lambda: grp.attach_graph(g))
            grp.close()
        run_ranks(world, rank_main_w)
    step("graphs that differ in n or in one weight: EINVAL on every rank at attach, and the group has no graph")
    # a poisoned rank: the same EKILLED everywhere, then the group still works
    for world in (2, 3, 8):
        def call(grp, poison):
            for fn in (lambda: grp.closeness(poison=poison), lambda: grp.betweenness(poison=poison),
                       lambda: grp.sssp_goals(np.arange(n), [1, 2], poison=poison),
                       lambda: grp.sssp_goals(np.arange(n), [1, 2], keep_ties=True, poison=poison)):
                expect_code(capi.E_KILLED, fn)
            return grp.closeness()[0]
        outs = group_call(world, n, src, dst, w, call, poison_rank=1)
        assert all(np.array_equal(bits(o), bits(outs[0])) for o in outs)
    step("poison on rank 1: EKILLED from every call on every rank; the next call on the group succeeds")
    # a zero-weight cycle that only the last slice reaches: 57 -> 58 -> 59 -> 58, reached from source 57 alone
    zs = np.concatenate([src[(src < 57) & (dst < 57)], [57, 58, 59]]).astype(np.uint32)
    zd = np.concatenate([dst[(src < 57) & (dst < 57)], [58, 59, 58]]).astype(np.uint32)
    zw = np.concatenate([w[(src < 57) & (dst < 57)], [1.0, 0.0, 0.0]]).astype(np.float32)
    expect_code(capi.E_UNSUP, lambda: capi.Graph(n, zs, zd, zw).betweenness())
    for world in (1, 2, 3, 8):
        def call(grp, _):
            expect_code(capi.E_UNSUP, lambda: grp.betweenness())
            return grp.closeness()[0]
        group_call(world, n, zs, zd, zw, call)
    step("a zero-weight cycle reached from the last slice only: EUNSUP on every rank at world 1, 2, 3, 8")
    # row capacity too small: the same costs, offsets and total as on one GPU, no row written; the retry completes
    w = unique(rng, m)
    g = capi.Graph(n, src, dst, w)
    sources, goals = np.arange(30, dtype=np.uint32), np.array([5, 9, 13, 40], np.uint32)
    single = capi.load().cozo_gpu_sssp_goals
    for kt in (False, True):
        wc, wo, _, _ = capi.sssp_goals_once(single, g._h, sources, goals, kt, 1)
        full = g.sssp_goals(sources, goals, keep_ties=kt)
        assert int(wo[-1]) > 1
        for world in (2, 3):
            def call(grp, _):
                return (capi.sssp_goals_once(capi.load().cozo_gpu_sssp_goals_sharded, grp._h, sources, goals, kt, 1),
                        grp.sssp_goals(sources, goals, keep_ties=kt))
            for (gc, go, gr, _), again in group_call(world, n, src, dst, w, call):
                assert np.array_equal(bits(gc), bits(wc)) and np.array_equal(go, wo)
                assert not gr.any()
                assert np.array_equal(bits(again[0]), bits(full[0]))
                if kt:
                    assert all(np.array_equal(sort_rows(a), sort_rows(b)) for a, b in zip(again[1], full[1]))
                else:
                    assert again[1] == full[1]
    step("capacity 1: costs, offsets and total as on one GPU, no row written; the retry equals the single-GPU call")
    # more ranks than sources, no goals, no sources
    want = g.sssp_goals([4, 7, 11], [2, 30])
    for got in group_call(8, n, src, dst, w, lambda grp, _: (grp.sssp_goals([4, 7, 11], [2, 30]),
                                                             grp.sssp_goals([1, 2], []), grp.sssp_goals([], [3]))):
        assert np.array_equal(bits(got[0][0]), bits(want[0])) and got[0][1] == want[1]
        assert got[1][0].shape == (2, 0) and got[2][0].shape == (0, 1)
    e = capi.Graph(0, [], [])
    for got in group_call(3, 0, np.zeros(0, np.uint32), np.zeros(0, np.uint32), None,
                          lambda grp, _: (grp.closeness()[0], grp.betweenness()[0])):
        assert got[0].size == 0 and got[1].size == 0
    e.close()
    step("world 8 with 3 sources, no goals, no sources, an empty graph: as on one GPU")
    check_mismatched_calls(n, src, dst, w)


def check_mismatched_calls(n, src, dst, w):
    """ranks that make different calls at the same time (two rules of one stratum run in different orders), pass
    different arguments, or fail an argument check alone: the same error on every rank, no rank left waiting, and the
    group works afterwards"""
    L = capi.load()
    sources, goals = np.arange(20, dtype=np.uint32), np.array([5, 9], np.uint32)
    want_c = capi.Graph(n, src, dst, w).closeness()[0]
    for world in (2, 3, 8):
        def call(grp, _):
            r = grp.rank
            # closeness on rank 0, betweenness elsewhere: both computed their slices, then EINVAL everywhere
            expect_code(capi.E_INVAL, (lambda: grp.closeness()) if r == 0 else (lambda: grp.betweenness()))
            # sssp_goals with other sources, other goals, another keep_ties or another capacity on one rank
            for i, (srcs, gls, kt, cap) in enumerate([(sources[:-1], goals, False, 100), (sources, goals[:1], False, 100),
                                                      (sources, goals, True, 100), (sources, goals, False, 101)]):
                mine = (srcs, gls, kt, cap) if r == world - 1 else (sources, goals, False, 100)
                expect_code(capi.E_INVAL, lambda: capi.sssp_goals_once(L.cozo_gpu_sssp_goals_sharded, grp._h, *mine))
            # sssp_goals on rank 0 against closeness elsewhere
            expect_code(capi.E_INVAL, (lambda: grp.sssp_goals(sources, goals)) if r == 0 else (lambda: grp.closeness()))
            # a null output on one rank only: that rank's EINVAL on every rank
            if r == 1:
                assert L.cozo_gpu_closeness_sharded(grp._h, None, None, None) == capi.E_INVAL
            else:
                expect_code(capi.E_INVAL, lambda: grp.closeness())
            # an attach on rank 0 while the others run closeness: EINVAL everywhere; rank 0 now has no graph, so the
            # next closeness fails on every rank, and a collective attach restores the group
            g2 = grp.graph
            expect_code(capi.E_INVAL, (lambda: grp.attach_graph(g2)) if r == 0 else (lambda: grp.closeness()))
            expect_code(capi.E_INVAL, lambda: grp.closeness())
            grp.attach_graph(g2)
            return grp.closeness()[0]
        for got in group_call(world, n, src, dst, w, call):
            assert np.array_equal(bits(got), bits(want_c))
    step("different calls or arguments on different ranks, a null output or a missing graph on one rank: EINVAL on "
         "every rank at world 2, 3, 8, no rank left waiting; the group answers correctly afterwards")
    # a poisoned rank whose slice is empty (8 ranks, 3 sources) still stops the call on every rank
    for poisoned_rank in (0, 7):
        def call(grp, poison):
            for fn in (lambda: grp.sssp_goals([4, 7, 11], [2, 30], poison=poison),
                       lambda: grp.sssp_goals([4, 7, 11], [2, 30], keep_ties=True, poison=poison)):
                expect_code(capi.E_KILLED, fn)
        group_call(8, n, src, dst, w, call, poison_rank=poisoned_rank)
    tiny = np.array([0, 1], np.uint32), np.array([1, 2], np.uint32), np.array([1, 1], np.float32)
    for poisoned_rank in (0, 7):                        # 3 nodes on 8 ranks: ranks with empty slices
        def call(grp, poison):
            expect_code(capi.E_KILLED, lambda: grp.closeness(poison=poison))
            expect_code(capi.E_KILLED, lambda: grp.betweenness(poison=poison))
        group_call(8, 3, *tiny, call, poison_rank=poisoned_rank)
    step("poison on a rank with an empty slice (world 8, 3 sources / 3 nodes): EKILLED on every rank")


if __name__ == "__main__":
    capi.init(0)
    check_errors()
    check_chunks_and_forms()
    for name, n, src, dst, w, centrality in graphs():
        check_graph(name, n, src, dst, w, centrality)
    print("EMU_OK")
