"""PageRank judged by an exact f64 iteration and a rigorous per-node rounding bound, in both engines.

Both engines (`pagerank.mode=0`, the gather pull; `pagerank.mode=1`, propagation blocking) run the Jacobi iteration
    s_{t+1}[u] = base + d * sum_{v -> u} s_t[v] / od[v]
in f32.  The reference is the same iteration in f64 (scipy sparse) with the device's f32 constants widened:
d = fl32(theta), init = fl32(1/n), base = fl32(fl32(1 - d) / n).  Parallel edges count once per edge, a self-loop counts
in the in-row and in the out-degree, dangling nodes contribute nothing.  err_t = sum |s_t - s_{t-1}|; the run stops at
the first t with err_t < fl32(tol), or at t = max_iter.  The CPU oracle is never the judge: it rounds like the device.

Per-node bound (the main check).  With u = 2^-24 and gamma_L = L u / (1 - L u), an absolute bound A_t[x] >= |s^_t[x] - s_t[x]|
(rho = A / s in relative terms) is carried through the iteration:
- A_0 = 0; a row without in-edges is exactly `base`, so A = 0 there;
- a contribution s^/od gains one rounding: |c^ - c| <= (A + u (s + A)) / od;
- a sum of non-negative terms whose summation tree has chains of at most L additions is off by at most gamma_L times
  the sum of its terms; the errors of the terms add on top;
- base + d * S costs at most two roundings (an FMA costs one, which the same bound covers).
L comes from each engine's summation structure, computed from the layout (slots = stable sort by descending out-degree):
- mode 0: in-degree k <= 256 is one lane's serial sum, L = k; 256 < k <= 4096 is one warp: ceil(k/256) + 7 + 8 (8
  accumulators per lane, at most 7 tail terms into the first, 3 pairing and 5 shuffle levels); k > 4096 is cut into 4096
  chunks: 31 + ceil(k/4096) - 1 (the chunk partials are added serially);
- mode 1: L = max(L_hub, L_M) + 1 (hub part + M part).  A hub part of h <= 64 entries is serial, a longer one is summed
  by a warp: ceil(h/32) + 5.  The M part is cut at the window bins: a piece of l entries costs l when l <= 64, else
  ceil(l/32) + 5, and a row spanning several bins adds one addition per extra bin.
A wrong, missing or duplicated term is about 1/deg relative: far outside this bound on every row class tested here.
On top, the product promise of DESIGN.md §3.3 is asserted on every graph: <= 1e-5 relative to the truth at every node.
The f64 reference itself is off by far less than 1e-12 relative, which is allowed for.

Iterations and `out_err`.  The device adds fl32(s^_t - s^_{t-1}) exactly in 2^-62 fixed point, so |err_dev - err_ref| <=
sum (A_t + A_{t-1} + u (|s_t - s_{t-1}| + A_t + A_{t-1})) + n 2^-63 (+ the conversion to double).  The device's iteration
count must be a t where that interval reaches below tol (or max_iter), with every earlier interval reaching tol, and
`out_err` must lie in the interval at that t.

Determinism is bit for bit: reruns, mode 0 across `pagerank.dynamic` and `pagerank.warps`, mode 1 across
`pagerank.chunk` and `pagerank.accumulate_threads`, and a handle switched between modes and geometries against fresh
handles.  Different hub / group / window sizes change the summation order, so across them only the bound applies.
"""
import contextlib
import os

import numpy as np
import pytest
from scipy.sparse import csr_matrix

from tests.util import rmat_edges

U = 2.0 ** -24
NATURAL = pytest.mark.skipif(bool(os.environ.get("COZO_EMU_LIB")), reason="natural-size graphs: too large for the emulated library")
DEFAULTS = {"pagerank.mode": 0, "pagerank.hub_slots": 16384, "pagerank.group_slots": 32768, "pagerank.window": 24576,
            "pagerank.chunk": 262144, "pagerank.accumulate_threads": 0, "pagerank.dynamic": 1, "pagerank.warps": 32}
# engine 0, engine 1 at its default geometry, and engine 1 at small geometries that put every boundary in reach
ENGINES = {
    "pull": {"pagerank.mode": 0},
    "pb": {"pagerank.mode": 1},
    "pb_small": {"pagerank.mode": 1, "pagerank.hub_slots": 64, "pagerank.group_slots": 256, "pagerank.window": 512,
                 "pagerank.chunk": 1024},
    "pb_nohub": {"pagerank.mode": 1, "pagerank.hub_slots": 0, "pagerank.group_slots": 64, "pagerank.window": 64,
                 "pagerank.chunk": 1024},
    "pb_odd": {"pagerank.mode": 1, "pagerank.hub_slots": 8, "pagerank.group_slots": 128, "pagerank.window": 301,
               "pagerank.chunk": 1024, "pagerank.accumulate_threads": 1024},
    "pb_mid": {"pagerank.mode": 1, "pagerank.hub_slots": 1024, "pagerank.group_slots": 4096, "pagerank.window": 3001},
}


def engines(*names):
    return [pytest.param(n, id=n) for n in (names or ENGINES)]


@contextlib.contextmanager
def options(capi, opts):
    try:
        for k, v in {**DEFAULTS, **opts}.items():
            capi.set_option(k, v)
        yield
    finally:
        for k, v in DEFAULTS.items():
            capi.set_option(k, v)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---- layout: what each engine's summation structure is, from the options the library reads -------------------------
def geometry(opts, n):
    """(mode, NH, WIN) as pagerank.cu derives them from the options"""
    o = {**DEFAULTS, **opts}
    nh = min(65536, max(0, o["pagerank.hub_slots"])) & ~3
    win = min(49152, max(64, o["pagerank.window"]))
    return o["pagerank.mode"], min(nh, n), win


def slot_rows(n, src, dst):
    """slot space: slot[v] = rank by out-degree, descending, ties in id order; in-rows sorted by source slot.
    -> (od by id, in-degree by slot, source slots of the in-rows, row pointer)"""
    od = np.bincount(src, minlength=n).astype(np.int64)
    perm = np.argsort(-od, kind="stable")
    slot = np.empty(n, np.int64)
    slot[perm] = np.arange(n)
    rs, cs = slot[dst.astype(np.int64)], slot[src.astype(np.int64)]
    order = np.lexsort((cs, rs))
    k = np.bincount(rs, minlength=n)
    ptr = np.zeros(n + 1, np.int64)
    ptr[1:] = np.cumsum(k)
    return od, slot, k, rs[order], cs[order], ptr


def chain_warp(length):
    """a lane per run of <= 64 terms, else the warp: strided lanes + 5 shuffle levels"""
    length = np.asarray(length, np.int64)
    return np.where(length <= 64, length, -(-length // 32) + 5)


def chain_lengths(n, src, dst, opts):
    """L[x] (by node id): the longest chain of f32 additions in the row sum of x, for the engine `opts` selects"""
    mode, nh, win = geometry(opts, n)
    od, slot, k, rows, cols, ptr = slot_rows(n, src, dst)
    if mode == 0:
        L = np.where(k <= 256, k, -(-k // 256) + 15)
        L = np.where(k > 4096, 31 + (-(-k // 4096)) - 1, L)
    else:
        h = np.bincount(rows[cols < nh], minlength=n)
        mc = k - h
        mptr = np.zeros(n + 1, np.int64)
        mptr[1:] = np.cumsum(mc)
        ms, me = mptr[:-1], mptr[1:]
        bs, be = ms // win, np.maximum(me - 1, 0) // win
        nb = np.where(mc > 0, be - bs + 1, 0)
        first = np.minimum(me, (bs + 1) * win) - ms
        last = me - be * win
        lm = np.maximum(chain_warp(first), np.where(nb > 1, chain_warp(last), 0))
        lm = np.maximum(lm, np.where(nb > 2, chain_warp(win), 0)) + np.maximum(nb - 1, 0)
        L = np.maximum(chain_warp(h), np.where(mc > 0, lm, 0)) + 1
    return L[slot]


# ---- the f64 reference and the bound -------------------------------------------------------------------------------
class Truth:
    """the f64 iteration for max_iter steps, with the per-node bound A_t and the err interval at every t"""

    def __init__(self, n, src, dst, theta, tol, max_iter, L):
        self.n = n
        d = np.float32(theta)
        self.init = np.float32(1) / np.float32(n)
        self.base = (np.float32(1) - d) / np.float32(n)
        self.tol = float(np.float32(tol))
        d, base = float(d), float(self.base)
        od = np.bincount(src, minlength=n).astype(np.float64)
        ind = np.bincount(dst, minlength=n)
        inv = np.divide(1.0, od, out=np.zeros(n), where=od > 0)
        A = csr_matrix((np.ones(src.size), (dst.astype(np.int64), src.astype(np.int64))), shape=(n, n))
        gam = L * U / (1 - L * U)
        s = np.full(n, float(self.init))
        a = np.zeros(n)
        self.s, self.a, self.err, self.lo, self.hi = [s], [a], [None], [None], [None]
        for _ in range(max_iter):
            S = A @ (s * inv)
            dc = A @ ((a + U * (s + a)) * inv)
            es = dc + gam * (S + dc)
            x = d * (es * (1 + U) + U * S)
            s1 = base + d * S
            a1 = np.where((ind == 0) | (d == 0.0), 0.0, x + U * (s1 + x))
            err = float(np.abs(s1 - s).sum())
            b = float((a1 + a + U * (np.abs(s1 - s) + a1 + a)).sum()) + n * 2.0 ** -63 + 1e-12 * float((s1 + s).sum())
            b += 2.0 ** -52 * (err + b)
            self.s.append(s1)
            self.a.append(a1)
            self.err.append(err)
            self.lo.append(err - b)
            self.hi.append(err + b)
            s, a = s1, a1

    def check(self, scores, iters, err, contract=True, what=""):
        """scores within the bound at every node (and the 1e-5 promise), the iteration count and out_err consistent"""
        T = len(self.s) - 1
        assert 1 <= iters <= T, (what, iters)
        s, a = self.s[iters], self.a[iters]
        g = scores.astype(np.float64)
        dev = np.abs(g - s)
        over = dev > a + 1e-12 * s
        rel = np.divide(dev, s, out=np.zeros_like(dev), where=s > 0)
        w = int(np.argmax(dev - a))
        assert not over.any(), (f"{what}: {int(over.sum())} nodes outside the rounding bound, worst at node {w}: "
                                f"|dev| {dev[w]:.3e} bound {a[w]:.3e}; max relative error {rel.max():.2e} at node "
                                f"{int(np.argmax(rel))}")
        if contract:
            assert np.all(dev[s == 0] == 0) and rel.max() <= 1e-5, (what, float(rel.max()), int(np.argmax(rel)))
        for t in range(1, iters):
            assert self.hi[t] >= self.tol, f"{what}: err at t={t} is certainly below tol, the device went on to {iters}"
        assert iters == T or self.lo[iters] < self.tol, f"{what}: err at t={iters} is certainly >= tol, the device stopped"
        assert self.lo[iters] <= err <= self.hi[iters], (what, iters, err, self.lo[iters], self.hi[iters])


def run_checked(capi, n, src, dst, opts, theta=0.85, tol=0.0, max_iter=5, contract=True, g=None, what=""):
    src = np.asarray(src, np.uint32)
    dst = np.asarray(dst, np.uint32)
    with options(capi, opts):
        g = g or capi.Graph(n, src, dst)
        scores, iters, err, _ = g.pagerank(theta, tol, max_iter)
        again = g.pagerank(theta, tol, max_iter)
    truth = Truth(n, src, dst, theta, tol, max_iter, chain_lengths(n, src, dst, opts))
    truth.check(scores, iters, err, contract, what)
    assert np.array_equal(bits(scores), bits(again[0])) and again[1] == iters and again[2] == err, f"{what}: rerun differs"
    return scores


# ---- graphs --------------------------------------------------------------------------------------------------------
def fed_rows(hub_counts, m_counts=None, p_hub=64, p_m=0):
    """Target rows fed by in-degree-0 sources of equal out-degree within each of two pools, so that every term of a row
    is equal (the case where f32 drift is worst and systematic).  Row i takes hub_counts[i] edges from the first pool
    (the highest out-degree: the first slots) and m_counts[i] from the second, round robin.  Ids: targets 0..T-1 (slots
    in this order, after the sources), sources T.., and a last node that takes the padding edges that even out the
    pools' out-degrees.  -> (n, src, dst, number of sources)"""
    hub_counts = np.asarray(hub_counts, np.int64)
    m_counts = np.zeros_like(hub_counts) if m_counts is None else np.asarray(m_counts, np.int64)
    T = hub_counts.size
    pad = T + p_hub + p_m
    n = pad + 1
    H, M = int(hub_counts.sum()), int(m_counts.sum())
    dm = -(-M // p_m) if p_m else 0
    dh = max(-(-H // p_hub), dm + 1)
    src, dst = [], []
    hs = T + np.arange(H) % p_hub
    src.append(hs)
    dst.append(np.repeat(np.arange(T), hub_counts))
    src.append(T + (np.arange(H, dh * p_hub) % p_hub))
    dst.append(np.full(dh * p_hub - H, pad))
    if p_m:
        src.append(T + p_hub + np.arange(M) % p_m)
        dst.append(np.repeat(np.arange(T), m_counts))
        src.append(T + p_hub + (np.arange(M, dm * p_m) % p_m))
        dst.append(np.full(dm * p_m - M, pad))
    return n, np.concatenate(src).astype(np.uint32), np.concatenate(dst).astype(np.uint32), p_hub + p_m


# in-degrees on every boundary of both engines: lane / warp rows, the 8-accumulator tail, the 4096 chunks
LADDER = [0, 1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 479, 480, 481, 500, 511, 512, 513, 991, 992, 993, 1010, 1023,
          2047, 2048, 2049, 4095, 4096, 4097, 8192, 8193, 3 * 4096 - 5]
# mini-blocks of the pull: 32 rows of 8 (ends at 32 rows and at 256 entries at once), 100 + 100 + 56 (256 entries in 3
# rows), then 33 rows of 1 (the 33rd opens a block), and a 256 row after a 1 row
BLOCKS = [8] * 32 + [100, 100, 56, 1] + [1] * 33 + [1, 256, 7]
# 32-row groups of K_F (targets start at slot 64): the hub-entry total T of a group on both sides of the 2048 staging
GROUPS = ([1568] + [0] * 31 + [1500] + [0] * 31 + [1600] + [0] * 31 + [2047, 1] + [0] * 30 + [2048] + [0] * 31
          + [2049] + [0] * 31 + [2047, 2] + [0] * 30 + [64, 65] + [30] * 30 + [64] * 32 + [64] * 31 + [65] + [2040]
          + [0] * 31)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines())
@pytest.mark.parametrize("iters", [3, 30])
def test_row_class_ladder(gpu, engine, iters):
    """every in-degree boundary of both engines, rows of equal terms"""
    n, src, dst, _ = fed_rows(LADDER + BLOCKS, p_hub=64)
    run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=iters, what=f"ladder {engine}")
    # the same rows split between the two pools: hub parts and M parts of every length at once
    ks = np.array(LADDER + BLOCKS)
    n, src, dst, _ = fed_rows(ks - ks // 3, ks // 3, p_hub=64, p_m=512)
    run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=iters, what=f"ladder split {engine}")


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines("pull", "pb", "pb_small", "pb_mid"))
@pytest.mark.parametrize("iters", [3, 30])
def test_hub_sum_ladder(gpu, engine, iters):
    """rows with 64 ... 2049 hub in-edges and K_F groups whose hub total is 2048 / 2049: on a graph of n <= NH at the
    default geometry every in-edge is a hub entry and only K_F runs; with a small hub table part of each row is M"""
    n, src, dst, _ = fed_rows(GROUPS, p_hub=64)
    run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=iters, what=f"hub ladder {engine}")
    n, src, dst, _ = fed_rows(GROUPS, np.array(GROUPS) // 4, p_hub=64, p_m=320)
    run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=iters, what=f"hub ladder + M {engine}")


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines("pull", "pb", "pb_small"))
@pytest.mark.parametrize("iters", [3, 30])
def test_hub_star(gpu, engine, iters):
    """node 0 fed by L sources of out-degree 1: one row of L equal hub terms (a serial f32 chain of 1568 of them drifts
    by 2e-5)"""
    for L in (64, 65, 1500, 1568, 1600, 2040, 2047, 2048, 2049, 3000):
        src = np.arange(1, L + 1, dtype=np.uint32)
        run_checked(gpu, L + 1, src, np.zeros(L, np.uint32), ENGINES[engine], max_iter=iters, what=f"star {L} {engine}")


def blocking_rows(win):
    """M parts (window `win`) that start on a bin boundary and are exactly a window long, end exactly at a bin end, span
    two and many bins, and pieces of 64 / 65 entries inside a window"""
    m = [win, win // 4, win - win // 4, win, 64, 65, max(win - 129, 3), 2 * win, 7, win - 7 + 3, 64, 65, 9 * win + 5, 0, 1,
         win + 1, win - 1, 33]
    return np.array(m * 2)


@pytest.mark.gpu
@pytest.mark.parametrize("win", [64, 301, 512])
@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("k_groups", [1, 3])
def test_blocking_geometry(gpu, win, extra, k_groups):
    """engine 1 at small geometries: NH + k GS (+ 1) sources, trailing groups without out-edges, several K_A items per
    group (chunk 1024), both K_B widths, an odd window, NH = 0"""
    gs = 128
    for nh in (64, 0):
        mrows = blocking_rows(win)
        hrows = np.arange(mrows.size) % 5 * (nh > 0)
        # with NH = 0 the first pool (4 sources, no hub entries) is simply part of the M sources
        n, src, dst, nsrc = fed_rows(hrows, mrows, p_hub=max(nh, 4), p_m=k_groups * gs + extra - (0 if nh else 4))
        assert nsrc == nh + k_groups * gs + extra
        for threads in (0, 1024):
            opts = {"pagerank.mode": 1, "pagerank.hub_slots": nh, "pagerank.group_slots": gs, "pagerank.window": win,
                    "pagerank.chunk": 1024, "pagerank.accumulate_threads": threads}
            run_checked(gpu, n, src, dst, opts, max_iter=4, what=f"blocking nh={nh} win={win} threads={threads}")


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines())
def test_degenerate_inputs(gpu, engine):
    opts = ENGINES[engine]
    e = np.zeros(0, np.uint32)
    for n, src, dst in [(1, e, e), (1, [0], [0]), (2, [0], [1]), (2, [0, 1], [1, 0]), (7, e, e),
                        (6, [0, 0, 0, 1, 1, 2, 2, 2], [0, 1, 1, 1, 2, 2, 3, 0]),            # self-loops, parallel edges
                        (50, [0, 1, 2, 3, 3], [1, 2, 3, 0, 4])]:                            # dangling, isolated ids
        for theta, tol, it in [(0.85, 0.0, 5), (0.0, 0.0, 3), (1.0, 0.0, 3), (0.85, 0.0, 1), (0.85, 1.0, 10),
                               (0.85, 1e-4, 100)]:
            s = run_checked(gpu, n, src, dst, opts, theta, tol, it, what=f"n={n} m={len(src)} theta={theta} tol={tol}")
            if len(src) == 0 or theta == 0.0:
                assert np.all(s == np.float32(1 - np.float32(theta)) / np.float32(n))   # exactly base everywhere
    with options(gpu, opts):                                                                # tol 1: one iteration
        assert gpu.Graph(3, [0, 1], [1, 2]).pagerank(0.85, 1.0, 10)[1] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines())
def test_slot_permutation(gpu, engine):
    """out-degrees 1..3 in random order: many ties, distinct scores; a wrong un-permute is an error of order one"""
    rng = np.random.default_rng(11)
    n = 3000
    od = rng.integers(1, 4, n)
    src = np.repeat(np.arange(n), od)
    dst = rng.integers(0, n, src.size)
    s = run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=8, what=f"ties {engine}")
    assert np.unique(s).size > n // 2


RMAT = [(10, 5, 0.0), (12, 50, 0.0), (14, 5, 0.0), (16, 5, 0.0), (11, 200, 1e-9), (13, 100, 1e-4)]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines("pull", "pb", "pb_small", "pb_mid"))
@pytest.mark.parametrize("scale,iters,tol", RMAT, ids=[f"rmat{s}-{i}-{t:g}" for s, i, t in RMAT])
def test_rmat(gpu, engine, scale, iters, tol):
    n, src, dst = rmat_edges(scale, 16, 0x5EED0010 + scale)
    run_checked(gpu, n, src, dst, ENGINES[engine], tol=tol, max_iter=iters, what=f"rmat{scale} {engine}")


@NATURAL
@pytest.mark.gpu
@pytest.mark.parametrize("engine", engines("pull", "pb"))
def test_rmat20_natural(gpu, engine):
    n, src, dst = rmat_edges(20, 16, 0x5EED0020)
    run_checked(gpu, n, src, dst, ENGINES[engine], max_iter=10, what=f"rmat20 {engine}")


@pytest.mark.gpu
def test_bits_do_not_depend_on_the_schedule(gpu):
    """mode 0 across dynamic / warps; mode 1 across chunk and accumulate_threads; reruns"""
    n, src, dst = rmat_edges(13, 16, 0x5EED0013)
    ladder = fed_rows(LADDER + BLOCKS, np.array(LADDER + BLOCKS) // 3, p_hub=64, p_m=512)[:3]
    for n, src, dst in [(n, src, dst), ladder]:
        g = gpu.Graph(n, src, dst)
        ref = None
        for dyn in (0, 1):
            for warps in (8, 32):
                with options(gpu, {"pagerank.mode": 0, "pagerank.dynamic": dyn, "pagerank.warps": warps}):
                    s = bits(g.pagerank(0.85, 0.0, 6)[0])
                ref = s if ref is None else ref
                assert np.array_equal(s, ref), ("mode 0", dyn, warps)
        for geo in ("pb", "pb_small", "pb_odd"):
            ref = None
            for chunk in (1024, 4096, 262144):
                for threads in (512, 1024):
                    with options(gpu, {**ENGINES[geo], "pagerank.chunk": chunk, "pagerank.accumulate_threads": threads}):
                        s = bits(g.pagerank(0.85, 0.0, 6)[0])
                    ref = s if ref is None else ref
                    assert np.array_equal(s, ref), (geo, chunk, threads)


@pytest.mark.gpu
def test_switching_engines_on_one_handle(gpu):
    """re-staging one handle between modes and geometries gives the bits of a fresh handle every time"""
    n, src, dst = rmat_edges(12, 16, 0x5EED0012)
    fresh = {}
    for name, opts in ENGINES.items():
        with options(gpu, opts):
            fresh[name] = bits(gpu.Graph(n, src, dst).pagerank(0.85, 0.0, 4)[0])
    g = gpu.Graph(n, src, dst)
    for name in ["pb_small", "pull", "pb", "pb_nohub", "pb_small", "pb_odd", "pull", "pb_mid", "pb", "pb_small"]:
        with options(gpu, ENGINES[name]):
            assert np.array_equal(bits(g.pagerank(0.85, 0.0, 4)[0]), fresh[name]), name
