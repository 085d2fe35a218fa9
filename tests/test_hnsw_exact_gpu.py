"""HNSW search judged by exact references, in every search mode, with non-finite distances ordered as the reference
orders them.

References (numpy only, never the oracle):
- distances (hnsw.rs:66-109) in f64 from the f32 operands: L2 = sum (q - x)^2, cosine = 1 - q.x / sqrt(|q|^2 |x|^2),
  IP = 1 - q.x.  For F64 indexes the same formulas in long double (64-bit mantissa), since the device sums in f64.
- a bound per (query, row) from the kernel's summation order.  Each lane accumulates m = 4 ceil(ld / 128) elements
  with fmaf (the element step of L2, q - x, rounds once more), a 5-level shuffle tree adds the 32 partials, and
  `finish` does the metric's last step in f64 and rounds to f32.  With u = 2^-24 and g = (m + 8) u / (1 - (m + 8) u):
    L2      |d - t| <= g t                                          (every term is >= 0, so the sum of |terms| is t)
    IP      |d - t| <= g S + u (|t| + g S)                          S = sum |q_j x_j|
    cosine  |r^ - r| <= (g S / N + g |r|) / (1 - g),  |d - t| <= that + u (|t| + that)     r = q.x / N, N = |q| |x|;
            q.x is off by g S, |q|^2 and |x|^2 by g relative, so N by g (the square root halves it); S <= N
  plus an absolute (2 ld + 64) 2^-149 for roundings in the subnormal range, and 2^-50 S for the reference's own
  rounding.  F64 indexes: the same with u = 2^-53.  A device +-inf is within the bound when t +- bound reaches the
  f32 overflow threshold (2^128 - 2^103); NaN matches NaN only.
- the answer of an exhaustive beam: the hand-built graphs below have a layer 0 that is strongly connected (a
  Hamiltonian cycle in both directions plus random chords) and are searched with ef >= n.  The beam is then never
  full, every node is admitted and expanded (hnsw.rs:559-581), and the answer is the first k of all rows in
  OrderedFloat order: -inf, finite ascending, +inf, NaN (NaN equal to NaN).  Two rows may swap only when their
  truths lie within the sum of their bounds (a tie window, e.g. duplicated rows); NaN never swaps with a number.
- radius and filter: the epilogue of hnsw_knn (hnsw.rs:943-1006) applied to the device's own exhaustive beam: without
  a filter the beam is cut to k first; `d > radius` drops a row (so NaN passes), the filter drops rows, then k.  The
  radius verdict of every row must be the truth's, except where the truth lies within its bound of the radius.

Every case also runs all three search modes (hnsw.mode 0: ld.global rows, 1: warp per query with the bulk-copy ring
and, for L2 at 512 <= ld <= 2048, pruning from code rows, 2: the cooperative kernel), which share one formula and one
admission order: ids, distance bits, counts and the three traversal counters must be identical.
Sizes fit the CPU-emulated library (COZO_EMU_LIB=...); natural-size cases are skipped there.
"""
import os

import numpy as np
import pytest

EMU = bool(os.environ.get("COZO_EMU_LIB"))
NATURAL = pytest.mark.skipif(EMU, reason="natural size: too large for the emulated library")
NONE = 0xFFFFFFFF
F32_OVER = 2.0 ** 128 - 2.0 ** 103          # the smallest magnitude that rounds to inf in f32
DIMS = [1, 3, 4, 5, 127, 128, 129, 255, 257, 511, 512, 513, 1023, 2047, 2048, 2049, 3072]


# ---- references ----------------------------------------------------------------------------------------------------
def truth_and_bound(X, Q, metric, f64=False):
    """-> (t, b): (B, n) exact distances and the device's error bound (module docstring)"""
    ft = np.longdouble if f64 else np.float64
    x, q = np.asarray(X).astype(ft), np.asarray(Q).astype(ft)
    dim = x.shape[1]
    ld = dim if f64 else (dim + 3) // 4 * 4
    m = (dim + 31) // 32 if f64 else 4 * ((ld + 127) // 128)
    u = 2.0 ** -53 if f64 else 2.0 ** -24
    g = (m + 8) * u / (1 - (m + 8) * u)
    absb = (2 * ld + 64) * 2.0 ** -149 if not f64 else (2 * ld + 64) * 2.0 ** -1074
    with np.errstate(all="ignore"):
        if metric == 0:
            t = ((q[:, None, :] - x[None, :, :]) ** 2).sum(-1)
            S = t
            b = g * t
        else:
            a = q @ x.T
            S = np.abs(q) @ np.abs(x).T
            if metric == 2:
                t = 1 - a
                b = g * S + u * (np.abs(t) + g * S)
            else:
                N = np.sqrt((q * q).sum(1)[:, None] * (x * x).sum(1)[None, :])
                r = a / N
                t = 1 - r
                e = (g * S / N + g * np.abs(r)) / (1 - g)
                b = e + u * (np.abs(t) + e)
        b = b + absb + 2.0 ** -50 * S
    return t.astype(np.float64), np.where(np.isnan(b), np.inf, b).astype(np.float64)


def interval(t, b):
    """[lo, hi] of values the device may return for truth t; an end past the f32 range becomes infinite"""
    with np.errstate(invalid="ignore"):
        lo = np.where(np.isinf(t), t, t - b)
        hi = np.where(np.isinf(t), t, t + b)
    return np.where(lo <= -F32_OVER, -np.inf, lo), np.where(hi >= F32_OVER, np.inf, hi)


def check_within(d, t, b, f64=False):
    """every returned distance d lies within its bound of the truth t (same shape)"""
    d = np.asarray(d, np.float64)
    lo, hi = interval(t, b) if not f64 else (t - b, t + b)
    with np.errstate(invalid="ignore"):
        ok = np.where(np.isnan(t), np.isnan(d), ~np.isnan(d) & (lo <= d) & (d <= hi))
    bad = np.nonzero(~ok)
    assert ok.all(), [(d[i], t[i], b[i]) for i in zip(*bad)][:5]


def check_ordered(d):
    """OrderedFloat order: non-decreasing numbers (infinities included), then NaN"""
    d = np.asarray(d, np.float64)
    nan = np.isnan(d)
    assert not np.any(nan[:-1] & ~nan[1:]), d
    fin = d[~nan]
    assert np.all(fin[:-1] <= fin[1:]), d


def before(ts, bs, tr, br):
    """row s certainly precedes row r in OrderedFloat order of the truths"""
    _, hi_s = interval(ts, bs)
    lo_r, _ = interval(tr, br)
    with np.errstate(invalid="ignore"):
        return (~np.isnan(ts) & np.isnan(tr)) | (~np.isnan(ts) & ~np.isnan(tr) & (hi_s < lo_r))


def check_exhaustive(ids, dist, cnt, t, b, k, f64=False):
    """the first k of the exact ranking, up to tie windows, with every distance within its bound"""
    n = t.shape[1]
    assert np.all(cnt == min(k, n))
    for qi in range(len(cnt)):
        c = int(cnt[qi])
        got = ids[qi, :c].astype(np.int64)
        assert np.all(got < n) and np.unique(got).size == c
        assert np.all(ids[qi, c:] == NONE)
        check_within(dist[qi, :c], t[qi, got], b[qi, got], f64)
        check_ordered(dist[qi, :c])
        rest = np.setdiff1d(np.arange(n), got)
        if rest.size and c:
            bad = before(t[qi, rest][:, None], b[qi, rest][:, None], t[qi, got][None, :], b[qi, got][None, :])
            assert not bad.any(), (qi, rest[np.nonzero(bad)[0][:3]])


def epilogue(bi, bd, k, radius=None, row_pass=None):
    """hnsw_knn's tail (hnsw.rs:943-1006) on a beam in device order"""
    i, d = list(bi), list(bd)
    if row_pass is None:
        i, d = i[:k], d[:k]
    keep = [(a, x) for a, x in zip(i, d)
            if not (radius is not None and float(x) > radius) and (row_pass is None or row_pass[a])]
    return keep[:k]


# ---- graphs and searches -------------------------------------------------------------------------------------------
def ring_graph(n, seed, m_max0=16, m_max=8, levels=(24, 6)):
    """layer 0: a random Hamiltonian cycle in both directions plus random chords (degree <= m_max0); upper layers: the
    same on nested random subsets.  Rows in ascending id (key order)."""
    rng = np.random.default_rng(seed)
    node_ids, row_ptr, col_idx = [None], [], []
    nodes = np.arange(n)
    layers = [nodes]
    for size in levels:
        if size < len(layers[-1]):
            layers.append(np.sort(rng.choice(layers[-1], size, replace=False)))
    for L, ns in enumerate(layers):
        mm = m_max0 if L == 0 else m_max
        adj = {int(v): set() for v in ns}
        perm = rng.permutation(ns)
        for a, c in zip(perm, np.roll(perm, 1)):
            if a != c:
                adj[int(a)].add(int(c))
                adj[int(c)].add(int(a))
        for v in ns:
            extra = rng.choice(ns, min(len(ns), mm), replace=False)
            for w in extra:
                if len(adj[int(v)]) >= mm:
                    break
                if w != v:
                    adj[int(v)].add(int(w))
        rows = [sorted(adj[int(v)]) for v in ns]
        assert max(len(r) for r in rows) <= mm
        row_ptr.append(np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint64))
        col_idx.append(np.array([w for r in rows for w in r], np.uint32))
        if L:
            node_ids.append(ns.astype(np.uint32))
    return node_ids, row_ptr, col_idx, int(layers[-1][0])


def stage(gpu, X, metric, seed, **kw):
    ni, rp, ci, ep = ring_graph(X.shape[0], seed, **kw)
    return gpu.HnswIndex.stage(X, ni, rp, ci, ep, metric=metric, m_max0=16, m_max=8)


def search_modes(gpu, g, Q, k, ef, radius=None, row_pass=None, f64=False, modes=(0, 1, 2)):
    """the same search in every mode; asserts identical ids, distance bits, counts and traversal counters"""
    outs = []
    for mode in modes:
        gpu.set_option("hnsw.mode", mode)
        try:
            fn = g.search_f64 if f64 else g.search
            ids, dist, cnt, st = fn(Q, k, ef, radius=radius, row_pass=row_pass)
        finally:
            gpu.set_option("hnsw.mode", -1)
        outs.append((ids, dist, cnt, (st.dist_evals, st.nodes_expanded, st.nbr_reads)))
    i0, d0, c0, s0 = outs[0]
    view = np.uint64 if f64 else np.uint32
    for mode, (i, d, c, s) in zip(modes[1:], outs[1:]):
        assert np.array_equal(i, i0), f"mode {mode}: ids differ from mode {modes[0]}"
        assert np.array_equal(d.view(view), d0.view(view)), f"mode {mode}: distance bits differ"
        assert np.array_equal(c, c0) and s == s0, (mode, s, s0)
    return i0, d0, c0, s0


def check_all(gpu, g, X, Q, metric, f64=False, radius=None, row_pass=None, modes=(0, 1, 2)):
    """exhaustive beam (ef >= n): exact answer at k = n and k = 10, radius and filter through the epilogue"""
    n = X.shape[0]
    ef = (n + 31) // 32 * 32
    t, b = truth_and_bound(X, Q, metric, f64)
    bi, bd, bc, st = search_modes(gpu, g, Q, n, ef, f64=f64, modes=modes)
    check_exhaustive(bi, bd, bc, t, b, n, f64)
    assert st[1] >= n * len(Q)                                  # every node expanded on layer 0 ...
    ki, kd, kc, _ = search_modes(gpu, g, Q, 10, ef, f64=f64, modes=modes)
    check_exhaustive(ki, kd, kc, t, b, 10, f64)
    view = np.uint64 if f64 else np.uint32
    assert np.array_equal(ki, bi[:, :10]) and np.array_equal(kd.view(view), bd[:, :10].view(view))  # ... whatever k
    if radius is None:
        fin = np.isfinite(t)
        radius = float(np.median(t[fin])) if fin.any() else 0.0
    if row_pass is None:
        row_pass = np.random.default_rng(n).random(n) < 0.5
    for kk, rad, rp in ((n, radius, None), (10, radius, None), (10, None, row_pass), (7, radius, row_pass)):
        ri, rd, rc, _ = search_modes(gpu, g, Q, kk, ef, radius=rad, row_pass=rp, f64=f64, modes=modes)
        for qi in range(len(Q)):
            exp = epilogue(bi[qi, :bc[qi]], bd[qi, :bc[qi]], kk, rad, rp)
            assert rc[qi] == len(exp), (qi, kk, rad is not None, rp is not None)
            assert ri[qi, :rc[qi]].tolist() == [a for a, _ in exp]
            assert np.array_equal(rd[qi, :rc[qi]].view(view), np.array([x for _, x in exp], rd.dtype).view(view))
    for qi in range(len(Q)):
        c = int(bc[qi])                                         # the device's radius verdicts are the truth's
        tt, bb = t[qi, bi[qi, :c].astype(np.int64)], b[qi, bi[qi, :c].astype(np.int64)]
        lo, hi = interval(tt, bb)
        with np.errstate(invalid="ignore"):
            sure = np.isnan(tt) | (hi < radius) | (lo > radius)
            dev_out = bd[qi, :c].astype(np.float64) > radius
            assert np.array_equal(dev_out[sure], (tt > radius)[sure])
    return bi, bd, bc, t, b


def data(n, dim, seed, metric):
    """signed normal rows with two duplicated pairs (exact ties); queries: random, a row of the index, its negation"""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    if metric == 2:
        X *= np.float32(1 / np.sqrt(dim))
    X[5] = X[1]
    X[n - 1] = X[n // 2]
    Q = rng.standard_normal((6, dim)).astype(np.float32) * (np.float32(1 / np.sqrt(dim)) if metric == 2 else 1)
    Q[3] = X[7]
    Q[4] = -X[8]
    return X, Q


# ---- the references themselves, on the CPU -------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [0, 1, 2])
def test_bound_covers_f32_lane_order(metric):
    """the bound against a numpy emulation of the kernel's order (fmaf per lane in f64-then-f32 steps, shuffle tree),
    and the rank check rejects a swap outside a tie window"""
    rng = np.random.default_rng(7 + metric)
    for dim in (5, 129, 3072):
        X = rng.standard_normal((40, dim)).astype(np.float32) * np.float32(3)
        Q = rng.standard_normal((3, dim)).astype(np.float32)
        t, b = truth_and_bound(X, Q, metric)
        ld = (dim + 3) // 4 * 4
        xp = np.zeros((40, ld), np.float32)
        qp = np.zeros((3, ld), np.float32)
        xp[:, :dim], qp[:, :dim] = X, Q
        lane = (np.arange(ld) // 4) % 32

        def lane_sum(p):                      # p: (..., ld) f32 products summed per lane in element order, then tree
            acc = np.zeros(p.shape[:-1] + (32,), np.float32)
            for j in range(ld):
                acc[..., lane[j]] = (acc[..., lane[j]].astype(np.float64) + p[..., j]).astype(np.float32)
            for o in (16, 8, 4, 2, 1):
                acc = (acc + acc[..., np.arange(32) ^ o]).astype(np.float32)
            return acc[..., 0]
        if metric == 0:
            diff = (qp[:, None, :] - xp[None, :, :]).astype(np.float32)
            d = lane_sum(diff.astype(np.float64) ** 2)
        else:
            a = lane_sum(qp[:, None, :].astype(np.float64) * xp[None, :, :]).astype(np.float64)
            if metric == 2:
                d = (1.0 - a).astype(np.float32)
            else:
                qn = lane_sum(qp.astype(np.float64) ** 2).astype(np.float64)
                xn = lane_sum(xp.astype(np.float64) ** 2).astype(np.float64)
                d = (1.0 - a / np.sqrt(qn[:, None] * xn[None, :])).astype(np.float32)
        check_within(d, t, b)
        assert np.abs(d - t).max() > 0                           # the emulation does round
    # the rank check: row 1 (truth 1) certainly precedes row 2 (truth 2, or NaN), so [0, 2] is not a top 2
    cnt = np.array([2], np.uint32)
    ids = np.array([[0, 2]], np.uint32)
    tt = np.array([[0.0, 1.0, 2.0]])
    check_exhaustive(np.array([[0, 1]], np.uint32), np.array([[0, 1]], np.float32), cnt, tt, tt * 0 + 1e-9, 2)
    for t2, d2 in ((2.0, 2.0), (np.nan, np.nan)):
        tt[0, 2] = t2
        with pytest.raises(AssertionError):
            check_exhaustive(ids, np.array([[0, d2]], np.float32), cnt, tt, tt * 0 + 1e-9, 2)
    with pytest.raises(AssertionError):                         # NaN before a number
        check_ordered(np.array([0.0, np.nan, 1.0]))


def test_epilogue_keeps_nan_rows_inside_a_radius():
    assert [a for a, _ in epilogue([1, 2, 3], [0.5, 5.0, np.nan], 3, radius=1.0)] == [1, 3]
    assert [a for a, _ in epilogue([1, 2, 3], [0.5, 5.0, np.nan], 2, radius=1.0)] == [1]     # cut to k first


# ---- every register width, every metric, all modes: the exact answer -----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1, 2], ids=["l2", "cosine", "ip"])
@pytest.mark.parametrize("dim", DIMS)
def test_exhaustive_beam_exact(gpu, dim, metric):
    n = 96
    X, Q = data(n, dim, 1000 * dim + metric, metric)
    g = stage(gpu, X, metric, dim)
    check_all(gpu, g, X, Q, metric)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1, 2], ids=["l2", "cosine", "ip"])
@pytest.mark.parametrize("dim", [1, 129, 2049])
def test_exhaustive_beam_exact_f64(gpu, dim, metric):
    """F64 indexes have one kernel (no modes); zero rows make cosine NaN there too"""
    n = 96
    rng = np.random.default_rng(dim + metric)
    X = rng.standard_normal((n, dim))
    Q = rng.standard_normal((5, dim))
    X[5] = X[1]
    if metric == 1:
        X[[9, 40]] = 0.0
        Q[4] = 0.0
    g = stage(gpu, X, metric, dim)
    bi, bd, bc, t, b = check_all(gpu, g, X, Q, metric, f64=True, modes=(-1,))
    if metric == 1:
        assert np.isnan(bd[:4, n - 2:]).all() and set(bi[0, n - 2:]) == {9, 40} and np.isnan(bd[4]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1e12, 1e-12])
@pytest.mark.parametrize("dim", [16, 600])
def test_cosine_norm_product_outside_f32(gpu, dim, scale):
    """|q|^2 |x|^2 overflows (1e12) or underflows (1e-12) f32 while each norm does not: the final step is in f64"""
    X, Q = data(96, dim, dim + 5, 1)
    X, Q = X * np.float32(scale), Q * np.float32(scale)
    check_all(gpu, stage(gpu, X, 1, dim + 2), X, Q, 1)


# ---- non-finite distances ------------------------------------------------------------------------------------------
def nonfinite_case(kind, dim, n):
    rng = np.random.default_rng(dim + len(kind))
    X = rng.standard_normal((n, dim)).astype(np.float32)
    Q = rng.standard_normal((5, dim)).astype(np.float32)
    if kind == "cosine_zero":
        X[[3, 17, n - 1]] = 0.0
        Q[4] = 0.0                                               # every distance NaN
        return 1, X, Q
    if kind == "l2_nonfinite":
        X[3, 0] = np.nan
        X[17, dim // 2] = np.inf
        X[30, dim - 1] = -np.inf
        X[31, 0], X[31, dim - 1] = np.inf, -np.inf
        X[n - 1, :] = np.nan
        return 0, X, Q
    assert kind == "ip_overflow"
    Q = np.maximum(np.abs(Q), np.float32(1.0))
    X *= np.float32(1 / np.sqrt(dim))
    X[[4, 20]] = np.float32(3e38)                                # q.x overflows f32: 1 - q.x = -inf
    X[[6, 50]] = np.float32(-3e38)                               # 1 + inf = +inf
    X[9] = np.float32(3e38)
    X[9, 0] = np.nan                                             # NaN
    return 2, X, Q


NONFINITE = ["cosine_zero", "l2_nonfinite", "ip_overflow"]


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 600])
@pytest.mark.parametrize("kind", NONFINITE)
def test_nonfinite_exhaustive_in_ordered_float_order(gpu, kind, dim):
    """-inf, then finite ascending, then +inf, then NaN; a radius keeps the NaN rows (NaN > r is false)"""
    n = 96
    metric, X, Q = nonfinite_case(kind, dim, n)
    g = stage(gpu, X, metric, dim + 1)
    bi, bd, bc, t, b = check_all(gpu, g, X, Q, metric)
    nan_rows = np.isnan(t)
    assert nan_rows.any()
    for qi in range(len(Q)):
        c = int(bc[qi])
        assert np.isnan(bd[qi, :c]).sum() == nan_rows[qi].sum()
    if kind == "ip_overflow":
        assert (bd == -np.inf).any() and (bd == np.inf).any()
    # radius: every NaN row of the beam survives (k = n, so nothing is cut before the radius)
    ri, rd, rc, _ = search_modes(gpu, g, Q, n, (n + 31) // 32 * 32, radius=0.0)
    for qi in range(len(Q)):
        assert np.isnan(rd[qi, :rc[qi]]).sum() == nan_rows[qi].sum()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", NONFINITE)
def test_nonfinite_partial_beam(gpu, kind):
    """ef < n: results sorted in OrderedFloat order, finite answers within their bound, modes identical"""
    n, dim = 600, 520
    metric, X, Q = nonfinite_case(kind, dim, n)
    g = stage(gpu, X, metric, 77)
    t, b = truth_and_bound(X, Q, metric)
    for k, ef in ((10, 32), (32, 32)):
        ids, dist, cnt, _ = search_modes(gpu, g, Q, k, ef)
        for qi in range(len(Q)):
            c = int(cnt[qi])
            got = ids[qi, :c].astype(np.int64)
            assert c == k and np.unique(got).size == c
            check_ordered(dist[qi, :c])
            check_within(dist[qi, :c], t[qi, got], b[qi, got])


# ---- pruned search on hard data ------------------------------------------------------------------------------------
HARD = ["negative", "constant_rows", "outlier", "offset_1e6", "tiny_and_subnormal", "overflow_1e19", "nonfinite_rows"]


def hard_data(kind, n, dim, seed):
    rng = np.random.default_rng(seed)
    X = rng.random((n, dim), dtype=np.float32)
    if kind == "negative":
        X = rng.standard_normal((n, dim)).astype(np.float32) - np.float32(0.5)
    elif kind == "constant_rows":
        X[: n // 2] = rng.standard_normal((n // 2, 1)).astype(np.float32)
    elif kind == "outlier":
        X[np.arange(n), rng.integers(0, dim, n)] = np.float32(1e4)
    elif kind == "offset_1e6":
        X += np.float32(1e6)
    elif kind == "tiny_and_subnormal":
        X *= np.float32(1e-30)
        X[: n // 4] = rng.integers(0, 1 << 20, (n // 4, dim)).astype(np.uint32).view(np.float32)       # subnormals
    elif kind == "overflow_1e19":
        X[: n // 3] *= np.float32(1e19)
    elif kind == "nonfinite_rows":
        X[5, 3] = np.inf
        X[6, 0] = -np.inf
        X[7, dim - 1] = np.nan
        X[8] = np.nan
    assert X.dtype == np.float32
    step = np.abs(np.diff(X[:50], axis=0))
    scale = np.float32(np.median(step[np.isfinite(step)]))
    Q = X[rng.integers(0, n, 5)] + (rng.random((5, dim), dtype=np.float32) - np.float32(0.5)) * scale
    far = np.where(np.isfinite(X[0]), X[0], 0).astype(np.float32) * np.float32(1e4) + np.float32(1e4)
    qnan = Q[0].copy()
    qnan[dim // 3] = np.nan
    Q = np.vstack([Q, np.zeros((1, dim), np.float32), far[None, :], qnan[None, :]]).astype(np.float32)
    return X, Q


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [512, 1023, 2048])
@pytest.mark.parametrize("kind", HARD)
def test_pruned_search_on_hard_data(gpu, kind, dim):
    """L2 with code rows (512 <= ld <= 2048), beam full (ef < n): mode 1 prunes, 0 and 2 do not; all identical, and
    every answer within the f64 bound, in OrderedFloat order"""
    n = 400
    X, Q = hard_data(kind, n, dim, dim * 7 + len(kind))
    g = stage(gpu, X, 0, dim + len(kind))
    t, b = truth_and_bound(X, Q, 0)
    ids, dist, cnt, _ = search_modes(gpu, g, Q, 10, 32)
    assert np.all(cnt == 10)
    for qi in range(len(Q)):
        got = ids[qi].astype(np.int64)
        assert np.unique(got).size == 10
        check_ordered(dist[qi])
        check_within(dist[qi], t[qi, got], b[qi, got])
    if kind == "overflow_1e19":                                 # the far query's squared distances overflow f32
        assert np.isinf(dist).any() and np.isfinite(dist).any()


# ---- a device-built cosine index with zero rows --------------------------------------------------------------------
@pytest.mark.gpu
def test_device_build_with_zero_rows(gpu):
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    n, dim, m = 800, 24, 8
    rng = np.random.default_rng(31)
    X = rng.standard_normal((n, dim)).astype(np.float32)
    zero = rng.choice(n, n // 100, replace=False)
    X[zero] = 0.0
    g = gpu.HnswIndex.build(X, metric=gpu.COSINE, m=m, ef_construction=48, level_seed=5)
    ni, rp, ci, ep = g.export_levels()
    for L in range(len(rp)):
        deg = np.diff(rp[L].astype(np.int64))
        assert deg.max() <= (2 * m if L == 0 else m)
        nodes = np.arange(n) if L == 0 else ni[L].astype(np.int64)
        src = np.repeat(nodes, deg)
        assert np.all(ci[L] < n) and not np.any(src == ci[L])
        key = src * n + ci[L]
        assert np.unique(key).size == key.size, f"duplicate neighbours on layer {L}"
        if L:
            assert np.all(np.isin(ci[L], ni[L]))
    Q = rng.standard_normal((16, dim)).astype(np.float32)
    Q[3] = 0.0
    Q[4] = X[zero[0]] + 1.0
    t, b = truth_and_bound(X, Q, 1)
    for k, ef in ((10, 32), (40, 64)):
        ids, dist, cnt, _ = search_modes(gpu, g, Q, k, ef)
        for qi in range(len(Q)):
            c = int(cnt[qi])
            got = ids[qi, :c].astype(np.int64)
            assert np.unique(got).size == c
            check_ordered(dist[qi, :c])
            check_within(dist[qi, :c], t[qi, got], b[qi, got])
    a0 = csr_matrix((np.ones(ci[0].size), (np.repeat(np.arange(n), np.diff(rp[0].astype(np.int64))), ci[0])),
                    shape=(n, n))
    if connected_components(a0, directed=True, connection="strong")[0] == 1:
        staged = gpu.HnswIndex.stage(X, ni, rp, ci, ep, metric=gpu.COSINE, m_max0=2 * m, m_max=m)
        check_all(gpu, staged, X, Q, 1)


# ---- natural size --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@NATURAL
@pytest.mark.parametrize("metric", [0, 1, 2], ids=["l2", "cosine", "ip"])
def test_exhaustive_beam_natural_size(gpu, metric):
    """2000 rows at D = 768 with ef = 2016: the whole index in one beam, in every mode"""
    n, dim = 2000, 768
    X, Q = data(n, dim, 77 + metric, metric)
    if metric == 1:
        X[[11, 600]] = 0.0
    g = stage(gpu, X, metric, 78)
    check_all(gpu, g, X, Q, metric)
