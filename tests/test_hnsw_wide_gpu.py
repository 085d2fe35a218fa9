"""f32 indexes wider than the register query (ld > 2048): the search kernels keep the query in shared memory, the builder
and maintenance passes read base vectors in place.  Same bar as test_hnsw_gpu.py: GPU search == oracle search on the
same graph (equal counts, recall >= 0.999, identical sets >= 99.5 %, distances within 1e-5 relative, traversal
counters within 0.1 %).  Sizes are small enough for the emulated library too."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.util import uniform_vectors, recall, SEED_LEVEL

pytestmark = pytest.mark.gpu
EMU = bool(os.environ.get("COZO_EMU_LIB"))
DIST_RTOL = 1e-5


def _oracle_index(n, dim, m, efc, metric=O.L2, shift=0.0, seed=0):
    X = uniform_vectors(n, dim, seed) - np.float32(shift)
    ix = O.OracleHnsw.new(n, dim, metric=metric, m=m, ef_construction=efc, level_seed=SEED_LEVEL)
    ix.insert_all(X)
    return X, ix


def _stage(gpu, X, lv, metric, m):
    return gpu.HnswIndex.stage(X, lv.node_ids, lv.row_ptr, lv.col_idx, lv.entry, metric=metric, m_max0=2 * m, m_max=m)


def _view(g, X, metric=O.L2):
    ni, rp, ci, ep = g.export_levels()
    return (ni, rp, ci, ep), O.OracleHnsw.from_levels(X, O.HnswLevels(ni, rp, ci, ep), metric=metric)


def _search(gpu, g, Q, k, ef, mode=-1, radius=None):
    gpu.set_option("hnsw.mode", mode)
    try:
        return g.search(Q, k, ef, radius=radius)
    finally:
        gpu.set_option("hnsw.mode", -1)


def _compare(out, ref, rtol=DIST_RTOL):
    gi, gd, gc, st = out
    oi, od, oc, ost = ref
    assert np.array_equal(gc, oc)
    assert recall(gi, oi) >= 0.999
    assert np.mean([set(a[:c]) == set(b[:c]) for a, b, c in zip(gi, oi, gc)]) >= 0.995
    # distances id by id: a near-tie that sends the traversal elsewhere shifts a whole list by a rank
    for q in range(len(gi)):
        go = {i: d for i, d in zip(gi[q, :gc[q]], gd[q, :gc[q]])}
        pairs = np.array([(go[i], d) for i, d in zip(oi[q, :oc[q]], od[q, :oc[q]]) if i in go]).reshape(-1, 2)
        assert np.allclose(pairs[:, 0], pairs[:, 1], rtol=rtol, atol=1e-6)
    assert np.all(np.isinf(gd[np.arange(gd.shape[1])[None, :] >= gc[:, None]]))
    assert abs(int(st.dist_evals) - int(ost[:, 0].sum())) <= 0.001 * ost[:, 0].sum()
    assert abs(int(st.nodes_expanded) - int(ost[:, 1].sum())) <= 0.001 * ost[:, 1].sum()


@pytest.mark.parametrize("dim", [2045, 2048, 2049, 2052])
def test_register_and_wide_kernel_boundary(gpu, dim):
    """2048 is the widest register query; 2049 and 2052 (ld 2052) are the first wide rows"""
    X, ix = _oracle_index(1500, dim, 8, 60, seed=dim)
    g = _stage(gpu, X, ix.levels(), gpu.L2, 8)
    Q = uniform_vectors(256, dim, dim + 1)
    ref = ix.search(Q, 10, 64, n_threads=8)
    outs = [_search(gpu, g, Q, 10, 64, mode) for mode in (0, 1, 2)]
    for out in outs:
        _compare(out, ref)
    for out in outs[1:]:  # one summation order in every mode: bit-identical answers
        assert np.array_equal(out[0], outs[0][0]) and np.array_equal(out[1].view(np.uint32), outs[0][1].view(np.uint32))


WIDTHS = [(O.L2, 3072, 0.0), (O.COSINE, 3072, 0.5), (O.IP, 3072, 0.5), (O.L2, 4096, 0.0), (O.COSINE, 4096, 0.5),
          (O.IP, 4096, 0.5)]


@pytest.mark.parametrize("metric,dim,shift", WIDTHS)
def test_metrics_and_widths(gpu, metric, dim, shift):
    ef = 48
    X, ix = _oracle_index(1500, dim, 8, 60, metric=metric, shift=shift, seed=dim + metric)
    g = _stage(gpu, X, ix.levels(), metric, 8)
    Q = uniform_vectors(128, dim, dim + 7) - np.float32(shift)
    full = ix.search(Q, ef, ef, n_threads=8)
    radius = float(np.median(full[1][:, 5])) if metric == O.L2 else None
    for mode in (0, 1, 2):
        for k in (1, 10, ef):
            _compare(_search(gpu, g, Q, k, ef, mode), ix.search(Q, k, ef, n_threads=8))
        if radius is not None:
            _compare(_search(gpu, g, Q, 10, ef, mode, radius), ix.search(Q, 10, ef, radius=radius, n_threads=8))


@pytest.mark.skipif(EMU, reason="8192-wide rows: minutes on the emulated library")
def test_l2_8192(gpu):
    X, ix = _oracle_index(1500, 8192, 8, 40, seed=8192)
    g = _stage(gpu, X, ix.levels(), gpu.L2, 8)
    Q = uniform_vectors(128, 8192, 8193)
    ref = ix.search(Q, 10, 40, n_threads=8)
    for mode in (0, 1, 2):
        _compare(_search(gpu, g, Q, 10, 40, mode), ref)


@pytest.fixture(scope="module")
def wide3072(gpu):
    X, ix = _oracle_index(2000, 3072, 8, 60, seed=3072)
    return X, ix, _stage(gpu, X, ix.levels(), gpu.L2, 8), uniform_vectors(128, 3072, 3073)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_filter_trims_after_the_mask(gpu, wide3072, mode):
    X, ix, g, Q = wide3072
    n = X.shape[0]
    rng = np.random.default_rng(5)
    gpu.set_option("hnsw.mode", mode)
    try:
        full_i, full_d, full_c, _ = g.search(Q, 64, 64)
        keep = rng.random(n) < 0.3
        ids, dist, cnt, _ = g.search(Q, 10, 64, row_pass=keep)
    finally:
        gpu.set_option("hnsw.mode", -1)
    for q in range(len(Q)):
        sel = [(i, d) for i, d in zip(full_i[q, :full_c[q]], full_d[q, :full_c[q]]) if keep[i]][:10]
        assert cnt[q] == len(sel)
        assert ids[q, :cnt[q]].tolist() == [i for i, _ in sel]
        assert dist[q, :cnt[q]].tolist() == [d for _, d in sel]


@pytest.mark.skipif(EMU, reason="needs torch CUDA tensors")
def test_search_dev_and_scatter(gpu, wide3072):
    import torch
    X, ix, g, Q = wide3072
    B, k, ef = Q.shape[0], 10, 64
    dq = torch.from_numpy(Q).cuda()
    stream = torch.cuda.current_stream().cuda_stream
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    g.search_dev(dq.data_ptr(), B, k, ef, ids.data_ptr(), dist.data_ptr(), qstats_ptr=qs.data_ptr(), stream=stream)
    sids = torch.empty((1, B, k), dtype=torch.int32, device="cuda")
    sdist = torch.empty((1, B, k), dtype=torch.float32, device="cuda")
    g.search_scatter_dev(dq.data_ptr(), B, k, ef, [sids.data_ptr()], [sdist.data_ptr()], 0, stream=stream)
    torch.cuda.synchronize()
    hi, hd, hc, hs = g.search(Q, k, ef)
    di = ids.cpu().numpy().view(np.uint32)
    assert np.array_equal(di, hi) and np.array_equal(dist.cpu().numpy(), hd)
    assert np.array_equal(sids[0].cpu().numpy().view(np.uint32), di)
    assert np.array_equal(sdist[0].cpu().numpy(), dist.cpu().numpy())
    st = qs.cpu().numpy().view(np.uint32)
    assert st[:, 0].sum() == hs.dist_evals


@pytest.mark.parametrize("dim", [3072, 4096])
def test_device_build(gpu, dim):
    n, m, efc = 2000, 8, 60
    X = uniform_vectors(n, dim, 9000 + dim)
    g = gpu.HnswIndex.build(X, m=m, ef_construction=efc, level_seed=SEED_LEVEL)
    (ni, rp, ci, ep), view = _view(g, X)
    deg0 = np.diff(rp[0].astype(np.int64))
    assert deg0.max() <= 2 * m and deg0.min() >= 1
    for L in range(1, len(rp)):
        assert np.diff(rp[L].astype(np.int64)).max() <= m
    Q = uniform_vectors(128, dim, 9001 + dim)
    out = g.search(Q, 10, 64)
    _compare(out, view.search(Q, 10, 64, n_threads=8))
    bi, _ = O.bruteforce_knn(X, Q, 10, n_threads=8)
    seq = O.OracleHnsw.new(n, dim, m=m, ef_construction=efc, level_seed=SEED_LEVEL)
    seq.insert_all(X)
    assert recall(out[0], bi) >= recall(seq.search(Q, 10, 64, n_threads=8)[0], bi) - 0.02


def test_device_build_cosine_keep_pruned(gpu):
    n, dim, m = 1500, 3072, 8
    X = uniform_vectors(n, dim, 9100) - np.float32(0.5)
    g = gpu.HnswIndex.build(X, metric=gpu.COSINE, m=m, ef_construction=60, keep_pruned_connections=True)
    (_, rp, _, _), view = _view(g, X, O.COSINE)
    deg0 = np.diff(rp[0].astype(np.int64))
    assert deg0.max() <= 2 * m and deg0.mean() > m
    Q = uniform_vectors(128, dim, 9101) - np.float32(0.5)
    _compare(g.search(Q, 10, 64), view.search(Q, 10, 64, n_threads=8))


def _check_dists(g, X):
    """stored edge distances == the oracle's f32 distances on the exported edges"""
    ni, rp, ci, ep = g.export_levels()
    ds = g.export_dists()
    X64 = X.astype(np.float64)
    for L in range(len(rp)):
        nodes = np.arange(rp[0].size - 1) if L == 0 else ni[L].astype(np.int64)
        src = np.repeat(nodes, np.diff(rp[L].astype(np.int64)))
        dst = ci[L].astype(np.int64)
        exp = ((X64[src] - X64[dst]) ** 2).sum(1)
        assert np.allclose(ds[L], exp, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("staged", [False, True])
def test_maintenance(gpu, staged):
    """insert, insert_at, update, remove and export_level_dist on a wide handle, device-built or staged from the
    oracle's graph (whose edge distances are derived on the first maintenance call)"""
    n0, c, dim, m, efc = 1500, 400, 3072, 8, 60
    X = uniform_vectors(n0 + c, dim, 9200 + staged)
    Q = uniform_vectors(128, dim, 9300)

    def make():
        if staged:
            ix = O.OracleHnsw.new(n0, dim, m=m, ef_construction=efc, level_seed=SEED_LEVEL)
            ix.insert_all(X[:n0])
            h = _stage(gpu, X[:n0], ix.levels(), gpu.L2, m)
            _check_dists(h, X[:n0])
            return h
        return gpu.HnswIndex.build(X[:n0], m=m, ef_construction=efc, level_seed=21)

    def check(h, Xh):
        _, view = _view(h, Xh)
        _compare(h.search(Q, 10, 64), view.search(Q, 10, 64, n_threads=8))
        _check_dists(h, Xh)

    a, b = make(), make()
    b.insert(X[n0:], ef_construction=efc, keep_pruned_connections=0)
    check(b, X)
    # insert_at at random positions == insert read through the relabelling
    rng = np.random.default_rng(9)
    ni, rp, cib, ep = b.export_levels()
    lv_new = np.zeros(n0 + c, np.int64)
    for L in range(1, len(rp)):
        lv_new[ni[L]] = L
    lv_new = lv_new[n0:]
    P = np.sort(rng.integers(0, n0 + 1, c))
    P[(lv_new == len(rp) - 1) & (P <= ep)] = ep + 1
    P = np.maximum.accumulate(P).astype(np.uint32)
    ids = a.insert_at(P, X[n0:], ef_construction=efc, keep_pruned_connections=0)
    old = np.arange(n0) + np.searchsorted(P.astype(np.int64), np.arange(n0), side="right")
    pi = np.concatenate([old, P.astype(np.int64) + np.arange(c)])
    assert np.array_equal(ids, pi[n0:])
    (nia, rpa, cia, epa), _ = _view(a, X[np.argsort(pi)])
    assert epa == pi[ep]
    for L in range(len(rp)):
        srcb = np.repeat(np.arange(n0 + c) if L == 0 else ni[L].astype(np.int64), np.diff(rp[L].astype(np.int64)))
        srca = np.repeat(np.arange(n0 + c) if L == 0 else nia[L].astype(np.int64), np.diff(rpa[L].astype(np.int64)))
        eb = sorted(zip(pi[srcb].tolist(), pi[cib[L].astype(np.int64)].tolist()))
        ea = sorted(zip(srca.tolist(), cia[L].astype(np.int64).tolist()))
        assert ea == eb
    check(a, X[np.argsort(pi)])
    # update changed vectors, then remove
    upd = np.arange(100, 700, 3, dtype=np.uint32)
    newv = uniform_vectors(upd.size, dim, 9400)
    b.update(upd, newv)
    X2 = X.copy()
    X2[upd] = newv
    check(b, X2)
    dead = rng.choice(n0 + c, 300, replace=False).astype(np.uint32)
    b.remove(dead)
    (_, _, ci2, _), view = _view(b, X2)
    assert not any(np.isin(x, dead).any() for x in ci2)
    out = b.search(Q, 10, 64)
    assert not np.isin(out[0], dead).any()
    _compare(out, view.search(Q, 10, 64, n_threads=8))
    _check_dists(b, X2)


def test_envelope(gpu):
    """a width whose query and one ring stage exceed the shared-memory opt-in is refused, with its size in the message"""
    dim = 40000
    X = uniform_vectors(24, dim, 9500)
    for mode in (-1, 1, 2):
        ix = O.OracleHnsw.new(16, dim, m=4, ef_construction=10)
        ix.insert_all(X[:16])
        g = _stage(gpu, X[:16], ix.levels(), gpu.L2, 4)
        gpu.set_option("hnsw.mode", mode)
        try:
            with pytest.raises(gpu.CozoGpuError) as e:
                g.search(X[:2], 3, 10)
        finally:
            gpu.set_option("hnsw.mode", -1)
        assert e.value.code == gpu.E_UNSUP and "vec_dim 40000" in str(e.value) and "ef=10" in str(e.value)
    # mode 0 holds the query but no ring: it answers at this width
    ref = ix.search(X[:2], 3, 10)
    out = _search(gpu, g, X[:2], 3, 10, 0)
    assert np.array_equal(out[0], ref[0]) and np.array_equal(out[2], ref[2])
    with pytest.raises(gpu.CozoGpuError) as e:
        gpu.HnswIndex.build(X, m=4, ef_construction=10)
    assert e.value.code == gpu.E_UNSUP and "vec_dim 40000" in str(e.value)
    before = g.export_levels()
    with pytest.raises(gpu.CozoGpuError) as e:
        g.insert(X[16:], ef_construction=10, keep_pruned_connections=0)
    assert e.value.code == gpu.E_UNSUP
    after = g.export_levels()
    assert g.info()[0] == 16
    for x, y in zip(before[1] + before[2], after[1] + after[2]):
        assert np.array_equal(x, y)
    assert before[3] == after[3]
    out = _search(gpu, g, X[:2], 3, 10, 0)                  # a later valid call still works
    assert np.array_equal(out[0], ref[0])


def test_default_mode_takes_the_warp_kernel_where_the_cooperative_one_does_not_fit(gpu):
    """At 16384 elements the cooperative CTA (query + a ring stage per warp) exceeds the opt-in, the warp-per-query kernel
    (query + one stage) does not: small batches in the default mode run on the latter."""
    dim = 16384
    X, ix = _oracle_index(400, dim, 4, 20, seed=dim)
    g = _stage(gpu, X, ix.levels(), gpu.L2, 4)
    Q = uniform_vectors(2, dim, dim + 1)
    for B in (1, 2):
        out = g.search(Q[:B], 5, 20)
        ref = ix.search(Q[:B], 5, 20)
        assert np.array_equal(out[0], ref[0]) and np.array_equal(out[2], ref[2])
        assert np.allclose(out[1], ref[1], rtol=DIST_RTOL)
        assert np.array_equal(out[0], _search(gpu, g, Q[:B], 5, 20, 1)[0])
    with pytest.raises(gpu.CozoGpuError) as e:          # the cooperative kernel itself, asked for explicitly
        _search(gpu, g, Q[:1], 5, 20, 2)
    assert e.value.code == gpu.E_UNSUP and "vec_dim 16384" in str(e.value)


@pytest.mark.skipif(EMU, reason="reads device memory through torch")
def test_wide_l2_index_reserves_no_code_rows(gpu):
    """Code rows are reserved for L2 indexes with 512 <= ld <= 2048 only: staging the same rows as L2 and as IP (never
    coded) takes the same device memory at ld 3072, and one code row per vector more at ld 2048."""
    import torch
    n = 40000

    def staged_bytes(dim, metric):
        X = np.random.default_rng(dim).random((n, dim), dtype=np.float32)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        g = gpu.HnswIndex.stage(X, [None], [np.zeros(n + 1, np.uint64)], [np.zeros(0, np.uint32)], 0, metric=metric,
                                m_max0=8, m_max=4)
        used = free0 - torch.cuda.mem_get_info()[0]
        g.close()
        return used

    for dim in (2048, 3072):
        code_bytes = n * (16 + (dim + 15) // 16 * 16)
        extra = staged_bytes(dim, gpu.L2) - staged_bytes(dim, gpu.IP)
        if dim <= 2048:
            assert extra >= code_bytes // 2, extra             # the measurement sees code rows where they exist
        else:
            assert extra < code_bytes // 2, extra


def test_host_layer_3072(gpu):
    """HnswSearchRA::iter and the index relation write-back through the C++ host mirror with a 3072-element column"""
    from tests.hostmod import load
    from tests.test_host_gpu import _index_relation
    h = load()
    h.init(0)
    n, dim, m = 1500, 3072, 8
    X = uniform_vectors(n, dim, 9600)
    ix = O.OracleHnsw.new(n, dim, m=m, ef_construction=50)
    ix.insert_all(X)
    base = h.Relation("a", ["k"], ["v"])
    names = [f"key{i:05d}" for i in range(n)]
    for i in range(n):
        base.put([names[i], X[i]])
    index = h.HnswIndex()
    index.stage(base, _index_relation(ix, lambda i: [names[i]], 1), {"dim": dim, "m": m, "ef_construction": 50,
                                                                     "fields": [1]})
    Q = uniform_vectors(40, dim, 9601)
    out = h.HnswSearchRA(base, index, k=5, ef=40, bind_distance=True, bind_idx=1).iter([[qi, Q[qi]] for qi in range(40)])
    oi, od, oc, _ = ix.search(Q, 5, 40)
    assert len(out) == 40 * 5
    for qi in range(40):
        rows = [r for r in out if r[0] == qi]
        assert [r[2] for r in rows] == [names[j] for j in oi[qi]]
        assert np.allclose([r[4] for r in rows], od[qi], rtol=1e-5)
    # create_hnsw_index on the device, written back as rows of `rel:idx` and re-staged: the same answers
    mf = {"dim": dim, "m": m, "ef_construction": 40, "fields": [1]}
    built = h.HnswIndex()
    built.build(base, mf)
    rows = built.to_index_rows(base)
    assert len([r for r in rows if r[0] == 0 and r[1:4] == r[4:7]]) == n   # one self loop per vector on layer 0
    restaged = h.HnswIndex()
    restaged.stage(base, rows, mf)
    parent = [[q] for q in Q]
    a = h.HnswSearchRA(base, built, k=5, ef=40, bind_distance=True, bind_idx=0).iter(parent)
    b = h.HnswSearchRA(base, restaged, k=5, ef=40, bind_distance=True, bind_idx=0).iter(parent)
    assert [(r[1], r[3]) for r in a] == [(r[1], r[3]) for r in b] and len(a) == 200
