"""The pruned search on Cosine and IP indexes (code_dot_prunes in hnsw_codes.cuh: an upper bound on the kernel's f32 dot
product from the uint8 code row) against the ld.global search (hnsw.mode=0), which never prunes.  Ids, distance bits,
result counts and the three traversal counters must be equal; the fourth qstats word (f32 rows fetched) shows how many
rows were skipped.  Covered: built indexes at D = 516, 768 and 2048; U[0,1), U[0,1) + 1000 (the bound is loose there but
must stay valid) and normalised Gaussian data; rows that are zero or hold NaN; a staged index; the index after insert,
insert_at, update and remove + compact; filtered and radius searches; the sharded operator at world 1.  Rejection-rate
floors were set from the first H100 run (the rates it measured: profiles/h100_pytest_gpu_prune_metric.txt).  The code
rows of a Cosine or IP index are made by its first search; every index here is built or staged without them."""
import os

import numpy as np
import pytest

from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu
METRICS = [1, 2]  # COSINE, IP


def _gauss(n, dim, seed):
    x = np.random.default_rng(seed).standard_normal((n, dim))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _data(kind, n, dim, seed):
    if kind == "u01":
        return uniform_vectors(n, dim, seed)
    if kind == "u01+1000":
        return uniform_vectors(n, dim, seed) + np.float32(1000.0)
    return _gauss(n, dim, seed)


# COZO_EMU_LIB (tests/conftest.py): the CPU-emulated library, whose device memory is host memory: buffers are numpy arrays,
# and corpora and batches are 10x smaller (equality is checked there, the rejection-rate floors only on the GPU)
EMU = bool(os.environ.get("COZO_EMU_LIB"))
S = 10 if EMU else 1


def _buf(a):
    """a device copy of the numpy array a -> (buffer, pointer)"""
    a = np.ascontiguousarray(a)
    if EMU:
        a = a.copy()
        return a, a.ctypes.data
    import torch
    signed = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype)
    t = torch.from_numpy(a.view(signed) if signed else a).cuda()
    return t, t.data_ptr()


def _host(b):
    return b if EMU else b.cpu().numpy()


def _search(gpu, g, Q, k, ef, mode, radius=None, mask=None, grp=None):
    """one device search with per-query stats; mask: bool[n] filter verdicts; grp: the world-1 sharded operator"""
    B = Q.shape[0]
    dq, qp = _buf(Q)
    ids, ip = _buf(np.zeros((B, k), np.uint64 if grp else np.uint32))
    dist, dp = _buf(np.zeros((B, k), np.float32))
    cnt, cp = _buf(np.zeros(B, np.uint32))
    qs, sp = _buf(np.zeros((B, 4), np.uint32))
    dm, mp = _buf(gpu.pack_row_mask(mask)) if mask is not None else (None, None)
    r = -1.0 if radius is None else float(radius)
    stream = None
    if not EMU:
        import torch
        stream = torch.cuda.current_stream().cuda_stream
    L = gpu.load()
    gpu.set_option("hnsw.mode", mode)
    try:
        if grp is not None:
            grp.search_dev(qp, B, k, ef, ip, dp, qstats_ptr=sp, stream=stream, radius=radius, row_mask_ptr=mp)
        elif mask is None:
            gpu._check(L.cozo_gpu_hnsw_search_dev(g._h, qp, B, k, ef, r, ip, dp, cp, sp, stream))
        else:
            gpu._check(L.cozo_gpu_hnsw_search_filtered_dev(g._h, qp, B, k, ef, r, mp, ip, dp, cp, sp, stream))
        if not EMU:
            torch.cuda.synchronize()
    finally:
        gpu.set_option("hnsw.mode", -1)
    return _host(ids), _host(dist), _host(cnt), _host(qs)


def _check(gpu, g, Q, k, ef, **kw):
    """pruned (warp per query + bulk ring) == unpruned (ld.global); returns the share of evaluations not fetched"""
    i1, d1, c1, s1 = _search(gpu, g, Q, k, ef, 1, **kw)
    i0, d0, c0, s0 = _search(gpu, g, Q, k, ef, 0, **kw)
    assert np.array_equal(i1, i0)
    assert np.array_equal(d1.view(np.uint32), d0.view(np.uint32))
    assert np.array_equal(c1, c0)
    assert np.array_equal(s1[:, :3], s0[:, :3])
    assert np.array_equal(s0[:, 3], s0[:, 0])
    assert np.all(s1[:, 3] <= s1[:, 0])
    fetched, evals = int(s1[:, 3].astype(np.int64).sum()), int(s1[:, 0].astype(np.int64).sum())
    return 1.0 - fetched / evals


def _floor(rate, floor):
    if not EMU:
        assert rate > floor, f"rejection rate {rate}"


# data kind -> rejection floor at D = 768, ef 128 (first H100 run: Cosine 0.794 / IP 0.780 on U[0,1), 0.821 / 0.821 on
# normalised Gaussian data); the offset data has no floor: there the bound never pruned (0.000 for both metrics)
FLOORS = {"u01": 0.7, "gauss": 0.75, "u01+1000": None}


@pytest.fixture(scope="module")
def built768(gpu):
    out = {}
    for metric in METRICS:
        for kind in FLOORS:
            X = _data(kind, 20000 // S, 768, 5100 + metric)
            out[metric, kind] = X, gpu.HnswIndex.build(X, metric=metric, m=16, ef_construction=100, level_seed=31)
    return out


@pytest.mark.parametrize("kind", list(FLOORS))
@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_equals_unpruned(gpu, built768, metric, kind):
    X, g = built768[metric, kind]
    rate = _check(gpu, g, _data(kind, 1200 // S, 768, 5200 + metric), 10, 128)
    print(f"metric {metric} {kind}: rejection rate {rate:.3f}")
    if FLOORS[kind] is not None:
        _floor(rate, FLOORS[kind])


@pytest.mark.parametrize("dim", [516, 2048])
@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_row_lengths(gpu, metric, dim):
    X = _gauss(8000 // S, dim, 5300 + dim)
    g = gpu.HnswIndex.build(X, metric=metric, m=16, ef_construction=100, level_seed=32)
    rate = _check(gpu, g, _gauss(1000 // S, dim, 5400 + dim), 10, 128)
    print(f"metric {metric} dim {dim}: rejection rate {rate:.3f}")
    _floor(rate, 0.7)  # first H100 run: 0.809 at D = 516, 0.763 at D = 2048, both metrics


@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_zero_and_nan_rows(gpu, metric):
    """zero rows (Cosine: NaN distance) and rows holding NaN carry err = +inf and are never pruned.  A NaN at the end of a
    full beam (NaN sorts last) admits nothing and prunes nothing, so the rate is low (first H100 run: Cosine 0.033)."""
    X = uniform_vectors(8000 // S, 768, 5500) - np.float32(0.3)
    X[::97] = 0.0
    X[5::89, 100] = np.nan
    g = gpu.HnswIndex.build(X, metric=metric, m=16, ef_construction=100, level_seed=33)
    rate = _check(gpu, g, uniform_vectors(1000 // S, 768, 5501) - np.float32(0.3), 10, 128)
    print(f"metric {metric} zero and NaN rows: rejection rate {rate:.3f}")
    _floor(rate, 0.01)


@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_staged(gpu, built768, metric):
    """an index staged from its layers (not built) gets its code rows when it is staged"""
    X, g = built768[metric, "gauss"]
    s = gpu.HnswIndex.stage(X, *g.export_levels(), metric=metric, m_max0=32, m_max=16)
    Q = _data("gauss", 1000 // S, 768, 5600)
    rate = _check(gpu, s, Q, 10, 128)
    print(f"metric {metric} staged: rejection rate {rate:.3f}")
    _floor(rate, 0.5)
    assert np.array_equal(_search(gpu, s, Q, 10, 128, 1)[0], _search(gpu, g, Q, 10, 128, 1)[0])


@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_after_writes(gpu, metric):
    """the code rows follow every write of the vectors, in the index's metric: insert, insert_at, update, compact"""
    D, n = 768, 5000 // S
    X = _gauss(n + n * 3 // 10, D, 5700)
    g = gpu.HnswIndex.build(X[:n], metric=metric, m=12, ef_construction=80, level_seed=34)
    Q = _gauss(1000 // S, D, 5701)
    g.insert(X[n:n + n // 5])
    _check(gpu, g, Q, 10, 96)
    n1 = n + n // 5
    pos = np.sort(np.random.default_rng(5702).integers(0, n1, n // 10)).astype(np.uint32)
    g.insert_at(pos, X[n1:n1 + n // 10])
    _check(gpu, g, Q, 10, 96)
    n2 = n1 + n // 10
    g.update(np.arange(1, n2, 7, dtype=np.uint32), _gauss(len(range(1, n2, 7)), D, 5703))
    _check(gpu, g, Q, 10, 96)
    g.remove(np.arange(0, n2, 5, dtype=np.uint32))
    g.compact()
    assert g.info()[0] == n2 - len(range(0, n2, 5))
    rate = _check(gpu, g, Q, 10, 96)
    print(f"metric {metric} after writes: rejection rate {rate:.3f}")
    _floor(rate, 0.1)


@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_filtered_and_radius(gpu, built768, metric):
    X, g = built768[metric, "u01"]
    Q = _data("u01", 1000 // S, 768, 5800)
    keep = np.random.default_rng(5801).random(X.shape[0]) < 0.5
    _check(gpu, g, Q, 10, 128, mask=keep)
    d = _search(gpu, g, Q, 10, 128, 0)[1]
    r = float(np.median(d[:, 4]))
    _check(gpu, g, Q, 10, 128, radius=r)
    _check(gpu, g, Q, 10, 128, radius=r, mask=keep)


@pytest.mark.parametrize("metric", METRICS)
def test_metric_pruned_search_sharded_world1(gpu, built768, metric):
    if not EMU:
        import torch  # noqa: F401  (maps the libnccl the communicator resolves)
    X, g = built768[metric, "gauss"]
    grp = gpu.ShardGroup(gpu.ShardGroup.unique_id(), 0, 1)
    try:
        grp.attach(g)
        Q = _data("gauss", 1000 // S, 768, 5900)
        keep = np.random.default_rng(5901).random(X.shape[0]) < 0.7
        rate = _check(gpu, g, Q, 10, 128, grp=grp)
        print(f"metric {metric} sharded: rejection rate {rate:.3f}")
        _floor(rate, 0.5)
        _check(gpu, g, Q, 10, 128, grp=grp, mask=keep)
    finally:
        grp.close()


@pytest.mark.parametrize("metric", METRICS)
def test_metric_code_rows_made_by_the_first_search(gpu, built768, metric):
    """A Cosine or IP index gets its code rows from its first search, whichever kernel that search runs (here the
    cooperative one, which does not prune), and every later warp-per-query search prunes."""
    X, g = built768[metric, "gauss"]
    s = gpu.HnswIndex.stage(X, *g.export_levels(), metric=metric, m_max0=32, m_max=16)
    Q = _data("gauss", 1000 // S, 768, 6000)
    first = _search(gpu, s, Q[:8], 10, 128, 2)
    assert np.array_equal(first[3][:, 3], first[3][:, 0])
    rate = _check(gpu, s, Q, 10, 128)
    print(f"metric {metric} after a cooperative first search: rejection rate {rate:.3f}")
    _floor(rate, 0.5)
