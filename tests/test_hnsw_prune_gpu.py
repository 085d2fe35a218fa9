"""The pruned L2 search (hnsw_codes.cuh, code_prune in hnsw_device.cuh) against the ld.global search (hnsw.mode=0),
which never prunes: with a full beam most neighbours are rejected from their uint8 code rows alone, and that must change
nothing.  Ids, distances and the three traversal counters are compared for equality, not closeness; the fourth qstats
word (f32 rows fetched) must show that rows were actually skipped."""
import numpy as np
import pytest

from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu


def _search(gpu, g, Q, k, ef, mode):
    import torch
    B = Q.shape[0]
    dq = torch.from_numpy(Q).cuda()
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    gpu.set_option("hnsw.mode", mode)
    try:
        stream = torch.cuda.current_stream().cuda_stream
        g.search_dev(dq.data_ptr(), B, k, ef, ids.data_ptr(), dist.data_ptr(), qstats_ptr=qs.data_ptr(), stream=stream)
        torch.cuda.synchronize()
    finally:
        gpu.set_option("hnsw.mode", -1)
    return ids.cpu().numpy(), dist.cpu().numpy(), qs.cpu().numpy().view(np.uint32)


def _check_equal(gpu, g, Q, k, ef):
    i1, d1, s1 = _search(gpu, g, Q, k, ef, 1)   # warp per query + TMA ring: pruned
    i0, d0, s0 = _search(gpu, g, Q, k, ef, 0)   # ld.global rows: every row fetched
    assert np.array_equal(i1, i0)
    assert np.array_equal(d1.view(np.uint32), d0.view(np.uint32))
    assert np.array_equal(s1[:, :3], s0[:, :3])
    assert np.array_equal(s0[:, 3], s0[:, 0])
    fetched, evals = int(s1[:, 3].astype(np.int64).sum()), int(s1[:, 0].astype(np.int64).sum())
    assert fetched < evals
    assert np.all(s1[:, 3] <= s1[:, 0])
    return 1.0 - fetched / evals


@pytest.fixture(scope="module")
def built(gpu):
    X = uniform_vectors(50000, 768, 4242)
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=7)
    return X, g


@pytest.mark.parametrize("ef", [64, 200])
def test_pruned_search_equals_unpruned(gpu, built, ef):
    X, g = built
    Q = uniform_vectors(1500, 768, 4343)
    rate = _check_equal(gpu, g, Q, 10, ef)
    assert rate > 0.3, f"rejection rate {rate}"


def test_pruned_search_after_update_and_insert(gpu):
    """the code rows follow every write of the vectors: insert (grows the arrays) and update (rewrites rows)"""
    D = 514  # the f32 row (ld 516) and the code row (528 codes) both carry padding
    X = uniform_vectors(6000, D, 515)
    g = gpu.HnswIndex.build(X[:4000], m=12, ef_construction=80, level_seed=3)
    g.insert(X[4000:])
    ids = np.arange(100, 6000, 7, dtype=np.uint32)
    g.update(ids, uniform_vectors(len(ids), D, 616) * np.float32(0.5))
    Q = uniform_vectors(1000, D, 717)
    _check_equal(gpu, g, Q, 10, 96)
    # the updated rows are found where they now are
    i1, d1, _ = _search(gpu, g, uniform_vectors(len(ids), D, 616)[:50] * np.float32(0.5), 1, 64, 1)
    assert np.mean(i1[:, 0].view(np.uint32) == ids[:50]) >= 0.9
