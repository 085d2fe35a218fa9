"""The pruned L2 search's per-warp stream (prune_chunk in hnsw_device.cuh) on cases test_hnsw_prune_gpu.py does not reach:
adjacency rows of several 32-id chunks (m 48), a corpus with 30 % duplicate rows (many visited neighbours among the code
rows fetched before the visited test), and the largest ef the shared memory allows.  Each is compared bit for bit
against the ld.global search (hnsw.mode=0), which never prunes."""
import numpy as np
import pytest

from tests.test_hnsw_prune_gpu import _check_equal, _search
from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu


def test_pruned_stream_m48_three_chunks(gpu):
    X = uniform_vectors(20000, 768, 4801)
    g = gpu.HnswIndex.build(X, m=48, ef_construction=120, level_seed=11)
    rate = _check_equal(gpu, g, uniform_vectors(1000, 768, 4802), 10, 128)
    assert rate > 0.3, f"rejection rate {rate}"


def test_pruned_stream_duplicate_rows(gpu):
    X = uniform_vectors(20000, 768, 3001)
    rng = np.random.default_rng(3002)
    d = rng.choice(len(X), int(0.3 * len(X)), replace=False)
    X[d] = X[rng.integers(0, len(X), len(d))]
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=12)
    Q = uniform_vectors(1000, 768, 3003)
    Q[:250] = X[rng.integers(0, len(X), 250)]  # queries on (duplicated) rows: ties at distance 0
    for ef in (16, 200):
        _check_equal(gpu, g, Q, 10, ef)


def test_pruned_stream_largest_ef(gpu):
    # the largest ef the warp-per-query kernel can hold in shared memory at D = 768, found on a tiny index
    small = gpu.HnswIndex.build(uniform_vectors(300, 768, 5001), m=8, ef_construction=32, level_seed=13)
    q1 = uniform_vectors(1, 768, 5002)
    lo, hi = 64, 1 << 16  # lo fits, hi does not
    while hi - lo > 1:
        mid = (lo + hi) // 2
        try:
            _search(gpu, small, q1, 1, mid, 1)
            lo = mid
        except gpu.CozoGpuError as e:
            assert e.code == gpu.E_UNSUP
            hi = mid
    assert lo > 10000, lo
    X = uniform_vectors(40000, 768, 5003)
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=14)
    _check_equal(gpu, g, uniform_vectors(64, 768, 5004), 10, lo)
