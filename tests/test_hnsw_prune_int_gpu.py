"""The pruned L2 search with the integer code-row bound (code_idot2 / code_int_prunes: an exact int32 product of the
uint8 code row with a fixed-point copy of the query) against the ld.global search (hnsw.mode=0), which never prunes.
Covered beyond test_hnsw_prune_gpu.py: data whose offset dwarfs its spread (U[0,1) + 1000, where the bound is loose but
must stay valid), and rows of 516 and 2048 elements (the smallest padded row with codes, and the largest row)."""
import numpy as np
import pytest

from tests.test_hnsw_prune_gpu import _check_equal
from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu


def test_int_pruned_search_offset_data(gpu):
    X = uniform_vectors(20000, 768, 9101) + np.float32(1000.0)
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=21)
    Q = uniform_vectors(1000, 768, 9102) + np.float32(1000.0)
    _check_equal(gpu, g, Q, 10, 128)


@pytest.mark.parametrize("dim", [516, 2048])
def test_int_pruned_search_row_lengths(gpu, dim):
    X = uniform_vectors(12000, dim, 9200 + dim)
    g = gpu.HnswIndex.build(X, m=16, ef_construction=100, level_seed=22)
    rate = _check_equal(gpu, g, uniform_vectors(800, dim, 9300 + dim), 10, 128)
    assert rate > 0.3, f"rejection rate {rate}"
