"""The visited bitmap of a warp is cleared at the end of every layer (visit_clear in hnsw_device.cuh): by its log of set
ids, one atomic per id, when the layer set fewer than one id per VISIT_SWEEP_WORDS words, and otherwise by sweeping the
whole bitmap.  A bit left behind would make a later query served by the same warp skip that row, so a batch in which
every warp serves several queries must return exactly what the same queries return in small batches, where every warp
serves at most one.  Two indexes put layer 0 on either side of the threshold: 60 k rows at D = 512 (codes, the pruned
search; layer 0 sets thousands of ids in a 1 876-word bitmap: swept) and 1 M rows at D = 8, ef 10 (far fewer ids than
31 252 / 32 words: cleared by the log); the traversal counters confirm which side each run is on."""
import numpy as np
import pytest

from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu


def _search(gpu, g, Q, k, ef, mode, chunk, ctas_per_sm):
    gpu.set_option("hnsw.mode", mode)
    gpu.set_option("hnsw.max_ctas_per_sm", ctas_per_sm)
    try:
        ids, dist, evals, expanded = [], [], 0, 0
        for s in range(0, Q.shape[0], chunk):
            i, d, _, st = g.search(Q[s:s + chunk], k, ef)
            ids.append(i)
            dist.append(d)
            evals += st.dist_evals
            expanded += st.nodes_expanded
    finally:
        gpu.set_option("hnsw.mode", -1)
        gpu.set_option("hnsw.max_ctas_per_sm", 0)
    return np.concatenate(ids), np.concatenate(dist), evals, expanded


@pytest.fixture(scope="module")
def swept(gpu):
    return gpu.HnswIndex.build(uniform_vectors(60000, 512, 71), m=16, ef_construction=100, level_seed=3)


@pytest.fixture(scope="module")
def logged(gpu):
    return gpu.HnswIndex.build(uniform_vectors(1_000_000, 8, 72), m=16, ef_construction=64, level_seed=4)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("which,n,dim,ef", [("swept", 60000, 512, 64), ("swept", 60000, 512, 200),
                                            ("logged", 1_000_000, 8, 10)])
def test_reused_warps_return_what_fresh_warps_return(gpu, request, mode, which, n, dim, ef):
    g = request.getfixturevalue(which)
    Q = uniform_vectors(3000, dim, 73)
    threshold = (n + 31) // 32 / 32  # layer-0 ids below which the log clears the bitmap
    fresh = _search(gpu, g, Q, 10, ef, mode, 32, 0)     # at most one query per warp (per CTA in mode 2)
    reused = _search(gpu, g, Q, 10, ef, mode, 3000, 1)  # one CTA per SM: every warp serves several queries
    assert np.array_equal(fresh[0], reused[0])
    assert np.array_equal(fresh[1].view(np.uint32), reused[1].view(np.uint32))
    assert fresh[2:] == reused[2:]
    evals_per_query = fresh[2] / Q.shape[0]
    if which == "swept":
        assert evals_per_query > 4 * threshold
    else:
        assert evals_per_query + ef < threshold / 2
