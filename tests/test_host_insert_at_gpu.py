"""The host mirror's `insert_inside` policy: a `:put` whose new compound keys land inside the indexed key range goes to
cozo_gpu_hnsw_insert_at instead of re-indexing the base relation, and the key dictionary (`keys`, `key_ids`, `live`)
follows the device's relabelling, including rows whose list-of-vectors column gives several consecutive compound keys."""
import numpy as np
import pytest

from tests.hostmod import load
from tests.util import uniform_vectors

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def h(gpu):
    m = load()
    m.init(0)
    return m


def test_put_inside_the_key_range_inserts_in_place(h):
    n, dim, m = 600, 24, 8
    X = uniform_vectors(n + 100, dim, 81)
    mf = {"dim": dim, "m": m, "ef_construction": 60, "fields": [1, 2]}
    name = lambda i: f"key{i:05d}"                                   # noqa: E731
    base = h.Relation("a", ["k"], ["v", "chunks"])
    for i in range(n):
        base.put([name(2 * i), X[i], []])                           # even keys; the inserted keys are odd
    index = h.HnswIndex()
    index.build(base, mf)
    assert index.insert_inside is False
    index.insert_inside = True
    gone = [name(2 * i) for i in range(10, 20)]
    index.remove_rows(base, [[k] for k in gone])                    # removed ids keep their ids and keys

    def top1(vectors):
        out = h.HnswSearchRA(base, index, k=1, ef=80, bind_distance=True, bind_idx=0).iter([[v] for v in vectors])
        return [(r[1], r[4]) for r in out]

    inside = [1, 7, 7 * 2 + 1, 401, 2 * n - 3]
    rows = [[name(k), X[n + j], []] for j, k in enumerate(inside)]
    rows.append([name(99), X[n + 10], [X[n + 11], X[n + 12]]])      # one row, three compound keys
    rows.append([name(2 * n + 1), X[n + 13], []])                   # after every key
    index.put_rows(base, rows)
    info = index.info()
    assert info["rebuilt"] == 0 and info["put_inserted"] == len(inside) + 3 + 1 and info["put_appended"] == 0
    assert info["n_vectors"] == n + len(inside) + 4
    want = [name(k) for k in inside] + [name(99)] * 3 + [name(2 * n + 1)]
    got = top1(np.concatenate([X[n:n + len(inside)], X[n + 10:n + 14]]))
    assert [k for k, _ in got] == want and all(d == 0.0 for _, d in got)
    old = [i for i in range(0, n, 7) if not 10 <= i < 20]
    hits = top1(X[old])
    assert sum(k == name(2 * i) and d == 0.0 for i, (k, d) in zip(old, hits)) >= 0.95 * len(old)
    found = {r[1] for r in h.HnswSearchRA(base, index, k=10, ef=80, bind_idx=0).iter([[v] for v in X[10:20]])}
    assert not (found & set(gone))
    # the dictionary follows the relabelling: a changed vector under a moved key updates that key's row
    index.put_rows(base, [[name(2 * 500), X[n + 20], []]])
    assert index.info()["put_updated"] == 1
    assert top1(X[n + 20:n + 21])[0] == (name(2 * 500), 0.0)
    # write-back as rows of `rel:idx`, re-stage from them: same answers
    fresh = h.HnswIndex()
    fresh.stage(base, index.to_index_rows(base), mf)
    Q = uniform_vectors(60, dim, 82)
    a = h.HnswSearchRA(base, index, k=5, ef=40, bind_distance=True, bind_idx=0).iter([[q] for q in Q])
    b = h.HnswSearchRA(base, fresh, k=5, ef=40, bind_distance=True, bind_idx=0).iter([[q] for q in Q])
    assert [(r[1], r[4]) for r in a] == [(r[1], r[4]) for r in b] and len(a) == 300
