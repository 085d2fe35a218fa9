"""Tiny end-to-end exercise of every kernel for compute-sanitizer (memcheck / racecheck / initcheck)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cozo_b200 import capi  # noqa: E402

capi.init(0)
rng = np.random.default_rng(0)
for dim, metric in [(64, capi.L2), (100, capi.COSINE)]:
    X = rng.random((1500, dim), dtype=np.float32) - 0.5
    g = capi.HnswIndex.build(X, metric=metric, m=8, ef_construction=40, keep_pruned_connections=(metric == capi.COSINE))
    Q = rng.random((64, dim), dtype=np.float32) - 0.5
    for mode in (1, 0, 2):                        # TMA ring, ld.global.nc, cooperative CTA-per-query
        capi.set_option("hnsw.mode", mode)
        ids, dist, cnt, st = g.search(Q, 5, 40)
        assert (cnt == 5).all()
    capi.set_option("hnsw.mode", -1)
    ni, rp, ci, ep = g.export_levels()
    g2 = capi.HnswIndex.stage(X, ni, rp, ci, ep, metric=metric, m_max0=16, m_max=8)
    ids2, _, _, _ = g2.search(Q, 5, 40, radius=float(np.median(dist)))
    # maintenance: append, change vectors under existing ids (non-tail ranges), remove, search again
    first = g.insert(rng.random((200, dim), dtype=np.float32) - 0.5)
    assert first == 1500
    g.update(np.array([3, 4, 5, 900, 1699], np.uint32), rng.random((5, dim), dtype=np.float32) - 0.5)
    g.remove(np.arange(100, 160, dtype=np.uint32))
    ids3, _, cnt3, _ = g.search(Q, 5, 40)
    assert (cnt3 == 5).all() and not np.isin(ids3, np.arange(100, 160)).any()
    # rows inside the key range (front, middle, end), then the removed rows dropped: both relabellings
    for pos in (0, 850, g.info()[0]):
        g.insert_at(np.full(3, pos, np.uint32), rng.random((3, dim), dtype=np.float32) - 0.5)
    g.remove(np.arange(400, 420, dtype=np.uint32))
    g.compact()
    assert (g.search(Q, 5, 40)[2] == 5).all()
    g.export_levels(); g.export_dists(); g.export_live()
src = rng.integers(0, 300, 3000).astype(np.uint32)
dst = rng.integers(0, 300, 3000).astype(np.uint32)
w = (rng.random(3000) + 0.1).astype(np.float32)
gg = capi.Graph(300, src, dst, w)
gg.pagerank(0.85, 1e-4, 5)
gg.sssp(np.arange(0, 300, 50, dtype=np.uint32))
gg.closeness()
gg.betweenness()
gg.clustering()
gg.sssp_paths(np.array([0, 5], np.uint32), np.array([7, 9], np.uint32), forb_nodes=[[3], []], forb_edges=[[], [(5, 9)]])
# PageRank work items of every kind: a hub row (> 4096 in-edges), a medium row (257..4096), mini-blocks
hsrc = np.concatenate([np.arange(1, 6000), np.arange(2, 900), rng.integers(0, 6000, 4000)]).astype(np.uint32)
hdst = np.concatenate([np.zeros(5999), np.ones(898), rng.integers(0, 6000, 4000)]).astype(np.uint32)
hub = capi.Graph(6000, hsrc, hdst)
capi.set_option("pagerank.mode", 0)                     # round-1 gather pull
for warps in (32, 8):
    capi.set_option("pagerank.warps", warps)
    for dyn in (1, 0):
        capi.set_option("pagerank.dynamic", dyn)
        hub.pagerank(0.85, 0.0, 2)
capi.set_option("pagerank.mode", 1)                     # propagation blocking: defaults and small geometries
hub.pagerank(0.85, 0.0, 2)
for nh, gs, win in ((64, 256, 512), (0, 64, 64), (1024, 4096, 3001)):
    capi.set_option("pagerank.hub_slots", nh)
    capi.set_option("pagerank.group_slots", gs)
    capi.set_option("pagerank.window", win)
    capi.set_option("pagerank.chunk", 1024)
    hub.pagerank(0.85, 0.0, 2)
    gg.pagerank(0.85, 1e-4, 3)
# the pruned search (code rows: 512 <= ld <= 2048) on an index of each metric, also after writes of the vectors
for metric in (capi.L2, capi.COSINE, capi.IP):
    X = rng.random((1200, 516), dtype=np.float32) - (0.0 if metric == capi.L2 else 0.3)
    g = capi.HnswIndex.build(X, metric=metric, m=8, ef_construction=40)
    Q = rng.random((40, 516), dtype=np.float32) - (0.0 if metric == capi.L2 else 0.3)
    capi.set_option("hnsw.mode", 1)
    g.search(Q, 5, 16)
    g.update(np.array([2, 700], np.uint32), rng.random((2, 516), dtype=np.float32))
    g.insert_at(np.array([10], np.uint32), rng.random((1, 516), dtype=np.float32))
    g.search(Q, 5, 16, row_pass=rng.random(1201) < 0.5)
    capi.set_option("hnsw.mode", -1)
# filter mask in every search mode, F64 index, the compacted-frontier SSSP, sharded operator at world size 1
X = rng.random((1500, 48), dtype=np.float32)
g = capi.HnswIndex.build(X, m=8, ef_construction=40)
Q = rng.random((40, 48), dtype=np.float32)
for mode in (1, 0, 2):
    capi.set_option("hnsw.mode", mode)
    g.search(Q, 5, 40, row_pass=rng.random(1500) < 0.3)
capi.set_option("hnsw.mode", -1)
ni, rp, ci, ep = g.export_levels()
g64 = capi.HnswIndex.stage(X.astype(np.float64), ni, rp, ci, ep, m_max0=16, m_max=8)
g64.search_f64(Q.astype(np.float64), 5, 40, row_pass=rng.random(1500) < 0.5)
capi.set_option("sssp.frontier", 1)
gg.sssp(np.arange(0, 300, 50, dtype=np.uint32))
gg.closeness()
capi.set_option("sssp.frontier", 0)
capi.set_option("sssp.wide", 1)
gg.sssp(np.arange(0, 300, 100, dtype=np.uint32))
gg.sssp_paths(np.array([0, 5], np.uint32), np.array([7, 9], np.uint32), forb_nodes=[[3], []], forb_edges=[[], [(5, 9)]])
capi.set_option("sssp.wide", 0)
for exch in (1, 0):
    capi.set_option("shard.exchange", exch)
    capi.set_option("shard.tile", 16)
    grp = capi.ShardGroup(capi.ShardGroup.unique_id(), 0, 1)
    grp.attach(g)
    grp.search(Q, 5, 40)
    grp.close()
gx = capi.HnswIndex.build(X[:300], m=6, ef_construction=30, max_batch=1, extend_candidates=True)
gx.search(Q, 5, 30)
print("sanitize workload done")
