"""The filtered and F64 forms of the sharded operator (cozo_gpu_hnsw_search_sharded_filtered[_dev],
cozo_gpu_hnsw_search_sharded_f64) at world 1 with the ShardGroup in this process: the sharded result equals the
single-GPU search of the same shard bit for bit (ids as u64, distances, counts), under both exchanges and with tiles
smaller than the batch.  The two-GPU run lives in tests/sharded_filter_worker.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE64 = np.uint64(0xFFFFFFFFFFFFFFFF)
N, DIM, M, K, EF, B = 3000, 48, 8, 10, 64, 333


def _as_global(ids, dist, cnt):
    """single-GPU lists -> the sharded form at world 1 (offset 0): u64 ids, UINT64_MAX padding"""
    g = ids.astype(np.uint64)
    g[ids == 0xFFFFFFFF] = NONE64
    return g, dist, cnt


def _group(capi, index, exchange, tile):
    """a fresh communicator re-negotiates the exchange"""
    capi.set_option("shard.exchange", exchange)
    capi.set_option("shard.tile", tile)
    grp = capi.ShardGroup(capi.ShardGroup.unique_id(), 0, 1)
    grp.attach(index)
    return grp


def _einval(capi, fn):
    with pytest.raises(capi.CozoGpuError) as e:
        fn()
    assert e.value.code == capi.E_INVAL


@pytest.fixture(scope="module")
def shards(gpu):
    import torch  # noqa: F401  (maps the libnccl the communicator resolves)
    out = {}
    rng = np.random.default_rng(3)
    for metric in (gpu.L2, gpu.COSINE, gpu.IP):
        X = rng.random((N, DIM), dtype=np.float32) - (0.0 if metric == gpu.L2 else 0.4)
        g = gpu.HnswIndex.build(X, metric=metric, m=M, ef_construction=60, level_seed=11 + metric)
        X64 = rng.random((N, DIM)) - (0.0 if metric == gpu.L2 else 0.4)
        g64 = gpu.HnswIndex.stage(X64, *g.export_levels(), metric=metric, m_max0=2 * M, m_max=M)
        out[metric] = (X, g, g64)
    yield out
    gpu.set_option("shard.exchange", 1)
    gpu.set_option("shard.tile", 65536)


@pytest.mark.parametrize("tile", [65536, 100])
@pytest.mark.parametrize("exchange", [1, 0])
@pytest.mark.parametrize("metric", [0, 1, 2])
def test_filtered_equals_single_gpu(gpu, shards, metric, exchange, tile):
    import torch
    X, g, _ = shards[metric]
    rng = np.random.default_rng(40 + metric)
    Q = rng.random((B, DIM), dtype=np.float32) - (0.0 if metric == gpu.L2 else 0.4)
    keep = rng.random(N) < 0.5
    grp = _group(gpu, g, exchange, tile)
    try:
        ids, dist, cnt, _ = grp.search(Q, K, EF, row_pass=keep)
        assert grp.info()["exchange"] == ("fused" if exchange else "nccl")
        ei, ed, ec = _as_global(*g.search(Q, K, EF, row_pass=keep)[:3])
        assert np.array_equal(ids, ei) and np.array_equal(dist.view(np.uint32), ed.view(np.uint32))
        assert np.array_equal(cnt, ec) and ec.min() > 0
        # radius with a mask
        r = float(np.median(ed[:, 3]))
        ids, dist, cnt, _ = grp.search(Q, K, EF, radius=r, row_pass=keep)
        ri, rd, rc = _as_global(*g.search(Q, K, EF, radius=r, row_pass=keep)[:3])
        assert np.array_equal(ids, ri) and np.array_equal(dist.view(np.uint32), rd.view(np.uint32))
        assert np.array_equal(cnt, rc)
        # all pass == the unfiltered sharded search; all reject == padding only
        ui, ud, uc, _ = grp.search(Q, K, EF)
        ids, dist, cnt, _ = grp.search(Q, K, EF, row_pass=np.ones(N, bool))
        assert np.array_equal(ids, ui) and np.array_equal(dist, ud) and np.array_equal(cnt, uc)
        ids, dist, cnt, _ = grp.search(Q, K, EF, row_pass=np.zeros(N, bool))
        assert np.all(ids == NONE64) and np.all(dist == np.inf) and np.all(cnt == 0)
        # device form on a caller stream, three times back to back (the gather sets alternate)
        qd = torch.from_numpy(Q).cuda()
        md = torch.from_numpy(gpu.pack_row_mask(keep).view(np.int32)).cuda()
        oi = torch.empty((B, K), dtype=torch.int64, device="cuda")
        od = torch.empty((B, K), dtype=torch.float32, device="cuda")
        for _ in range(3):
            grp.search_dev(qd.data_ptr(), B, K, EF, oi.data_ptr(), od.data_ptr(), None,
                           torch.cuda.current_stream().cuda_stream, row_mask_ptr=md.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(oi.cpu().numpy().view(np.uint64), ei)
        assert np.array_equal(od.cpu().numpy().view(np.uint32), ed.view(np.uint32))
        # misuse: the F64 entry point on an f32 group, a NULL mask on a non-empty shard
        _einval(gpu, lambda: grp.search_f64(Q.astype(np.float64), K, EF))
        L = gpu.load()
        st = gpu.SearchStats()
        assert L.cozo_gpu_hnsw_search_sharded_filtered(grp._h, Q.ctypes.data, B, K, EF, -1.0, -1, None, ids.ctypes.data,
                                                       dist.ctypes.data, None, gpu.C.byref(st)) == gpu.E_INVAL
        assert L.cozo_gpu_hnsw_search_sharded_filtered_dev(grp._h, qd.data_ptr(), B, K, EF, -1.0, None, oi.data_ptr(),
                                                           od.data_ptr(), None, None) == gpu.E_INVAL
    finally:
        grp.close()


@pytest.mark.parametrize("tile", [65536, 100])
@pytest.mark.parametrize("exchange", [1, 0])
@pytest.mark.parametrize("metric", [0, 1, 2])
def test_f64_equals_single_gpu(gpu, shards, metric, exchange, tile):
    _, g, g64 = shards[metric]
    rng = np.random.default_rng(50 + metric)
    Q = rng.random((B, DIM)) - (0.0 if metric == gpu.L2 else 0.4)
    keep = rng.random(N) < 0.5
    grp = _group(gpu, g64, exchange, tile)
    try:
        for row_pass in (None, keep):
            ei, ed, ec = _as_global(*g64.search_f64(Q, K, EF, row_pass=row_pass)[:3])
            for root in (0, -1):
                ids, dist, cnt, _ = grp.search_f64(Q, K, EF, root=root, row_pass=row_pass)
                assert dist.dtype == np.float64
                assert np.array_equal(ids, ei) and np.array_equal(dist.view(np.uint64), ed.view(np.uint64))
                assert np.array_equal(cnt, ec)
        r = float(np.median(ed[:, 3]))
        ri, rd, rc = _as_global(*g64.search_f64(Q, K, EF, radius=r, row_pass=keep)[:3])
        ids, dist, cnt, _ = grp.search_f64(Q, K, EF, radius=r, row_pass=keep)
        assert np.array_equal(ids, ri) and np.array_equal(dist, rd) and np.array_equal(cnt, rc)
        # misuse: the f32 entry points on an F64 group
        Q32 = Q.astype(np.float32)
        _einval(gpu, lambda: grp.search(Q32, K, EF))
        _einval(gpu, lambda: grp.search(Q32, K, EF, row_pass=keep))
    finally:
        grp.close()


def test_filtered_and_f64_world2(gpu):
    if gpu.device_count() < 2:
        pytest.skip("needs two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29621", os.path.join(ROOT, "tests", "sharded_filter_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "SHARDED_FILTER_OK world=2" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
