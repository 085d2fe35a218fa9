"""The source-sharded graph calls (cozo_gpu_graph_attach_sharded, cozo_gpu_closeness_sharded,
cozo_gpu_betweenness_sharded, cozo_gpu_sssp_goals_sharded) on the device.

World 1 with the ShardGroup in this process, in both state forms and across source chunks (`sssp.smem`,
`sssp.max_chunk_sources`): closeness, betweenness and the goal costs equal the single-GPU calls bit for bit, and so do
the tie-edge offsets and, per source, the tie-edge multisets (the single-GPU call lists a source's tie edges in no
particular order).  Among tied shortest paths the single-GPU call may return any one, so the paths are compared bit for
bit on a graph whose shortest paths are unique.  World 2 (tests/graph_sharded_worker.py under torchrun) needs two
GPUs."""
import contextlib
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests.util import rmat_edges

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULTS = {"sssp.smem": 1, "sssp.max_chunk_sources": 0}
COMBOS = [{"sssp.smem": smem, "sssp.max_chunk_sources": k} for smem in (1, 0) for k in (0, 1, 7, 97)]
CIDS = [f"smem{c['sssp.smem']}-chunk{c['sssp.max_chunk_sources']}" for c in COMBOS]


@contextlib.contextmanager
def options(capi, opts):
    try:
        for k, v in opts.items():
            capi.set_option(k, v)
        yield
    finally:
        for k, v in DEFAULTS.items():
            capi.set_option(k, v)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def sort_rows(r):
    r = np.asarray(r, np.uint32).reshape(-1, 2)
    return r[np.lexsort((r[:, 1], r[:, 0]))]


def graphs():
    rng = np.random.default_rng(0x5A50)
    n, m = 1000, 6000
    src, dst = rng.integers(0, n - 24, m).astype(np.uint32), rng.integers(0, n - 24, m).astype(np.uint32)
    yield "unique", n, src, dst, (rng.integers(1, 1 << 20, m) / 1024.0).astype(np.float32)   # no tied paths
    n, src, dst = rmat_edges(10, 8, 0x5A51)
    yield "rmat10", n + 16, src, dst, (np.random.default_rng(3).integers(1, 64, src.size) / 8.0).astype(np.float32)
    n, src, dst = rmat_edges(10, 8, 0x5A52)
    yield "rmat10-unweighted", n + 16, src, dst, None


@pytest.fixture(scope="module")
def group(gpu):
    import torch  # noqa: F401  (maps the libnccl the communicator resolves)
    grp = gpu.ShardGroup(gpu.ShardGroup.unique_id(), 0, 1)
    yield grp
    grp.close()


@pytest.fixture(scope="module")
def staged(gpu):
    return [(name, n, gpu.Graph(n, src, dst, w)) for name, n, src, dst, w in graphs()]


@pytest.mark.parametrize("opts", COMBOS, ids=CIDS)
def test_world1_equals_single_gpu(gpu, group, staged, opts):
    single = gpu.load().cozo_gpu_sssp_goals
    sharded = gpu.load().cozo_gpu_sssp_goals_sharded
    with options(gpu, opts):
        for name, n, g in staged:
            group.attach_graph(g)
            assert np.array_equal(bits(group.closeness()[0]), bits(g.closeness()[0])), name
            assert np.array_equal(bits(group.betweenness()[0]), bits(g.betweenness()[0])), name
            rng = np.random.default_rng(n)
            sources = np.sort(rng.choice(n, 150, replace=False)).astype(np.uint32)
            goals = rng.choice(n, 12, replace=False).astype(np.uint32)
            wc, wo, wr, _ = gpu.sssp_goals_once(single, g._h, sources, goals, False, 1 << 22)
            gc, go, gr, _ = gpu.sssp_goals_once(sharded, group._h, sources, goals, False, 1 << 22)
            assert np.array_equal(bits(gc), bits(wc)), name
            if name == "unique":
                assert np.array_equal(go, wo) and np.array_equal(gr, wr)
            _, wo, wr, _ = gpu.sssp_goals_once(single, g._h, sources, goals, True, 1 << 22)
            tc, to, tr, _ = gpu.sssp_goals_once(sharded, group._h, sources, goals, True, 1 << 22)
            assert np.array_equal(bits(tc), bits(wc)) and np.array_equal(to, wo), name
            o = to.astype(np.int64)
            for si in range(sources.size):
                a, b = 2 * o[si], 2 * o[si + 1]
                assert np.array_equal(sort_rows(tr[a:b]), sort_rows(wr[a:b])), (name, si)


def test_world1_errors(gpu, group, staged):
    _, n, g = staged[0]
    group.attach_graph(g)
    poison = np.ones(1, np.int32)
    for fn in (lambda: group.closeness(poison=poison), lambda: group.betweenness(poison=poison),
               lambda: group.sssp_goals([1, 2], [3], poison=poison)):
        with pytest.raises(gpu.CozoGpuError) as e:
            fn()
        assert e.value.code == gpu.E_KILLED
    sources, goals = np.arange(40, dtype=np.uint32), np.array([5, 9, 13, 400], np.uint32)
    wc, wo, _, _ = gpu.sssp_goals_once(gpu.load().cozo_gpu_sssp_goals, g._h, sources, goals, False, 1)
    gc, go, gr, _ = gpu.sssp_goals_once(gpu.load().cozo_gpu_sssp_goals_sharded, group._h, sources, goals, False, 1)
    assert int(wo[-1]) > 1 and np.array_equal(go, wo) and np.array_equal(bits(gc), bits(wc)) and not gr.any()
    bare = gpu.ShardGroup(gpu.ShardGroup.unique_id(), 0, 1)             # no graph attached
    out = np.zeros(n, np.float32)
    assert gpu.load().cozo_gpu_closeness_sharded(bare._h, out.ctypes.data, None, None) == gpu.E_INVAL
    bare.close()
    cyc = gpu.Graph(4, np.array([0, 1, 2], np.uint32), np.array([1, 2, 1], np.uint32), np.array([1, 0, 0], np.float32))
    group.attach_graph(cyc)
    with pytest.raises(gpu.CozoGpuError) as e:
        group.betweenness()
    assert e.value.code == gpu.E_UNSUP


def free_port():
    """a TCP port that no other process holds right now, for torchrun's rendezvous"""
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as sock:
        sock.bind(("127.0.0.1", 0))
        return sock.getsockname()[1]


def test_world2(gpu):
    if gpu.device_count() < 2:
        pytest.skip("needs two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(free_port()), os.path.join(ROOT, "tests", "graph_sharded_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "GRAPH_SHARDED_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
