"""Worker of tests/test_graph_sharded_gpu.py::test_world2: one process per GPU (torchrun).  Every rank stages the same
graph, attaches it to the group and checks the sharded closeness, betweenness and sssp_goals against its own
single-GPU calls; torch.distributed (gloo) only carries the unique id and the betweenness of rank 0."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist
    from cozo_b200 import capi
    from tests.util import rmat_edges
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    dist.init_process_group("gloo")
    torch.cuda.set_device(local)
    capi.init(local)
    n, src, dst = rmat_edges(12, 8, 0x5A53)
    w = (np.random.default_rng(4).integers(1, 1 << 20, src.size) / 1024.0).astype(np.float32)
    g = capi.Graph(n, src, dst, w)
    uid = [capi.ShardGroup.unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    grp = capi.ShardGroup(uid[0], rank, world)
    grp.attach_graph(g)
    c, _ = grp.closeness()
    assert np.array_equal(c.view(np.uint32), g.closeness()[0].view(np.uint32))
    b, _ = grp.betweenness()
    b1, _ = g.betweenness()
    assert np.allclose(b, b1, rtol=2.0 ** -22, atol=0)
    both = [None] * world
    dist.all_gather_object(both, b)
    assert all(np.array_equal(x.view(np.uint32), b.view(np.uint32)) for x in both)
    rng = np.random.default_rng(9)
    sources = np.sort(rng.choice(n, 301, replace=False)).astype(np.uint32)
    goals = rng.choice(n, 16, replace=False).astype(np.uint32)
    cost, paths, _ = grp.sssp_goals(sources, goals)
    cost1, paths1, _ = g.sssp_goals(sources, goals)
    assert np.array_equal(cost.view(np.uint32), cost1.view(np.uint32)) and paths == paths1
    _, ties, _ = grp.sssp_goals(sources, goals, keep_ties=True)
    _, ties1, _ = g.sssp_goals(sources, goals, keep_ties=True)
    key = lambda r: r[np.lexsort((r[:, 1], r[:, 0]))]  # noqa: E731
    assert all(np.array_equal(key(a), key(b)) for a, b in zip(ties, ties1))
    # two calls reaching the group in different orders on different ranks: EINVAL on both, then the group still works
    try:
        grp.closeness() if rank == 0 else grp.betweenness()
        raise AssertionError("expected EINVAL")
    except capi.CozoGpuError as e:
        assert e.code == capi.E_INVAL
    assert np.array_equal(grp.closeness()[0].view(np.uint32), c.view(np.uint32))
    poison = np.ones(1, np.int32) if rank == 1 else None
    try:
        grp.closeness(poison=poison)
        raise AssertionError("expected EKILLED")
    except capi.CozoGpuError as e:
        assert e.code == capi.E_KILLED
    dist.barrier()
    grp.close()
    if rank == 0:
        print(f"GRAPH_SHARDED_OK world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
