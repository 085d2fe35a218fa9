"""Worker of tests/test_sharded_filter_gpu.py::test_filtered_and_f64_world2: one process per GPU (torchrun).  Every rank
evaluates its filter over its own shard's rows; the filtered and F64 sharded searches must equal
cozo_b200.sharded.merge_lists of every rank's single-GPU filtered / F64 lists, bit for bit, under both exchanges and
with tiles smaller than the batch.  torch.distributed (gloo) only carries the unique id and the reference lists."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cozo_b200.sharded import merge_lists  # noqa: E402


def main():
    import torch
    import torch.distributed as dist
    from cozo_b200 import capi
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    dist.init_process_group("gloo")
    torch.cuda.set_device(local)
    capi.init(local)
    n = 2000 + 700 * rank                      # ragged shards
    dim, m, k, ef, B = 48, 8, 10, 64, 333
    rng = np.random.default_rng(200 + rank)
    X = rng.random((n, dim), dtype=np.float32)
    X64 = rng.random((n, dim))
    keep = rng.random(n) < 0.3
    Q = np.random.default_rng(9).random((B, dim), dtype=np.float32)
    Q64 = np.random.default_rng(10).random((B, dim))
    g = capi.HnswIndex.build(X, m=m, ef_construction=60, level_seed=5 + rank)
    g64 = capi.HnswIndex.stage(X64, *g.export_levels(), m_max0=2 * m, m_max=m)
    rows = [None] * world
    dist.all_gather_object(rows, n)
    offsets = np.cumsum([0] + rows[:-1])
    mine = (g.search(Q, k, ef, row_pass=keep)[:2], g64.search_f64(Q64, k, ef, row_pass=keep)[:2],
            g64.search_f64(Q64, k, ef)[:2])
    every = [None] * world
    dist.all_gather_object(every, mine)
    exp = [merge_lists(np.stack([e[j][0] for e in every]), np.stack([e[j][1] for e in every]), offsets, k)
           for j in range(3)]
    md = torch.from_numpy(capi.pack_row_mask(keep).view(np.int32)).cuda()
    qd = torch.from_numpy(Q).cuda()
    for exchange in (1, 0):
        for tile in (65536, 100):
            capi.set_option("shard.exchange", exchange)
            capi.set_option("shard.tile", tile)
            for index, forms in ((g, "f32"), (g64, "f64")):
                uid = [capi.ShardGroup.unique_id() if rank == 0 else None]
                dist.broadcast_object_list(uid, src=0)
                grp = capi.ShardGroup(uid[0], rank, world)
                grp.attach(index)
                for root in (-1, 0, world - 1):
                    if forms == "f32":
                        ids, dd, _, _ = grp.search(Q if root in (-1, rank) else None, k, ef, root=root, B=B,
                                                   row_pass=keep)
                        assert np.array_equal(ids, exp[0][0]) and np.array_equal(dd, exp[0][1]), (exchange, tile, root)
                    else:
                        for j, rp in ((1, keep), (2, None)):
                            ids, dd, _, _ = grp.search_f64(Q64 if root in (-1, rank) else None, k, ef, root=root, B=B,
                                                           row_pass=rp)
                            assert np.array_equal(ids, exp[j][0]) and np.array_equal(dd, exp[j][1]), (exchange, tile, j)
                if forms == "f32":
                    oi = torch.empty((B, k), dtype=torch.int64, device="cuda")
                    od = torch.empty((B, k), dtype=torch.float32, device="cuda")
                    for _ in range(3):
                        grp.search_dev(qd.data_ptr(), B, k, ef, oi.data_ptr(), od.data_ptr(), None,
                                       torch.cuda.current_stream().cuda_stream, row_mask_ptr=md.data_ptr())
                    torch.cuda.synchronize()
                    assert np.array_equal(oi.cpu().numpy().view(np.uint64), exp[0][0])
                    assert np.array_equal(od.cpu().numpy(), exp[0][1])
                dist.barrier()
                grp.close()
    dist.barrier()
    if rank == 0:
        print(f"SHARDED_FILTER_OK world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
