"""Row-sharded corpus: one process per GPU, one HNSW graph per shard (SURVEY.md §8e).

The operator itself lives behind the C ABI (`cozo_gpu_shards_*`, `cozo_gpu_hnsw_stage_sharded`,
`cozo_gpu_hnsw_search_sharded[_dev]` in csrc/sharded.cu; Python class `capi.ShardGroup`): query broadcast,
per-shard search, exchange of the per-shard top-k lists (fused peer stores over CUDA IPC, or ONE NCCL
all-gather per list) and the k-way merge all happen inside libcozo_gpu.so.

What is left here is host-side plumbing that does not need a GPU and is covered by the world_size-2 gloo test:
  * `ShardedTopK`  — shard offsets (row-contiguous partition) and the list exchange over any torch.distributed
                     backend, i.e. the collective contract the library implements with NCCL;
  * `merge_lists`  — the merge specification in numpy (what topk_merge_kernel computes);
  * `make_group`   — rendezvous helper: rank 0 creates the 128-byte NCCL unique id, torch.distributed carries it.
The result is the k-NN over the union of the shards *as searched shard by shard* — parity is defined against the
oracle run with the same sharding, not against a single big graph.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


class ShardedTopK:
    """Collective plumbing shared by the tests: shard offsets + list exchange."""

    def __init__(self, local_rows: int, device: torch.device, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.device = device
        rows = torch.tensor([local_rows], dtype=torch.int64, device=device)
        if self.world > 1:
            allr = torch.empty(self.world, dtype=torch.int64, device=device)
            dist.all_gather_into_tensor(allr, rows, group=group)
        else:
            allr = rows
        # global id of shard s' row 0 = rows of the shards before it (row-contiguous partition)
        self.offsets = torch.cumsum(allr, 0) - allr
        self.total_rows = int(allr.sum().item())

    def gather(self, local_dist: torch.Tensor, local_ids: torch.Tensor):
        """[B,k] per rank -> ([S,B,k] dist, [S,B,k] ids); exactly one all-gather per tensor."""
        B, k = local_dist.shape
        if self.world == 1:
            return local_dist.view(1, B, k), local_ids.view(1, B, k)
        all_d = torch.empty((self.world, B, k), dtype=local_dist.dtype, device=self.device)
        all_i = torch.empty((self.world, B, k), dtype=local_ids.dtype, device=self.device)
        dist.all_gather_into_tensor(all_d.view(-1), local_dist.contiguous().view(-1), group=self.group)
        dist.all_gather_into_tensor(all_i.view(-1), local_ids.contiguous().view(-1), group=self.group)
        return all_d, all_i


def merge_lists(all_ids: np.ndarray, all_dist: np.ndarray, offsets, k: int):
    """[S,B,k] per-shard lists (local u32 ids, 0xFFFFFFFF padded, nearest first) -> global top-k:
    ids u64 = offsets[s] + local id (UINT64_MAX padded), dist f32, or f64 for f64 lists (+inf padded); ties go to the
    lower shard."""
    S, B, _ = all_ids.shape
    out_i = np.full((B, k), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    out_d = np.full((B, k), np.inf, np.float64 if np.asarray(all_dist).dtype == np.float64 else np.float32)
    for q in range(B):
        cand = [(float(all_dist[s, q, j]), s, j, int(offsets[s]) + int(all_ids[s, q, j]))
                for s in range(S) for j in range(all_ids.shape[2]) if all_ids[s, q, j] != 0xFFFFFFFF]
        cand.sort(key=lambda t: (t[0], t[1], t[2]))
        for r, c in enumerate(cand[:k]):
            out_i[q, r] = c[3]
            out_d[q, r] = c[0]
    return out_i, out_d


def make_group(index, rank: int | None = None, world: int | None = None):
    """collective: a capi.ShardGroup over the ranks of the default torch.distributed group, with `index` attached"""
    from . import capi
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    uid = [capi.ShardGroup.unique_id() if rank == 0 else None]
    if world > 1:
        dist.broadcast_object_list(uid, src=0)
    grp = capi.ShardGroup(uid[0], rank, world)
    grp.attach(index)
    return grp
