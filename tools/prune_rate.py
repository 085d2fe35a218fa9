"""How many f32 row fetches the pruned L2 search skips (hnsw_codes.cuh): builds an index of U[0,1) vectors on the GPU,
runs one batch with the warp-per-query kernel and prints, from the per-query counters, the evaluations (word 0) and the
f32 rows actually fetched (word 3).  Rejection rate = 1 - fetched / evaluations.

    python tools/prune_rate.py [--rows 1000000] [--dim 768] [--ef 200] [--batch 4096]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from cozo_b200 import capi
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    a = ap.parse_args()
    capi.init(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    X = torch.rand((a.rows, a.dim), dtype=torch.float32, device="cuda", generator=gen)
    Q = torch.rand((a.batch, a.dim), dtype=torch.float32, device="cuda", generator=gen)
    g = capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(), n_vectors=a.rows,
                             dim=a.dim)
    ids = torch.empty((a.batch, a.k), dtype=torch.int32, device="cuda")
    dd = torch.empty((a.batch, a.k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((a.batch, 4), dtype=torch.int32, device="cuda")
    capi.set_option("hnsw.mode", 1)
    g.search_dev(Q.data_ptr(), a.batch, a.k, a.ef, ids.data_ptr(), dd.data_ptr(), None, qs.data_ptr(),
                 torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    s = qs.to(torch.int64).sum(dim=0).cpu().tolist()
    print(json.dumps({"rows": a.rows, "dim": a.dim, "ef": a.ef, "batch": a.batch, "gpu": torch.cuda.get_device_name(0),
                      "dist_evals_per_query": s[0] / a.batch, "f32_rows_per_query": s[3] / a.batch,
                      "rejection_rate": 1.0 - s[3] / s[0]}))


if __name__ == "__main__":
    main()
