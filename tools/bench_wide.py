"""Search throughput of f32 HNSW indexes wider than the register query (ld > 2048), built on the device.

For each `N x D` configuration: U[0,1) vectors generated on the device (seeded), an index built with the device
builder (m, ef_construction), then `--steps` timed batches of `--batch` queries at ef, k through cozo_gpu_hnsw_search_dev,
each batch a distinct set of queries, after `--warmup` untimed batches.  Each step is timed with CUDA events.  Prints one
JSON line per configuration, then one with the card and its power limit (read in the same run):

  qps             queries per second over the timed steps
  alg_GB_per_s    algorithmic bytes per second: per query dist_evals * ld * 4 + nodes_expanded * 8 + nbr_reads * 4 + ld * 4
                  (from the per-query counters): the rows scored, the adjacency reads, the query
  recall_at_10    GPU search vs the oracle search on the exported graph, on a `--sample` of the first batch
  identical_sets  fraction of the sample whose top-k id sets are equal
  build_s         device build time (host clock around the call, which synchronises)

  python tools/bench_wide.py [--configs 250000x4096,330000x3072] [--m 16] [--efc 200] [--ef 200] [--k 10]
                             [--batch 4096] [--steps 10] [--warmup 2] [--sample 256] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cozo_b200 import capi  # noqa: E402


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, plim, clk = (r.stdout.strip().splitlines()[0].split(", ") + ["", "", ""])[:3] if r.returncode == 0 else ("", "", "")
    return {"gpu": name, "power_limit_w": float(plim) if plim else None, "sm_max_mhz": float(clk) if clk else None}


def run(n, dim, a, emit):
    import torch
    from oracle import oracle as O
    gen = torch.Generator(device="cuda").manual_seed(1000 + dim)
    X = torch.rand((n, dim), generator=gen, device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    t = time.perf_counter()
    g = capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(), n_vectors=n, dim=dim)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t
    ld = (dim + 3) // 4 * 4
    B, k = a.batch, a.k
    Qs = torch.rand((a.warmup + a.steps, B, dim), generator=gen, device="cuda", dtype=torch.float32)
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    ms, evals, expanded, reads = [], 0, 0, 0
    for s in range(a.warmup + a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        g.search_dev(Qs[s].data_ptr(), B, k, a.ef, ids.data_ptr(), dist.data_ptr(), qstats_ptr=qs.data_ptr(),
                     stream=stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        if s >= a.warmup:
            ms.append(e0.elapsed_time(e1))
            st = qs.cpu().numpy().view(np.uint32).astype(np.int64)
            evals += int(st[:, 0].sum())
            expanded += int(st[:, 1].sum())
            reads += int(st[:, 2].sum())
    secs = sum(ms) / 1e3
    nq = B * a.steps
    alg_bytes = evals * ld * 4 + expanded * 8 + reads * 4 + nq * ld * 4
    # quality on a sample of the first timed batch: GPU vs the oracle on the exported graph
    Xh = X.cpu().numpy()
    ni, rp, ci, ep = g.export_levels()
    view = O.OracleHnsw.from_levels(Xh, O.HnswLevels(ni, rp, ci, ep))
    Qh = Qs[a.warmup, : a.sample].cpu().numpy()
    gi, _, _, _ = g.search(Qh, k, a.ef)
    oi, _, _, _ = view.search(Qh, k, a.ef, n_threads=os.cpu_count() or 1)
    rec = float(np.mean([len(set(x) & set(y)) / k for x, y in zip(gi, oi)]))
    same = float(np.mean([set(x) == set(y) for x, y in zip(gi, oi)]))
    emit({"n": n, "dim": dim, "m": a.m, "ef_construction": a.efc, "ef": a.ef, "k": k, "batch": B, "steps": a.steps,
          "build_s": round(build_s, 2), "qps": round(nq / secs, 1), "step_ms_median": round(float(np.median(ms)), 3),
          "step_ms_min": round(min(ms), 3), "step_ms_max": round(max(ms), 3),
          "dist_evals_per_query": round(evals / nq, 1), "alg_GB_per_s": round(alg_bytes / secs / 1e9, 1),
          "recall_at_10": round(rec, 4), "identical_sets": round(same, 4), "sample": a.sample})
    g.close()
    del X, Qs
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="250000x4096,330000x3072")
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    capi.init(0)
    out = open(a.out, "a") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    for c in a.configs.split(","):
        n, dim = (int(x) for x in c.lower().split("x"))
        run(n, dim, a, emit)
    emit(card())


if __name__ == "__main__":
    main()
