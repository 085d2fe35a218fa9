"""Search throughput of Cosine and IP indexes at config-2 size, with the code-row pruned search.

For each metric (Cosine, IP) and each dataset (U[0,1), normalised Gaussian): `--n x --dim` f32 vectors generated on the
device (seeded), an index built with the device builder (m, ef_construction), then `--steps` timed batches of `--batch`
queries at ef, k through cozo_gpu_hnsw_search_dev (hnsw.mode=1, the warp-per-query kernel, which prunes), each batch a
distinct set of queries, after `--warmup` untimed batches.  Each step is timed with CUDA events.  Prints one JSON line
per configuration, then one with the card and its power limit (read in the same run):

  qps                      queries per second over the timed steps
  f32_rows_per_query       f32 rows fetched per query (the fourth per-query stats word)
  dist_evals_per_query     neighbour evaluations per query (pruned or not)
  rejection_rate           1 - f32 rows fetched / evaluations
  recall_at_10             GPU search vs the oracle search on the exported graph, on a `--sample` of the first batch
  identical_sets           fraction of the sample whose top-k id sets are equal

`--lib` loads another build of libcozo_gpu.so (for example the parent commit's), so that two builds can be compared in
alternating processes on the same card.  The device builder is deterministic, so both build the same graph.

  python tools/bench_metric.py [--n 1000000] [--dim 768] [--metrics cosine,ip] [--data u01,gauss] [--m 16] [--efc 200]
                               [--ef 200] [--k 10] [--batch 4096] [--steps 10] [--warmup 2] [--sample 256]
                               [--lib PATH] [--tag NAME] [--out FILE]
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

METRICS = {"cosine": capi.COSINE, "ip": capi.IP}


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, plim, clk = (r.stdout.strip().splitlines()[0].split(", ") + ["", "", ""])[:3] if r.returncode == 0 else ("", "", "")
    return {"gpu": name, "power_limit_w": float(plim) if plim else None, "sm_max_mhz": float(clk) if clk else None}


def gen(shape, data, g):
    import torch
    if data == "u01":
        return torch.rand(shape, generator=g, device="cuda", dtype=torch.float32)
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float32)
    return x / torch.linalg.vector_norm(x, dim=-1, keepdim=True)


def run(metric_name, data, a, emit):
    import torch
    from oracle import oracle as O
    metric = METRICS[metric_name]
    g = torch.Generator(device="cuda").manual_seed(7000 + a.dim + (0 if data == "u01" else 1))
    X = gen((a.n, a.dim), data, g)
    torch.cuda.synchronize()
    t = time.perf_counter()
    ix = capi.HnswIndex.build(None, metric=metric, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(),
                              n_vectors=a.n, dim=a.dim)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t
    B, k = a.batch, a.k
    Qs = gen((a.warmup + a.steps, B, a.dim), data, g)
    ids = torch.empty((B, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((B, k), dtype=torch.float32, device="cuda")
    qs = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    ms, evals, fetched = [], 0, 0
    capi.set_option("hnsw.mode", 1)
    try:
        for s in range(a.warmup + a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ix.search_dev(Qs[s].data_ptr(), B, k, a.ef, ids.data_ptr(), dist.data_ptr(), qstats_ptr=qs.data_ptr(),
                          stream=stream.cuda_stream)
            e1.record(stream)
            torch.cuda.synchronize()
            if s >= a.warmup:
                ms.append(e0.elapsed_time(e1))
                st = qs.cpu().numpy().view(np.uint32).astype(np.int64)
                evals += int(st[:, 0].sum())
                fetched += int(st[:, 3].sum())
        # quality on a sample of the first timed batch: GPU vs the oracle on the exported graph
        Qh = Qs[a.warmup, : a.sample].cpu().numpy()
        gi, _, _, _ = ix.search(Qh, k, a.ef)
    finally:
        capi.set_option("hnsw.mode", -1)
    rec = same = None
    if a.sample > 0:
        Xh = X.cpu().numpy()
        ni, rp, ci, ep = ix.export_levels()
        view = O.OracleHnsw.from_levels(Xh, O.HnswLevels(ni, rp, ci, ep), metric=metric)
        oi, _, _, _ = view.search(Qh, k, a.ef, n_threads=os.cpu_count() or 1)
        rec = round(float(np.mean([len(set(x) & set(y)) / k for x, y in zip(gi, oi)])), 4)
        same = round(float(np.mean([set(x) == set(y) for x, y in zip(gi, oi)])), 4)
    secs = sum(ms) / 1e3
    nq = B * a.steps
    emit({"tag": a.tag, "metric": metric_name, "data": data, "n": a.n, "dim": a.dim, "m": a.m, "ef_construction": a.efc,
          "ef": a.ef, "k": k, "batch": B, "steps": a.steps, "build_s": round(build_s, 2), "qps": round(nq / secs, 1),
          "step_ms_median": round(float(np.median(ms)), 3), "step_ms_min": round(min(ms), 3),
          "step_ms_max": round(max(ms), 3), "dist_evals_per_query": round(evals / nq, 1),
          "f32_rows_per_query": round(fetched / nq, 1), "rejection_rate": round(1.0 - fetched / evals, 4),
          "recall_at_10": rec, "identical_sets": same, "sample": a.sample})
    ix.close()
    del X, Qs
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--metrics", default="cosine,ip")
    ap.add_argument("--data", default="u01,gauss")
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--lib", default=None, help="another build of libcozo_gpu.so to load instead of the tree's")
    ap.add_argument("--tag", default="tree", help="label of this run's library in the output")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.lib:
        capi.LIB_PATH = os.path.abspath(a.lib)
    capi.init(0)
    out = open(a.out, "a") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    for metric_name in a.metrics.split(","):
        for data in a.data.split(","):
            run(metric_name, data, a, emit)
    emit(card())


if __name__ == "__main__":
    main()
