"""ShortestPathDijkstra with a termination relation: cozo_gpu_sssp_goals (each search stops once its goals are settled,
only the goal answers come back) against cozo_gpu_sssp_multi (every search to the fixed point, n_src x n distances and
predecessors back to the host, where the goal columns are picked out).  Prints one JSON line per (graph, case), then a
line with the card and its power limit.

Graphs: weighted R-MAT (edge factor 16, weights k/8 with 1 <= k < 64).  Cases, with --goals goals each:
  random  goals and --sources sources drawn uniformly from the nodes (many R-MAT nodes have no in-edges, so a goal may
          be unreachable and its searches cannot stop early);
  near    sources drawn from the 2-hop in-neighbourhood of the goals, where every goal settles within a few hops.
sssp_multi runs on as many of the same sources as --multi-bytes of host buffers allow (8 bytes per (source, node)).
Per call: the call's own device time (CUDA events on its stream from the first copy to the last, `kernel_ms`), the
host wall clock around it, ms per source for both, and the bytes each call returns to the host.

  python tools/bench_graph_goals.py [--scales 22 24] [--sources 256] [--goals 8] [--multi-bytes 8e9] [--out F]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cozo_b200 import capi  # noqa: E402
from tests.util import rmat_edges  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def near_sources(src, dst, goals, k, rng):
    hop1 = np.unique(src[np.isin(dst, goals)])
    hop2 = np.unique(src[np.isin(dst, hop1)])
    pool = np.setdiff1d(np.union1d(hop1, hop2), goals)
    return np.sort(rng.choice(pool, min(k, pool.size), replace=False)).astype(np.uint32)


def run_case(g, n, name, scale, sources, goals, multi_bytes):
    t = time.perf_counter()
    cost, paths, goals_ms = g.sssp_goals(sources, goals)
    goals_wall = time.perf_counter() - t
    path_nodes = sum(len(p) for row in paths for p in row)
    goals_bytes = cost.nbytes + (cost.size + 1) * 8 + path_nodes * 4
    k = int(min(sources.size, max(1, multi_bytes // (n * 8))))
    t = time.perf_counter()
    dist, pred, multi_ms = g.sssp(sources[:k])
    multi_wall = time.perf_counter() - t
    same = bool(np.array_equal(dist[:, goals].view(np.uint32), cost[:k].view(np.uint32)))
    del dist, pred
    return {"graph": f"rmat{scale}", "case": name, "n": n, "m": g.m, "n_src": int(sources.size),
            "n_goals": int(goals.size), "reachable_pairs": int(np.isfinite(cost).sum()),
            "goals_ms": round(goals_ms, 3), "goals_wall_s": round(goals_wall, 3),
            "goals_ms_per_src": round(goals_ms / sources.size, 4), "goals_host_bytes": int(goals_bytes),
            "multi_n_src": k, "multi_ms": round(multi_ms, 3), "multi_wall_s": round(multi_wall, 3),
            "multi_ms_per_src": round(multi_ms / k, 4), "multi_host_bytes": int(k * n * 8),
            "multi_host_bytes_all_sources": int(sources.size * n * 8), "costs_equal_on_shared_sources": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24])
    ap.add_argument("--sources", type=int, default=256)
    ap.add_argument("--goals", type=int, default=8)
    ap.add_argument("--multi-bytes", type=float, default=8e9)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    capi.init(0)
    lines = []
    # warm-up: module load and first launches of every kernel both calls use
    n, s, d = rmat_edges(12, 16, 0)
    g = capi.Graph(n, s, d, np.full(s.size, 0.5, np.float32))
    g.sssp_goals(np.arange(4), np.arange(4, 8))
    g.sssp(np.arange(4))
    g.close()
    for scale in args.scales:
        rng = np.random.default_rng(args.seed + scale)
        n, src, dst = rmat_edges(scale, 16, args.seed + scale)
        w = (rng.integers(1, 64, src.size) / 8.0).astype(np.float32)
        g = capi.Graph(n, src, dst, w)
        goals = rng.choice(n, args.goals, replace=False).astype(np.uint32)
        sources = np.sort(rng.choice(n, args.sources, replace=False)).astype(np.uint32)
        cases = [("random", sources, goals)]
        goals = rng.choice(np.unique(dst), args.goals, replace=False).astype(np.uint32)  # goals with in-edges
        cases.append(("near", near_sources(src, dst, goals, args.sources, rng), goals))
        del src, dst, w
        for name, srcs, gls in cases:
            r = run_case(g, n, name, scale, srcs, gls, int(args.multi_bytes))
            print(json.dumps(r), flush=True)
            lines.append(json.dumps(r))
        g.close()
    tail = json.dumps({"card": card(), "note": "goals_ms / multi_ms: CUDA events around each call's stream"})
    print(tail)
    lines.append(tail)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
