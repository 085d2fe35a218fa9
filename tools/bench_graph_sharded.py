"""What the source-sharded graph calls cost at world 1: cozo_gpu_closeness_sharded and cozo_gpu_betweenness_sharded
(status all-gather, result all-gather, rank-order sum) against cozo_gpu_closeness and cozo_gpu_betweenness on the same
graph, alternated call by call.  Weighted R-MAT (edge factor 16, weights k/8 with 1 <= k < 64).  Prints one JSON line
per (call, form, repetition) with the call's device time (`kernel_ms`, CUDA events on its stream) and the host wall
clock around it, a summary line per call, then a line with the card and its power limit.  Speed-up above world 1 is not
measured here: that needs a machine with several GPUs.

  python tools/bench_graph_sharded.py [--scale 16] [--reps 3] [--out F]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch  # noqa: F401  (maps the libnccl the communicator resolves)
    capi.init(0)
    grp = capi.ShardGroup(capi.ShardGroup.unique_id(), 0, 1)
    n, src, dst = rmat_edges(args.scale, 16, 1)
    w = (np.random.default_rng(1).integers(1, 64, src.size) / 8.0).astype(np.float32)
    g = capi.Graph(n, src, dst, w)
    grp.attach_graph(g)
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))
    for name in ("closeness", "betweenness"):
        forms = {"single": getattr(g, name), "sharded_w1": getattr(grp, name)}
        for f in forms.values():  # warm-up: first launches of every kernel
            f()
        ms = {k: [] for k in forms}
        out = {}
        for rep in range(args.reps):
            for form, f in forms.items():
                t = time.perf_counter()
                out[form], kms = f()
                wall = time.perf_counter() - t
                ms[form].append(wall * 1e3)
                emit({"graph": f"rmat{args.scale}", "n": n, "m": int(src.size), "call": name, "form": form, "rep": rep,
                      "kernel_ms": round(kms, 3), "wall_ms": round(wall * 1e3, 3)})
        same = bool(np.array_equal(out["single"].view(np.uint32), out["sharded_w1"].view(np.uint32)))
        emit({"call": name, "median_wall_ms": {k: round(float(np.median(v)), 3) for k, v in ms.items()},
              "extra_ms_at_w1": round(float(np.median(ms["sharded_w1"]) - np.median(ms["single"])), 3),
              "outputs_bit_equal": same})
    grp.close()
    emit({"card": card(), "note": "kernel_ms: CUDA events around the slice's stream; wall_ms: host clock around the "
                                  "whole call, exchange included"})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
