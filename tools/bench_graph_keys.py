"""Cost of turning node keys into dense graph ids: the host std::map assignment that as_directed_graph used to run
(fixed_rule/mod.rs:164-179) against memcmp encoding plus the device assignment (cozo_gpu_graph_stage_keys).  Prints one
JSON line per workload, then a summary line with the card and its power limit.

Per workload (RMAT graphs with Int keys, edge factor 16, ids permuted and spread over i64; air-routes with its string
codes):
  map_s      host std::map<DataValue, u32> lookup per endpoint, single-threaded (_cozo_host.bench_id_assign)
  encode_s   host memcmp encoding of the same endpoints into one buffer + offsets
  stage_s    H2D of keys (+ offsets) and cozo_gpu_graph_stage_keys through to the CSR, host wall clock (the call ends
             in a stream synchronise); median of --reps after one warm-up
  stage_event_ms  the same call between two CUDA events on the default stream
  rule_s     the PageRank rule end to end through the host mirror (tuple scan, encoding, staging, PageRank, the
             RegularTempStore fill); rows are built before the clock starts
Anything skipped (over --map-max-scale / --rule-max-scale) is written as "not measured".

  python tools/bench_graph_keys.py [--scales 20 22 24] [--map-max-scale 20] [--rule-max-scale 22] [--reps 3] [--out F]
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
from tests.hostmod import load  # noqa: E402
from tests.util import rmat_edges  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def stage_times(kb, ko, reps):
    import torch
    walls, events, n = [], [], 0
    for i in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t = time.perf_counter()
        e0.record()
        g = capi.Graph.from_keys(kb, ko)
        e1.record()
        wall = time.perf_counter() - t
        e1.synchronize()
        n, m = g.n, g.m
        g.close()
        if i:
            walls.append(wall)
            events.append(e0.elapsed_time(e1))
    return float(np.median(walls)), float(np.median(events)), n, m


def workload(h, name, keys, src_dst, scale, args):
    run_map = scale is None or scale <= args.map_max_scale
    enc = h.bench_id_assign(keys, run_map)
    kb, ko = enc["key_bytes"], enc["key_off"]
    stage_s, stage_ms, n, m = stage_times(kb, ko, args.reps)
    if run_map:
        assert enc["distinct"] == n, (enc["distinct"], n)
    del kb, ko, enc["key_bytes"], enc["key_off"]
    rec = {"workload": name, "edges": m, "endpoints": enc["endpoints"], "nodes": n,
           "map_s": enc["map_s"] if run_map else "not measured", "encode_s": enc["encode_s"],
           "stage_s": stage_s, "stage_event_ms": stage_ms}
    if src_dst is not None and (scale is None or scale <= args.rule_max_scale):
        r = h.bench_rule_int_edges("PageRank", src_dst[0], src_dst[1], {})
        assert r["rows"] == n
        rec["rule_s"] = r["seconds"]
    else:
        rec["rule_s"] = "not measured"
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="*", default=[20, 22, 24])
    ap.add_argument("--map-max-scale", type=int, default=20)
    ap.add_argument("--rule-max-scale", type=int, default=22)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    h = load()
    h.init(0)
    capi.init(0)
    recs = []
    d = np.load(os.path.join(ROOT, "tests", "golden", "air_routes.npz"))
    codes = [str(c) for c in d["codes"]]
    keys = [codes[i] for pair in zip(d["fr"], d["to"]) for i in pair]
    recs.append(workload(h, "air-routes (string codes)", keys, None, None, args))
    rows = [[codes[a], codes[b]] for a, b in zip(d["fr"], d["to"])]
    t = time.perf_counter()
    out = h.Db().run_fixed_rule("PageRank", [rows], {})
    recs[-1]["rule_s"] = time.perf_counter() - t     # includes converting the Python rows
    assert len(out) == recs[-1]["nodes"]
    for scale in args.scales:
        n, s, t = rmat_edges(scale, 16, scale)
        perm = np.random.default_rng(scale + 1).permutation(n).astype(np.int64) * 1_000_003 - (1 << 45)
        src, dst = perm[s], perm[t]
        del s, t
        keys = np.stack([src, dst], 1).ravel()
        recs.append(workload(h, f"rmat-{scale} (int keys)", keys, (src, dst), scale, args))
        del keys, src, dst
    lines = [json.dumps(r) for r in recs]
    lines.append(json.dumps({"card": card(), "reps": args.reps}))
    for ln in lines:
        print(ln, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
