"""Cost of inserting rows inside the key range of a device-built HNSW index (cozo_gpu_hnsw_insert_at), against an append
and against a full rebuild.  Prints one JSON line per measurement, then a summary line with the card and its power limit.

  (a) insert of `--rows` appended rows                      (keys after every indexed key)
  (b) insert_at of the same number of rows at uniformly random positions
  (c) insert_at of 1 row at position 0: every existing row moves
  (d) a full device build of the index: what re-staging costs when only a rebuild can absorb a :put

Every call ends in a device synchronise, so host wall time is the call's time.  `relabel_bytes` counts each moved row
once (vector, code row, layer-0 ids and distances, degree, upper offset, level, removed flag) plus the id remap pass over
the adjacency arrays (read and write); (c) divides it by the whole call, which also links one row.

  python tools/bench_insert_at.py [--n 1000000] [--dim 768] [--rows 1000] [--reps 3] [--out FILE]
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


# the relabel's device work; shift_rows_kernel / relabel_ids_kernel are its kernels in builds before the shared routine,
# so that one script times both
RELABEL_KERNELS = ("move_rows_kernel", "map_ids_kernel", "shift_rows_kernel", "relabel_ids_kernel", "Memcpy DtoD")


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def relabel_bytes(n_moved, n_total, up_rows, dim, m):
    ld = (dim + 3) // 4 * 4
    code = 16 + (ld + 15) // 16 * 16 if ld >= 512 else 0
    s0, su = (2 * m + 31) // 32 * 32, (m + 31) // 32 * 32
    per_row = ld * 4 + code + 2 * s0 * 4 + 4 + 4 + 1 + 1
    remap = 2 * 4 * (n_total * s0 + up_rows * su + up_rows)
    return n_moved * per_row + remap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--rows", type=int, default=1000)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    capi.init(0)
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    gen = torch.Generator(device="cuda").manual_seed(1)
    X = torch.rand((a.n, a.dim), generator=gen, device="cuda", dtype=torch.float32)
    rng = np.random.default_rng(2)
    t_build, g = timed(lambda: capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(),
                                                    n_vectors=a.n, dim=a.dim))
    emit({"what": "d_build", "n": a.n, "dim": a.dim, "s": t_build})
    del X
    torch.cuda.empty_cache()
    for rep in range(a.reps):
        V = rng.random((a.rows, a.dim), dtype=np.float32)
        n = g.info()[0]
        t, _ = timed(lambda: g.insert(V))
        emit({"what": "a_insert_append", "rep": rep, "rows": a.rows, "n": n, "ms": t * 1e3})
        V = rng.random((a.rows, a.dim), dtype=np.float32)
        n = g.info()[0]
        P = np.sort(rng.integers(0, n + 1, a.rows)).astype(np.uint32)
        t, _ = timed(lambda: g.insert_at(P, V))
        emit({"what": "b_insert_at_random", "rep": rep, "rows": a.rows, "n": n, "rows_moved": int(n - P[0]),
              "ms": t * 1e3})
        V1 = rng.random((1, a.dim), dtype=np.float32)
        n = g.info()[0]
        t, _ = timed(lambda: g.insert_at(np.zeros(1, np.uint32), V1))
        # upper rows ~ n / (m - 1) (level law with multiplier 1/ln m)
        nb = relabel_bytes(n, n + 1, n // (a.m - 1), a.dim, a.m)
        emit({"what": "c_insert_at_front", "rep": rep, "n": n, "ms": t * 1e3, "relabel_bytes": nb,
              "relabel_GBps_lower_bound": nb / t / 1e9})
    # the relabel's own device time, from a profiled run of one more (c): the staging copies, the row moves and the id
    # remap (kernel names and DtoD copies from torch.profiler; the link step and host work are excluded)
    from torch.profiler import ProfilerActivity, profile
    V1 = rng.random((1, a.dim), dtype=np.float32)
    n = g.info()[0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.insert_at(np.zeros(1, np.uint32), V1)
    us = 0.0
    for e in prof.key_averages():
        if any(k in e.key for k in RELABEL_KERNELS):
            us += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    nb = relabel_bytes(n, n + 1, n // (a.m - 1), a.dim, a.m)
    emit({"what": "c_relabel_device_time", "n": n, "relabel_ms": us / 1e3, "relabel_bytes": nb,
          "relabel_GBps": nb / (us * 1e-6) / 1e9 if us else None,
          "note": "bytes count each moved row once; through the staging buffer each is read and written twice"})
    emit({"what": "card", "gpu": card()})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
