"""Cost of dropping removed rows from a device-built HNSW index in place (cozo_gpu_hnsw_remove + cozo_gpu_hnsw_compact),
against re-staging the index.  Prints one JSON line per measurement, then a line with the card and its power limit.

One handle `a` goes through four removal steps, each followed by a compaction: 1 row at id 0, then 1 %, 10 % and 50 %
of the remaining rows at random.  For each step:
  remove_ms, compact_ms   host clock around the calls (each ends in a device synchronise)
  moved_bytes             each moved per-node row once (vector, code row, layer-0 ids and distances, degree, upper
                          offset, level, removed flag), every upper-layer row once (an upper bound: rows before the
                          first dropped one stay), and the id remap (read and write) over the kept adjacency
  stage_ms                cozo_gpu_hnsw_stage of the compacted graph (as exported) plus its vectors from host memory:
                          the device part of a re-stage.  The re-stage also decodes `rel:idx` with scan_all first;
                          that runs in the database and is not measured here.
A twin handle `b` (same seed, same build) takes the same removals without compacting.  On the 50 %-removed pair a batch
of queries is timed on b (before) and a (after), alternated, and the outputs are compared through the id map.

  python tools/bench_compact.py [--n 1000000] [--dim 768] [--m 16] [--efc 200] [--reps 5] [--out FILE]
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

NONE = 0xFFFFFFFF


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def moved_bytes(n0, n1, first, up_rows, up_kept, dim, m):
    ld = (dim + 3) // 4 * 4
    code = 16 + (ld + 15) // 16 * 16 if ld >= 512 else 0
    s0, su = (2 * m + 31) // 32 * 32, (m + 31) // 32 * 32
    node_row = ld * 4 + code + 2 * s0 * 4 + 4 + 4 + 1 + 1
    up_row = 2 * su * 4 + 4 + 4
    remap = 2 * 4 * (n1 * s0 + up_kept * su + up_kept + n1)
    return (n0 - first) * node_row + up_rows * up_row + remap


def upper_rows(levels):
    ni = levels[0]
    return sum(int(ni[L].size) for L in range(1, len(ni)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
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
    Xh = X.cpu().numpy()
    t_build, ga = timed(lambda: capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(),
                                                     n_vectors=a.n, dim=a.dim))
    emit({"what": "build", "n": a.n, "dim": a.dim, "s": t_build})
    gb = capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(), n_vectors=a.n,
                              dim=a.dim)
    del X
    torch.cuda.empty_cache()
    rng = np.random.default_rng(2)
    orig = np.arange(a.n)              # original id of every id of `a`
    up0 = upper_rows(ga.export_levels())
    for what, frac in (("1_row_at_0", None), ("1_pct", 0.01), ("10_pct", 0.10), ("50_pct", 0.50)):
        n0 = ga.info()[0]
        ids = np.zeros(1, np.uint32) if frac is None else np.sort(rng.choice(n0, int(n0 * frac), replace=False)).astype(np.uint32)
        gb.remove(orig[ids].astype(np.uint32))
        t_rm, _ = timed(lambda: ga.remove(ids))
        t_c, pi = timed(lambda: ga.compact())
        keep = pi != NONE
        orig = orig[keep]
        n1 = int(keep.sum())
        lv = ga.export_levels()
        up1 = upper_rows(lv)
        nb = moved_bytes(n0, n1, int(ids[0]), up0, up1, a.dim, a.m)
        up0 = up1
        ni, rp, ci, ep = lv
        V = np.ascontiguousarray(Xh[orig])
        t_st, s = timed(lambda: capi.HnswIndex.stage(V, ni, rp, ci, ep, m_max0=2 * a.m, m_max=a.m))
        del s, V
        emit({"what": what, "n_before": n0, "removed": int(ids.size), "n_after": n1, "remove_ms": t_rm * 1e3,
              "compact_ms": t_c * 1e3, "moved_bytes": nb, "moved_GBps_lower_bound": nb / t_c / 1e9,
              "stage_ms": t_st * 1e3})
    # queries on the 50 %-removed index: b before compaction, a after, alternated
    Q = np.random.default_rng(3).random((a.batch, a.dim), dtype=np.float32)
    new_of = np.full(a.n, NONE, np.int64)
    new_of[orig] = np.arange(orig.size)
    for g in (gb, ga):
        g.search(Q, a.k, a.ef)                       # warm-up
    ta, tb = [], []
    for _ in range(a.reps):
        t, rb = timed(lambda: gb.search(Q, a.k, a.ef))
        tb.append(t)
        t, ra = timed(lambda: ga.search(Q, a.k, a.ef))
        ta.append(t)
        valid = np.arange(a.k)[None, :] < rb[2][:, None]
        same = (np.array_equal(ra[2], rb[2]) and np.array_equal(ra[1].view(np.uint32), rb[1].view(np.uint32))
                and np.array_equal(ra[0][valid].astype(np.int64), new_of[rb[0][valid].astype(np.int64)]))
        assert same, "compacted index answers differently"
    emit({"what": "search_50_pct", "batch": a.batch, "ef": a.ef, "k": a.k, "n_before_compact": int(gb.info()[0]),
          "n_after_compact": int(ga.info()[0]), "before_ms": [x * 1e3 for x in tb], "after_ms": [x * 1e3 for x in ta],
          "before_qps_median": a.batch / float(np.median(tb)), "after_qps_median": a.batch / float(np.median(ta)),
          "outputs_equal": True})
    emit({"what": "card", "gpu": card()})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
