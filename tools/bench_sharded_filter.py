"""Cost of the filtered and F64 forms of the sharded HNSW search, at world 1 on one GPU.

One index of `--n` x `--dim` U[0,1) f32 vectors (generated on the device, seeded) is built with the device builder
(m, ef_construction) and attached to a one-rank shard group.  Each step searches a distinct batch of `--batch` queries
at ef, k; the forms alternate step by step, after `--warmup` untimed steps of each, and every step is timed with CUDA
events on the calling stream (device forms) or with a host clock around the call (host forms, which synchronise):

  sharded            cozo_gpu_hnsw_search_sharded_dev
  sharded_filt_P     cozo_gpu_hnsw_search_sharded_filtered_dev, mask passing P % of the rows (seeded)
  single_filt_50     cozo_gpu_hnsw_search_filtered_dev on the same index and mask as sharded_filt_50
  f64_single         cozo_gpu_hnsw_search_f64 on an F64 copy (the f32 vectors widened, same graph; host form)
  f64_sharded        cozo_gpu_hnsw_search_sharded_f64 on a one-rank group holding that copy (host form)

The filtered sharded lists of the last timed step are compared with the single-GPU ones (ids and distances), and the
two F64 forms with each other.  World sizes above 1 are not measured here.  The last line names the card and its power
limit, read in the same run.

  python tools/bench_sharded_filter.py [--n 1000000] [--dim 768] [--m 16] [--efc 200] [--ef 200] [--k 10]
                                       [--batch 4096] [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import ctypes as C
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


def stats(ms):
    return {"steps": len(ms), "ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3),
            "ms_max": round(max(ms), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    capi.init(0)
    out = open(a.out, "a") if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    n, dim, B, k, ef = a.n, a.dim, a.batch, a.k, a.ef
    gen = torch.Generator(device="cuda").manual_seed(2024)
    X = torch.rand((n, dim), generator=gen, device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    t = time.perf_counter()
    g = capi.HnswIndex.build(None, m=a.m, ef_construction=a.efc, vectors_dev_ptr=X.data_ptr(), n_vectors=n, dim=dim)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t
    grp = capi.ShardGroup(capi.ShardGroup.unique_id(), 0, 1)
    grp.attach(g)
    rng = np.random.default_rng(7)
    masks = {p: torch.from_numpy(capi.pack_row_mask(rng.random(n) < p / 100).view(np.int32)).cuda()
             for p in (100, 50, 1)}
    total = a.warmup + a.steps
    Qs = torch.rand((total, B, dim), generator=gen, device="cuda", dtype=torch.float32)
    oi = torch.empty((B, k), dtype=torch.int64, device="cuda")
    od = torch.empty((B, k), dtype=torch.float32, device="cuda")
    si = torch.empty((B, k), dtype=torch.int32, device="cuda")
    sd = torch.empty((B, k), dtype=torch.float32, device="cuda")
    L = capi.load()
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream

    def single_filtered(q, mask):
        capi._check(L.cozo_gpu_hnsw_search_filtered_dev(g._h, q.data_ptr(), B, k, ef, -1.0, mask.data_ptr(),
                                                        si.data_ptr(), sd.data_ptr(), None, None, sp))

    forms = {
        "sharded": lambda q: grp.search_dev(q.data_ptr(), B, k, ef, oi.data_ptr(), od.data_ptr(), None, sp),
        **{f"sharded_filt_{p}": (lambda q, p=p: grp.search_dev(q.data_ptr(), B, k, ef, oi.data_ptr(), od.data_ptr(),
                                                               None, sp, row_mask_ptr=masks[p].data_ptr()))
           for p in (100, 50, 1)},
        "single_filt_50": lambda q: single_filtered(q, masks[50]),
    }
    ms = {f: [] for f in forms}
    for s in range(total):
        for f, fn in forms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn(Qs[s])
            e1.record(stream)
            torch.cuda.synchronize()
            if s >= a.warmup:
                ms[f].append(e0.elapsed_time(e1))
    # the last step again, filtered at 50 %: sharded == single-GPU (offset 0)
    forms["sharded_filt_50"](Qs[-1])
    single_filtered(Qs[-1], masks[50])
    torch.cuda.synchronize()
    s_ids = si.cpu().numpy().view(np.uint32).astype(np.uint64)
    s_ids[s_ids == 0xFFFFFFFF] = np.uint64(0xFFFFFFFFFFFFFFFF)
    same32 = bool(np.array_equal(oi.cpu().numpy().view(np.uint64), s_ids) and
                  np.array_equal(od.cpu().numpy(), sd.cpu().numpy()))
    base = float(np.median(ms["sharded"]))
    for f in forms:
        emit({"form": f, **stats(ms[f]), "vs_sharded_unfiltered": round(float(np.median(ms[f])) / base, 4)})
    emit({"check": "sharded_filt_50 == single_filt_50 (ids, distances)", "equal": same32})
    grp.close()
    # F64: the same graph over the widened vectors
    lv = g.export_levels()
    X64 = X.double().cpu().numpy()
    del X
    torch.cuda.empty_cache()
    t = time.perf_counter()
    g64 = capi.HnswIndex.stage(X64, *lv, m_max0=2 * a.m, m_max=a.m)
    stage64_s = time.perf_counter() - t
    del X64
    grp64 = capi.ShardGroup(capi.ShardGroup.unique_id(), 0, 1)
    grp64.attach(g64)
    Q64 = [Qs[s].double().cpu().numpy() for s in range(total)]
    ms64 = {"f64_single": [], "f64_sharded": []}
    kms64 = {"f64_single": [], "f64_sharded": []}
    res = {}
    for s in range(total):
        for f in ms64:
            t = time.perf_counter()
            r = g64.search_f64(Q64[s], k, ef) if f == "f64_single" else grp64.search_f64(Q64[s], k, ef)
            dt = (time.perf_counter() - t) * 1e3
            if s >= a.warmup:
                ms64[f].append(dt)
                kms64[f].append(r[3].kernel_ms)
            res[f] = r
    si64, sd64 = res["f64_single"][0].astype(np.uint64), res["f64_single"][1]
    si64[res["f64_single"][0] == 0xFFFFFFFF] = np.uint64(0xFFFFFFFFFFFFFFFF)
    same64 = bool(np.array_equal(res["f64_sharded"][0], si64) and np.array_equal(res["f64_sharded"][1], sd64))
    for f in ms64:
        emit({"form": f, **stats(ms64[f]), "device_ms_median": round(float(np.median(kms64[f])), 3),
              "clock": "host, around the synchronising call (query upload and result download included)"})
    emit({"check": "f64_sharded == f64_single (ids, distances)", "equal": same64})
    emit({"n": n, "dim": dim, "m": a.m, "ef_construction": a.efc, "ef": ef, "k": k, "batch": B, "world": 1,
          "exchange": grp64.info()["exchange"], "build_s": round(build_s, 2), "f64_stage_s": round(stage64_s, 2),
          "f64_vector_GB": round(n * dim * 8 / 1e9, 2), **card()})
    grp64.close()


if __name__ == "__main__":
    main()
