"""Where a warp of the warp-per-query search spends its cycles, per phase of a hop, at bench.py config 2's shapes.

Builds libcozo_gpu.so with -DCOZO_HOP_CLOCKS into its own directory (or takes --lib), builds config 2's index (1 M x 768
U[0,1), m 16, ef_construction 200, bench.py's seeds), runs one warm-up and one measured batch of 4096 queries at ef 200
with the warp-per-query kernel, and prints the clock64 totals over all warps of the measured batch:
pop + adjacency read, visited test, code-ring waits, code scoring, f32-ring waits, f32 scoring + admissions.

    python tools/hop_clocks.py [--rows 1000000] [--dim 768] [--ef 200] [--batch 4096] [--lib PATH] [--out-lib DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PHASES = ["pop_adjacency", "visited_test", "code_ring_wait", "code_scoring", "f32_ring_wait", "f32_scoring_admission"]


def build_instrumented(outdir: str) -> str:
    from cozo_b200 import build as B
    os.makedirs(outdir, exist_ok=True)
    flags = B.NVCC_FLAGS + ["-DCOZO_HOP_CLOCKS"]

    def one(s):
        obj = os.path.join(outdir, s.replace(".cu", ".o"))
        subprocess.run([B._nvcc()] + flags + ["-c", os.path.join(B.CSRC, s), "-o", obj], check=True)
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(one, B.SOURCES))
    lib = os.path.join(outdir, "libcozo_gpu.so")
    subprocess.run([B._nvcc(), "-shared", "-o", lib] + objs + B.ARCH + ["-cudart", "static", "-ldl"], check=True)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--ef", type=int, default=200)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--lib", default=None, help="an already instrumented libcozo_gpu.so")
    ap.add_argument("--out-lib", default=None, help="build the instrumented library here and stop")
    a = ap.parse_args()
    if a.out_lib:
        print(build_instrumented(a.out_lib))
        return
    with tempfile.TemporaryDirectory() as tmp:
        lib = a.lib or build_instrumented(tmp)
        import torch
        from bench import gen_vectors
        from cozo_b200 import capi
        capi.LIB_PATH = lib
        L = capi.load()
        if not hasattr(L, "cozo_gpu_hop_clocks"):
            raise SystemExit(f"{lib} was not built with -DCOZO_HOP_CLOCKS")
        capi.init(0)
        X = gen_vectors(a.rows, a.dim, 0x5EED0001)
        g = capi.HnswIndex.build(X, m=16, ef_construction=200, level_seed=0x5EED0003)
        Q = torch.from_numpy(gen_vectors(2 * a.batch, a.dim, 0x5EED0002).reshape(2, a.batch, a.dim)).cuda()
        ids = torch.empty((a.batch, a.k), dtype=torch.int32, device="cuda")
        dd = torch.empty((a.batch, a.k), dtype=torch.float32, device="cuda")
        qs = torch.zeros((a.batch, 4), dtype=torch.int32, device="cuda")
        capi.set_option("hnsw.mode", 1)
        clk = (C.c_ulonglong * len(PHASES))()
        for s in range(2):
            L.cozo_gpu_hop_clocks(clk)  # reset
            g.search_dev(Q[s].data_ptr(), a.batch, a.k, a.ef, ids.data_ptr(), dd.data_ptr(), None, qs.data_ptr(),
                         torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
        if L.cozo_gpu_hop_clocks(clk):
            raise SystemExit(capi.load().cozo_gpu_last_error().decode())
        st = qs.to(torch.int64).sum(0).cpu().tolist()
        tot = sum(clk)
        print(json.dumps({
            "gpu": torch.cuda.get_device_name(), "rows": a.rows, "dim": a.dim, "ef": a.ef, "batch": a.batch,
            "cycles": dict(zip(PHASES, list(clk))), "share": {p: round(c / tot, 4) for p, c in zip(PHASES, clk)},
            "cycles_per_hop": {p: round(c / st[1], 1) for p, c in zip(PHASES, clk)},
            "dist_evals": st[0], "nodes_expanded": st[1], "nbr_reads": st[2], "f32_rows_fetched": st[3]}), flush=True)


if __name__ == "__main__":
    main()
