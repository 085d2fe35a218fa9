"""The random-gather ceiling that bench.py config 2 is judged against: cp.async.bulk + mbarrier gathers of random rows in
the search kernel's geometry (tools/gather_ceiling.cu: 4 CTAs x 4 warps per SM, or the CTAs that fit for rows over 14 KB, one issuing lane per warp, a per-warp
ring of depth 1..16), over buffers the size of config 2's: 1 M rows of 3072 B (f32, D = 768) and 1 M rows of 784 B (the
uint8 code rows), 16-byte aligned; --row-bytes takes other sizes (12288,16384: the rows of 3072- and 4096-wide f32
indexes).  Prints one JSON line per (row size, depth) with GB/s and the mean latency per request,
then one line with the card, its power limit and the best rate per row size.

    python tools/gather_ceiling.py [--rows 1000000] [--reqs 2000] [--depths 1,2,3,4,6,8,12,16] [--row-bytes 3072,784]
                                   [--lib PATH]

The kernel is compiled with nvcc into a temporary directory (or taken from --lib).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def compile_lib(tmp: str) -> str:
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    out = os.path.join(tmp, "gather_ceiling.so")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                    "-shared", os.path.join(HERE, "gather_ceiling.cu"), "-o", out], check=True)
    return out


def card() -> dict:
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk = (q[torch.cuda.current_device()].split(", ") + ["", "", ""])[:3] if q else ("", "", "")
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": float(plim) if plim else None,
            "sm_max_mhz": float(clk) if clk else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reqs", type=int, default=2000, help="requests per warp and launch")
    ap.add_argument("--depths", default="1,2,3,4,6,8,12,16")
    ap.add_argument("--row-bytes", default="3072,784", help="comma-separated row sizes, multiples of 16")
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        L = C.CDLL(a.lib or compile_lib(tmp))
        L.gather_run.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_float),
                                 C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint32)]
        info = card()
        clk_mhz = info["sm_max_mhz"] or 1980.0
        best = {}
        for row_bytes in [int(r) for r in a.row_bytes.split(",")]:
            buf = torch.empty(a.rows * row_bytes, dtype=torch.uint8, device="cuda")
            buf.fill_(1)
            for depth in [int(d) for d in a.depths.split(",")]:
                ms, lat, nw = C.c_float(), C.c_ulonglong(), C.c_uint32()
                for _ in range(2):  # the first launch warms up; the second is reported
                    rc = L.gather_run(C.c_void_p(buf.data_ptr()), a.rows, row_bytes, depth, a.reqs, C.byref(ms),
                                      C.byref(lat), C.byref(nw))
                    if rc:
                        raise SystemExit(f"gather_run failed with CUDA error {rc}")
                warps = nw.value  # resident warps: 16 per SM, fewer for rows wider than 14 KB
                nbytes = warps * a.reqs * row_bytes
                gbs = nbytes / (ms.value * 1e-3) / 1e9
                lat_cyc = lat.value / (warps * a.reqs)
                best[row_bytes] = max(best.get(row_bytes, 0.0), gbs)
                print(json.dumps({"row_bytes": row_bytes, "depth": depth, "warps": warps, "GB_per_s": round(gbs, 1),
                                  "mean_latency_cycles": round(lat_cyc), "mean_latency_us_at_max_clock":
                                  round(lat_cyc / clk_mhz, 3), "ms": round(ms.value, 3)}), flush=True)
            del buf
            torch.cuda.empty_cache()
        print(json.dumps({**info, "best_GB_per_s": {str(k): round(v, 1) for k, v in best.items()}}), flush=True)


if __name__ == "__main__":
    main()
