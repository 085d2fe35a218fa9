"""The random-gather ceiling that bench.py config 2 is judged against: gathers of random rows in the search kernel's
geometry (tools/gather_ceiling.cu: 4 CTAs x 4 warps per SM, or the CTAs that fit for rows over 14 KB, `depth` rows in
flight per warp), over buffers the size of config 2's: 1 M rows of 3072 B (f32, D = 768) and 1 M rows of 784 B (the
uint8 code rows), 16-byte aligned; --row-bytes takes other sizes (12288,16384: the rows of 3072- and 4096-wide f32
indexes, bulk mode only).  Two modes (--mode, comma-separated):

  bulk  one cp.async.bulk + mbarrier per row from one issuing lane into a per-warp shared-memory ring (depth 1..16)
  ldg   every lane loads its words (lane + 32 i) with ld.global.nc.L1::no_allocate into registers, `depth` rows in
        flight as register sets; depths past 96 words per lane in flight are skipped
  ldg128  the same with 16-byte loads (vector lane + 32 i): 2 warp instructions per 784-byte row instead of 7;
          depths past 72 words per lane in flight are skipped

--visited adds one random atomicOr per row into a per-warp bitmap of rows / 32 words, as the search's visited test does.
Prints one JSON line per (mode, row size, depth) with GB/s, rows/s and the mean latency per request, then one line with
the card, its power limit and the best rate per mode and row size.

    python tools/gather_ceiling.py [--mode bulk,ldg,ldg128] [--visited] [--rows 1000000] [--reqs 2000]
                                   [--depths 1,2,3,4,6,8,12,16] [--row-bytes 3072,784] [--lib PATH]

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
    ap.add_argument("--mode", default="bulk", help="comma-separated: bulk, ldg, ldg128")
    ap.add_argument("--visited", action="store_true", help="one random atomicOr per row into a per-warp bitmap")
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    modes = {"bulk": 0, "ldg": 1, "ldg128": 2}
    if set(a.mode.split(",")) - set(modes):
        raise SystemExit(f"--mode takes {', '.join(modes)}")
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        L = C.CDLL(a.lib or compile_lib(tmp))
        L.gather_run.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                 C.POINTER(C.c_float), C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint32)]
        info = card()
        clk_mhz = info["sm_max_mhz"] or 1980.0
        visited = None
        if a.visited:  # one bitmap per resident warp (16 per SM at most)
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            visited = torch.zeros(sms * 16 * ((a.rows + 31) // 32), dtype=torch.int32, device="cuda")
        best = {}
        for row_bytes in [int(r) for r in a.row_bytes.split(",")]:
            buf = torch.empty(a.rows * row_bytes, dtype=torch.uint8, device="cuda")
            buf.fill_(1)
            for mode in a.mode.split(","):
                for depth in [int(d) for d in a.depths.split(",")]:
                    if mode == "ldg" and depth * ((row_bytes + 127) // 128) > 96:
                        continue  # words per lane in flight past the 128-register budget (they would spill)
                    if mode == "ldg128" and depth * ((row_bytes + 511) // 512 * 4) > 72:
                        continue
                    ms, lat, nw = C.c_float(), C.c_ulonglong(), C.c_uint32()
                    for _ in range(2):  # the first launch warms up; the second is reported
                        if visited is not None:
                            visited.zero_()
                        rc = L.gather_run(modes[mode], C.c_void_p(buf.data_ptr()), a.rows, row_bytes, depth, a.reqs,
                                          C.c_void_p(visited.data_ptr() if visited is not None else None),
                                          C.byref(ms), C.byref(lat), C.byref(nw))
                        if rc:
                            raise SystemExit(f"gather_run failed with CUDA error {rc}")
                    warps = nw.value  # resident warps: 16 per SM, fewer for rows wider than 14 KB
                    nbytes = warps * a.reqs * row_bytes
                    gbs = nbytes / (ms.value * 1e-3) / 1e9
                    lat_cyc = lat.value / (warps * a.reqs)
                    key = f"{mode}/{row_bytes}"
                    best[key] = max(best.get(key, 0.0), gbs)
                    print(json.dumps({"mode": mode, "visited": a.visited, "row_bytes": row_bytes, "depth": depth,
                                      "warps": warps, "GB_per_s": round(gbs, 1),
                                      "G_rows_per_s": round(warps * a.reqs / (ms.value * 1e-3) / 1e9, 3),
                                      "mean_latency_cycles": round(lat_cyc), "mean_latency_us_at_max_clock":
                                      round(lat_cyc / clk_mhz, 3), "ms": round(ms.value, 3)}), flush=True)
            del buf
            torch.cuda.empty_cache()
        print(json.dumps({**info, "visited": a.visited, "best_GB_per_s": {k: round(v, 1) for k, v in best.items()}}),
              flush=True)


if __name__ == "__main__":
    main()
