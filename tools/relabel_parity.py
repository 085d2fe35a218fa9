"""Digests of everything a seeded maintenance sequence leaves in an HNSW handle, one JSON line per export.  Run it with
two builds of the library, in separate processes: identical output means byte-identical exports.

The sequence: build (L2, D = 512 by default, so that the index has code rows), insert_at at the front, at random
positions and at the end, remove a tenth, compact, update, insert.  Exported at the end: info, every level (node ids,
row offsets, neighbour ids), the edge distances, the live flags, the vectors read back through
cozo_gpu_hnsw_vectors_dev, and the ids, distances, counts and four per-query stats words of a seeded search_dev batch.
Code rows have no export; the fourth stats word counts the f32 rows fetched past them, so it reflects them.

  python tools/relabel_parity.py [--lib PATH] [--emu] [--n 2000] [--dim 512]
    --lib  the library to load (default: the in-tree build)
    --emu  PATH is the CPU-emulated library (tests/emu/build_emu_lib.py): device pointers are host pointers
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cozo_b200 import capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--emu", action="store_true")
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--dim", type=int, default=512)
    a = ap.parse_args()
    if a.lib:
        capi.LIB_PATH = os.path.abspath(a.lib)
    capi.init(0)
    if not a.emu:
        import torch

    def dev_buffer(shape, dtype):
        if a.emu:
            buf = np.zeros(shape, dtype)
            return buf.ctypes.data, lambda: buf.copy()
        t = torch.zeros(shape, dtype={np.float32: torch.float32, np.uint32: torch.int32}[dtype], device="cuda")
        return t.data_ptr(), lambda: t.cpu().numpy().view(dtype)

    def read_dev(ptr, count):
        if a.emu:
            return np.frombuffer((C.c_char * (count * 4)).from_address(ptr), np.float32).copy()

        class View:
            __cuda_array_interface__ = {"shape": (count,), "typestr": "<f4", "data": (ptr, False), "version": 3}
        return torch.as_tensor(View(), device="cuda").cpu().numpy()

    rng = np.random.default_rng(2024)
    n, dim = a.n, a.dim
    X = rng.random((n + 1000, dim), dtype=np.float32)
    g = capi.HnswIndex.build(X[:n], metric=capi.L2, m=8, ef_construction=60, level_seed=17)
    g.insert_at(np.zeros(40, np.uint32), X[n:n + 40])
    m0 = g.info()[0]
    g.insert_at(np.sort(rng.integers(0, m0 + 1, 200)).astype(np.uint32), X[n + 40:n + 240])
    m0 = g.info()[0]
    g.insert_at(np.full(60, m0, np.uint32), X[n + 240:n + 300])
    m0 = g.info()[0]
    g.remove(np.sort(rng.choice(m0, m0 // 10, replace=False)).astype(np.uint32))
    g.compact()
    m0 = g.info()[0]
    g.update(np.sort(rng.choice(m0, 50, replace=False)).astype(np.uint32), X[n + 300:n + 350])
    g.insert(X[n + 350:n + 450])

    out = {}
    info = g.info()
    out["info"] = np.array([info[0], info[1], info[2], -1 if info[3] is None else info[3]], np.int64)
    ni, rp, ci, _ = g.export_levels()
    for L in range(len(rp)):
        if L:
            out[f"level{L}_nodes"] = ni[L]
        out[f"level{L}_row_ptr"] = rp[L]
        out[f"level{L}_col_idx"] = ci[L]
    for L, d in enumerate(g.export_dists()):
        out[f"level{L}_dist"] = d
    out["live"] = g.export_live()
    p, stride = g.vectors_dev()
    out["vectors"] = read_dev(p, info[0] * stride)
    B, k, ef = 64, 10, 64
    Q = rng.random((B, dim), dtype=np.float32)
    Qd = Q if a.emu else torch.from_numpy(Q).cuda()
    q_ptr = Qd.ctypes.data if a.emu else Qd.data_ptr()
    ids_p, ids = dev_buffer((B, k), np.uint32)
    dist_p, dist = dev_buffer((B, k), np.float32)
    cnt_p, cnt = dev_buffer((B,), np.uint32)
    qs_p, qs = dev_buffer((B, 4), np.uint32)
    g.search_dev(q_ptr, B, k, ef, ids_p, dist_p, count_ptr=cnt_p, qstats_ptr=qs_p)
    if not a.emu:
        torch.cuda.synchronize()
    out["search_ids"], out["search_dist"], out["search_count"], out["search_qstats"] = ids(), dist(), cnt(), qs()

    total = hashlib.sha256()
    for name, arr in out.items():
        b = np.ascontiguousarray(arr).tobytes()
        total.update(name.encode() + b)
        print(json.dumps({"export": name, "bytes": len(b), "sha256": hashlib.sha256(b).hexdigest()[:16]}))
    print(json.dumps({"export": "all", "sha256": total.hexdigest()}))


if __name__ == "__main__":
    main()
