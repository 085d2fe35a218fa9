"""The filtered and F64 forms of the sharded operator on the emulated library (tests/emu/build_emu_lib.py), with the
ranks of a communicator as threads of this process (tests/emu/fake_nccl.cpp).  Usage: sharded_filter_emu.py <path to
libcozo_gpu_emu.so>.  Prints EMU_OK at the end.  TEST INFRASTRUCTURE ONLY.

For every world size, metric, exchange and tile: the operator's result on every rank == cozo_b200.sharded.merge_lists
of each shard's own single-device filtered (or F64) lists, bit for bit; the same merge of the oracle's lists, run shard
by shard with the same masks, agrees on at least 0.995 of the result sets; a group whose shards mix F32 and F64 and
the wrong-dtype entry points fail on every rank without a rank left waiting.
"""
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from cozo_b200 import capi  # noqa: E402

capi.LIB_PATH = os.path.abspath(sys.argv[1])
assert capi._lib is None
os.environ["COZO_GPU_NCCL_LIB"] = os.path.join(os.path.dirname(capi.LIB_PATH), "libfake_nccl.so")
from cozo_b200.sharded import merge_lists  # noqa: E402
from oracle import oracle as O  # noqa: E402

T0 = time.time()
NONE64 = np.uint64(0xFFFFFFFFFFFFFFFF)
DIM, M, K, EF, B = 16, 4, 5, 16, 23


def step(msg):
    print(f"[{time.time() - T0:7.1f}s] {msg}", flush=True)


def run_ranks(world, fn):
    """fn(rank) on `world` threads; every exception is collected, a rank that never returns fails the run"""
    errors = []

    def main(r):
        try:
            fn(r)
        except BaseException as e:  # noqa: BLE001
            import traceback
            errors.append(f"rank {r}: {e!r}\n{traceback.format_exc()}")
    th = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(600)
    assert not any(t.is_alive() for t in th), "a rank hangs"
    assert not errors, "\n".join(errors)


def expect_einval(fn):
    try:
        fn()
    except capi.CozoGpuError as e:
        assert e.code == capi.E_INVAL, e
        return
    raise AssertionError("expected COZO_GPU_EINVAL")


def oracle_lists(search_full, keep, radius):
    """the reference's tail on the oracle's full beam: radius, filter, then the first K"""
    fi, fd, fc, _ = search_full
    ids = np.full((len(fi), K), 0xFFFFFFFF, np.uint32)
    dist = np.full((len(fi), K), np.inf, fd.dtype)
    for q in range(len(fi)):
        sel = [(int(i), d) for i, d in zip(fi[q, :fc[q]], fd[q, :fc[q]])
               if (radius is None or not d > radius) and (keep is None or keep[i])][:K]
        for j, (i, d) in enumerate(sel):
            ids[q, j], dist[q, j] = i, d
    return ids, dist


def same_sets(a, b):
    return np.mean([set(x[x != NONE64].tolist()) == set(y[y != NONE64].tolist()) for x, y in zip(a, b)])


def make_shards(world, metric, seed):
    rng = np.random.default_rng(seed)
    rows = [1] + [int(rng.integers(2, 70)) for _ in range(world - 1)]      # down to a one-row shard
    shards = []
    for r, n in enumerate(rows):
        X = rng.random((n, DIM), dtype=np.float32) - 0.5 + (0.05 if metric == capi.COSINE else 0)
        g = capi.HnswIndex.build(X, metric=metric, m=M, ef_construction=16, level_seed=seed + r)
        lv = g.export_levels()
        X64 = rng.random((n, DIM)) - 0.5 + (0.05 if metric == capi.COSINE else 0)
        g64 = capi.HnswIndex.stage(X64, *lv, metric=metric, m_max0=2 * M, m_max=M)
        shards.append(dict(X=X, X64=X64, g=g, g64=g64, lv=O.HnswLevels(*lv), keep=rng.random(n) < 0.5))
    return rows, np.cumsum([0] + rows[:-1]), shards


def check_world(world, metric):
    rows, offsets, shards = make_shards(world, metric, 1000 * world + metric)
    rng = np.random.default_rng(7 + world)
    Q = rng.random((B, DIM), dtype=np.float32) - 0.5
    Q64 = rng.random((B, DIM)) - 0.5
    sh_lists = [sh["g"].search(Q, K, EF) for sh in shards]
    radius = float(np.median(merge_lists(np.stack([x[0] for x in sh_lists]), np.stack([x[1] for x in sh_lists]),
                                         offsets, K)[1][:, 2])) * (1 + 1e-4)

    def merged(per_shard):
        return merge_lists(np.stack([x[0] for x in per_shard]), np.stack([x[1] for x in per_shard]), offsets, K)
    exp = {  # form -> merged lists of the single-device calls
        ("f32", None): merged([sh["g"].search(Q, K, EF, row_pass=sh["keep"]) for sh in shards]),
        ("f32", radius): merged([sh["g"].search(Q, K, EF, radius=radius, row_pass=sh["keep"]) for sh in shards]),
        "f64": merged([sh["g64"].search_f64(Q64, K, EF, row_pass=sh["keep"]) for sh in shards]),
        "f64u": merged([sh["g64"].search_f64(Q64, K, EF) for sh in shards]),
    }
    # the oracle, shard by shard with the same masks
    orc32, orc64 = [], []
    for sh in shards:
        ix = O.OracleHnsw.from_levels(sh["X"], sh["lv"], metric=metric)
        orc32.append(oracle_lists(ix.search(Q, EF, EF, n_threads=2), sh["keep"], None))
        ix64 = O.OracleHnsw.from_levels(sh["X64"].astype(np.float32), sh["lv"], metric=metric)
        orc64.append(oracle_lists(ix64.search_f64(sh["X64"], Q64, EF, EF, n_threads=2), sh["keep"], None))
    rec32 = same_sets(merged(orc32)[0], exp[("f32", None)][0])
    rec64 = same_sets(merged(orc64)[0], exp["f64"][0])
    assert rec32 >= 0.995 and rec64 >= 0.995, (rec32, rec64)
    for exchange in (1, 0):
        for tile in (65536, 7):
            capi.set_option("shard.exchange", exchange)
            capi.set_option("shard.tile", tile)
            uid32, uid64 = capi.ShardGroup.unique_id(), capi.ShardGroup.unique_id()

            def rank_main(r):
                sh = shards[r]
                grp = capi.ShardGroup(uid32, r, world)
                assert grp.attach(sh["g"]) == (int(offsets[r]), sum(rows))
                for root in (-1, 0):
                    for rad in (None, radius):
                        ids, dd, cnt, _ = grp.search(Q if root in (-1, r) else None, K, EF, radius=rad, root=root, B=B,
                                                     row_pass=sh["keep"])
                        ei, ed = exp[("f32", rad)]
                        assert np.array_equal(ids, ei) and np.array_equal(dd, ed), (exchange, tile, root, rad)
                        assert np.array_equal(cnt, (ei != NONE64).sum(1))
                # device form, twice back to back (double-buffered sets); the emulated device memory is host memory
                mask = capi.pack_row_mask(sh["keep"])
                oi, od = np.zeros((B, K), np.uint64), np.zeros((B, K), np.float32)
                for _ in range(2):
                    grp.search_dev(Q.ctypes.data, B, K, EF, oi.ctypes.data, od.ctypes.data, None, None,
                                   row_mask_ptr=mask.ctypes.data)
                assert np.array_equal(oi, exp[("f32", None)][0]) and np.array_equal(od, exp[("f32", None)][1])
                expect_einval(lambda: grp.search_f64(Q64, K, EF))                     # F64 entry point, F32 group
                grp.close()
                grp = capi.ShardGroup(uid64, r, world)
                grp.attach(sh["g64"])
                for root in (-1, 0):
                    for key, keep in (("f64", sh["keep"]), ("f64u", None)):
                        ids, dd, cnt, _ = grp.search_f64(Q64 if root in (-1, r) else None, K, EF, root=root, B=B,
                                                         row_pass=keep)
                        assert dd.dtype == np.float64
                        assert np.array_equal(ids, exp[key][0]) and np.array_equal(dd, exp[key][1]), (key, root)
                        assert np.array_equal(cnt, (exp[key][0] != NONE64).sum(1))
                expect_einval(lambda: grp.search(Q, K, EF))                          # f32 entry points, F64 group
                expect_einval(lambda: grp.search(Q, K, EF, row_pass=sh["keep"]))
                grp.close()
            run_ranks(world, rank_main)
    capi.set_option("shard.exchange", 1)
    capi.set_option("shard.tile", 65536)
    step(f"world {world} metric {metric} rows {rows}: filtered (host, device, radius, roots) and F64 (masked or not, "
         f"roots) == merge of the per-shard lists under both exchanges and tiles 65536 / 7; recall of identical sets "
         f"vs the oracle f32 {rec32:.4f}, f64 {rec64:.4f}")


def check_misuse():
    """mixed-dtype group: every entry point fails on every rank; a NULL mask on a non-empty shard fails (here on every
    rank, as the caller must make the same call everywhere)"""
    rows, offsets, shards = make_shards(2, capi.L2, 5)
    Q = np.random.default_rng(1).random((4, DIM), dtype=np.float32)
    uid, uid2 = capi.ShardGroup.unique_id(), capi.ShardGroup.unique_id()
    L = capi.load()

    def mixed(r):
        grp = capi.ShardGroup(uid, r, 2)
        grp.attach(shards[r]["g"] if r == 0 else shards[r]["g64"])
        expect_einval(lambda: grp.search(Q, K, EF))
        expect_einval(lambda: grp.search(Q, K, EF, row_pass=shards[r]["keep"]))
        expect_einval(lambda: grp.search_f64(Q.astype(np.float64), K, EF))
        oi, od = np.zeros((4, K), np.uint64), np.zeros((4, K), np.float32)
        expect_einval(lambda: grp.search_dev(Q.ctypes.data, 4, K, EF, oi.ctypes.data, od.ctypes.data))
        grp.close()

    def null_mask(r):
        grp = capi.ShardGroup(uid2, r, 2)
        grp.attach(shards[r]["g"])
        oi, od = np.zeros((4, K), np.uint64), np.zeros((4, K), np.float32)
        st = capi.SearchStats()
        rc = L.cozo_gpu_hnsw_search_sharded_filtered(grp._h, Q.ctypes.data, 4, K, EF, -1.0, -1, None, oi.ctypes.data,
                                                     od.ctypes.data, None, capi.C.byref(st))
        assert rc == capi.E_INVAL, rc
        rc = L.cozo_gpu_hnsw_search_sharded_filtered_dev(grp._h, Q.ctypes.data, 4, K, EF, -1.0, None, oi.ctypes.data,
                                                         od.ctypes.data, None, None)
        assert rc == capi.E_INVAL, rc
        ids, _, _, _ = grp.search(Q, K, EF)                 # the group still works after the refused calls
        assert ids.shape == (4, K)
        grp.close()
    run_ranks(2, mixed)
    run_ranks(2, null_mask)
    step("mixed-dtype group and wrong-dtype entry points: EINVAL on every rank, no rank left waiting; NULL mask: EINVAL")


if __name__ == "__main__":
    capi.init(0)
    check_misuse()
    for world in ((2, 3, 8) if (os.cpu_count() or 1) >= 8 else (2, 3)):
        for metric in (capi.L2, capi.COSINE, capi.IP):
            check_world(world, metric)
    print("EMU_OK")
