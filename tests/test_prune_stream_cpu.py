"""The pruned L2 search's per-warp stream (prune_chunk in hnsw_device.cuh) on a stricter CPU-emulated library, against
the ld.global search (hnsw.mode=0), which never prunes.

The library is built here the way tests/emu/build_emu_lib.py builds it, with two differences made in a scratch copy of
tests/emu: rows of 16 elements and up get code rows (CODES_MIN_LD, hnsw_codes.cuh), so that small dimensions run the
pruned search, and bulk copies land late into poisoned buffers (tests/emu/late_copies.hpp), so that a slot read before
its wait, or refilled while its copy is outstanding, fails here.  Covered: m 16 (one 32-id adjacency chunk) and m 48
(three), a corpus with 30 % duplicate rows (many visited neighbours among the speculatively fetched ones), ef 16 and 64.
Ids, distances (as bits) and qstats words 0-2 must be equal; word 3 (f32 rows fetched) must stay <= word 0 and be smaller
in total.  The library's scenarios that use bulk copies run on the same build."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")

SCRIPT = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[2])
from cozo_b200 import capi
capi.LIB_PATH = sys.argv[1]
m, dup, ef = int(sys.argv[3]), float(sys.argv[4]), int(sys.argv[5])
rng = np.random.default_rng(m * 1000 + ef + int(dup * 100))
n, dim, B, k = 500, 36, 24, 10
X = rng.random((n, dim), dtype=np.float32)
if dup:
    d = rng.choice(n, int(dup * n), replace=False)
    X[d] = X[rng.integers(0, n, len(d))]
Q = rng.random((B, dim), dtype=np.float32)
Q[: B // 4] = X[rng.integers(0, n, B // 4)]  # some queries sit on (duplicated) rows
g = capi.HnswIndex.build(X, m=m, ef_construction=40, level_seed=5)
out = {}
for mode in (1, 0):
    ids = np.zeros((B, k), np.uint32)
    dist = np.zeros((B, k), np.float32)
    qs = np.zeros((B, 4), np.uint32)
    capi.set_option("hnsw.mode", mode)
    g.search_dev(Q.ctypes.data, B, k, ef, ids.ctypes.data, dist.ctypes.data, None, qs.ctypes.data)
    out[mode] = (ids, dist, qs)
(i1, d1, s1), (i0, d0, s0) = out[1], out[0]
assert np.array_equal(i1, i0), "ids differ"
assert np.array_equal(d1.view(np.uint32), d0.view(np.uint32)), "distances differ"
assert np.array_equal(s1[:, :3], s0[:, :3]), "traversal counters differ"
assert np.array_equal(s0[:, 3], s0[:, 0])
assert np.all(s1[:, 3] <= s1[:, 0])
assert int(s1[:, 3].sum()) < int(s1[:, 0].sum()), "nothing was pruned"
print("fetched", int(s1[:, 3].sum()), "of", int(s1[:, 0].sum()), "EMU_OK")
'''


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("emu_late")
    emu = str(d / "emu")
    shutil.copytree(EMU, emu, ignore=shutil.ignore_patterns("__pycache__"))
    with open(os.path.join(EMU, "cuda_emu.hpp")) as f:
        src = f.read()
    with open(os.path.join(EMU, "late_copies.hpp")) as f:
        late = f.read()
    a = src.index("// ---- mbarrier + 1-D bulk copy")
    b = src.index("inline void fence_proxy_async_smem() {}")
    # every library source includes this header (through the fake cuda_runtime.h) before hnsw_codes.cuh
    src = src[:a] + late + src[b:]
    src = src.replace("#pragma once", "#pragma once\n#define CODES_MIN_LD 16u", 1)
    with open(os.path.join(emu, "cuda_emu.hpp"), "w") as f:
        f.write(src)
    sys.path.insert(0, EMU)
    try:
        import build_emu_lib
    finally:
        sys.path.remove(EMU)
    saved = build_emu_lib.EMU
    build_emu_lib.EMU = emu
    try:
        return build_emu_lib.build(str(d / "lib"))
    finally:
        build_emu_lib.EMU = saved


@pytest.mark.parametrize("ef", [16, 64])
@pytest.mark.parametrize("m,dup", [(16, 0.0), (48, 0.0), (16, 0.3)])
def test_pruned_stream_equals_unpruned_search(emu_lib, m, dup, ef):
    env = dict(os.environ, COZO_EMU_SM_COUNT="4", COZO_EMU_COPY_SEED=str(m + ef))
    r = subprocess.run([sys.executable, "-c", SCRIPT, emu_lib, ROOT, str(m), str(dup), str(ef)], capture_output=True,
                       text=True, timeout=1200, env=env, cwd=ROOT)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2500:] + r.stderr[-4000:]


@pytest.mark.parametrize("scenario", ["hnsw", "hnsw_maintenance", "builder_fidelity", "fuzz_hnsw", "graph", "pagerank"])
def test_library_scenarios_with_late_copies(emu_lib, scenario):
    env = dict(os.environ, COZO_EMU_SM_COUNT="4")
    r = subprocess.run([sys.executable, os.path.join(EMU, "run_emu_lib.py"), emu_lib, scenario], capture_output=True,
                       text=True, timeout=3000, env=env, cwd=ROOT)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2500:] + r.stderr[-4000:]
