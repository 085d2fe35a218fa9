"""The filtered and F64 sharded searches (cozo_gpu_hnsw_search_sharded_filtered[_dev], cozo_gpu_hnsw_search_sharded_f64)
on the CPU: the library's sources compiled against the CPU SIMT emulator (tests/emu/build_emu_lib.py), with the ranks
of a communicator as threads (tests/emu/fake_nccl.cpp), at world sizes 2, 3 and 8 (8 where 8 cores exist) and shards
down to one row.  The scenario itself is tests/emu/sharded_filter_emu.py.  COZO_EMU_SANITIZE=1 builds with ASan + UBSan."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
SANITIZE = os.environ.get("COZO_EMU_SANITIZE") == "1"


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    sys.path.insert(0, EMU)
    try:
        import build_emu_lib
    finally:
        sys.path.remove(EMU)
    return build_emu_lib.build(str(tmp_path_factory.mktemp("emu_lib_sharded_filter")), sanitize=SANITIZE)


def test_sharded_filter_and_f64_on_the_emulated_library(emu_lib):
    """every rank's result == merge_lists of the per-shard filtered / F64 lists, bit for bit, under both exchanges and
    tiles smaller than the batch; recall of identical sets vs the oracle >= 0.995; mixed-dtype groups and wrong-dtype
    entry points answer EINVAL on every rank without hanging"""
    env = dict(os.environ, UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1", ASAN_OPTIONS="detect_leaks=0")
    if SANITIZE:
        env["LD_PRELOAD"] = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True,
                                           text=True).stdout.strip()
    r = subprocess.run([sys.executable, os.path.join(EMU, "sharded_filter_emu.py"), emu_lib], capture_output=True,
                       text=True, timeout=3000, env=env, cwd=ROOT)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
