"""The source-sharded graph calls (cozo_gpu_graph_attach_sharded, cozo_gpu_closeness_sharded,
cozo_gpu_betweenness_sharded, cozo_gpu_sssp_goals_sharded) on the CPU: the library's sources compiled against the CPU
SIMT emulator (tests/emu/build_emu_lib.py), with the ranks of a communicator as threads (tests/emu/fake_nccl.cpp), at
world sizes 1, 2, 3 and 8 (8 where 8 cores exist).  The scenario itself is tests/emu/graph_sharded_emu.py.

The emulator runs a kernel's blocks one after the other and keeps every static `__shared__` array in one process-wide
copy, so two rank threads must not run graph.cu's kernels (which use such arrays) at the same time.  This file's build
of the emulated library therefore takes one process-wide lock around each launch in graph.cu; no kernel there waits on
a peer, so the ranks still meet in every collective as on the device."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
GRAPH_LAUNCH_LOCK = """#include <mutex>
inline std::mutex& cozo_emu_graph_mu() { static std::mutex m; return m; }
#define COZO_EMU_GRAPH_LAUNCH(...) \\
  do { std::lock_guard<std::mutex> cozo_emu_lk(cozo_emu_graph_mu()); emu::launch_k(__VA_ARGS__); } while (0)
"""


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    sys.path.insert(0, EMU)
    try:
        import build_emu_lib
    finally:
        sys.path.remove(EMU)
    plain = build_emu_lib.transform

    def transform(name, src):
        text = plain(name, src)
        if name != "graph.cu":
            return text
        return GRAPH_LAUNCH_LOCK + text.replace("emu::launch_k(", "COZO_EMU_GRAPH_LAUNCH(")
    build_emu_lib.transform = transform
    try:
        return build_emu_lib.build(str(tmp_path_factory.mktemp("emu_lib_graph_sharded")))
    finally:
        build_emu_lib.transform = plain


def test_graph_sharded_on_the_emulated_library(emu_lib):
    """closeness and sssp_goals equal the single-GPU calls on every rank; betweenness is equal across ranks and reruns
    and within 2^-23 of the exact judge; mismatched graphs, poison and zero-weight cycles fail alike on every rank"""
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, os.path.join(EMU, "graph_sharded_emu.py"), emu_lib], capture_output=True,
                       text=True, timeout=3000, env=env, cwd=ROOT)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
