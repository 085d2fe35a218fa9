"""cozo_gpu_sssp_goals on the CPU: the library's sources compiled against the CPU SIMT emulator
(tests/emu/build_emu_lib.py), driving tests/test_graph_goals_gpu.py unchanged through COZO_EMU_LIB.  The goal stop in
both state forms and across source chunks, the path read-out, the tied-edge closure, the edge cases and the rule
through the host mirror run here; the natural-size R-MAT-20 case is left to the GPU run."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    sys.path.insert(0, EMU)
    try:
        import build_emu_lib
    finally:
        sys.path.remove(EMU)
    return build_emu_lib.build(str(tmp_path_factory.mktemp("emu_lib_graph_goals")))


def test_graph_goals_gpu_file_on_the_emulated_library(emu_lib):
    env = dict(os.environ, COZO_EMU_LIB=emu_lib, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu",
                        "tests/test_graph_goals_gpu.py"], capture_output=True, text=True, timeout=3600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout
