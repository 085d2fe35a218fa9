"""The integer per-row prune test of the pruned L2 search (code_query_prepare / code_int_prunes in
cozo_b200/csrc/hnsw_codes.cuh): the query in fixed point, the exact integer product with the uint8 code row, and the
lower bound evaluated from it in f64.  tests/emu/codes_int_bound_emu.cpp runs the library's own functions on random and
adversarial rows and queries (huge and tiny magnitudes, subnormals, NaN, +-inf, large offsets, dims up to 2048 and not
multiples of 4) against worst distances around the row's distance, its bound, 0, +inf and NaN.  It asserts that a row
whose distance (summed in the search kernel's order) is below the worst distance is never pruned, that no int32 partial
of the product overflows, and that on U[0,1) data the test prunes about as often as the f32 test code_prunes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("codes_int_bound") / "codes_int_bound_emu")
    r = subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-o", out, os.path.join(EMU, "codes_int_bound_emu.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_int_prune_test_never_prunes_an_admissible_row(exe, seed):
    r = subprocess.run([exe, "20000", str(seed)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
