"""The code rows and the L2 lower bound of cozo_b200/csrc/hnsw_codes.cuh, which let the search skip f32 rows of neighbours
that cannot be admitted.  tests/emu/codes_bound_emu.cpp runs the library's own quantize_row / code_lower_bound on random
and adversarial rows (constant rows, rows on the code grid, magnitudes from 1e-38 to 3e38, subnormals, NaN, +-inf,
dims that are not a multiple of 4) and asserts that the bound never exceeds the distance summed in the search kernel's
order."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("codes") / "codes_bound_emu")
    r = subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-o", out, os.path.join(EMU, "codes_bound_emu.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_lower_bound_never_exceeds_the_kernel_distance(exe, seed):
    r = subprocess.run([exe, "20000", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
