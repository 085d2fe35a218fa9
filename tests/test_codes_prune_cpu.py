"""The per-row prune test of the pruned L2 search (code_prunes / code_prune_radius in cozo_b200/csrc/hnsw_codes.cuh),
which replaces `code_lower_bound(dt, err) >= worst` without a square root per row.  tests/emu/codes_prune_emu.cpp runs
the library's own functions on the random and adversarial rows of codes_bound_emu.cpp against worst distances around
the row's distance, its bound, 0, +inf and NaN, and asserts that a row whose distance (summed in the search kernel's
order) is below the worst distance is never pruned."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("codes_prune") / "codes_prune_emu")
    r = subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-o", out, os.path.join(EMU, "codes_prune_emu.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_prune_test_never_prunes_an_admissible_row(exe, seed):
    r = subprocess.run([exe, "20000", str(seed)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
