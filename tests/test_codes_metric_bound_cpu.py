"""The Cosine and IP per-row prune test of the pruned search (code_dot_query / code_dot_radius / code_dot_prunes in
cozo_b200/csrc/hnsw_codes.cuh): an upper bound on the kernel's f32 dot product from the exact integer product of the
uint8 code row with the fixed-point query, turned into a lower bound on the kernel's IP and Cosine distances.
tests/emu/codes_metric_bound_emu.cpp runs the library's own functions on random and adversarial rows and queries (huge
and tiny magnitudes, subnormals, NaN, +-inf, large offsets, normalised Gaussian, mixed-sign and zero rows, zero and
opposite queries, dims up to 2048 and not multiples of 4) against worst distances around the row's distance, around the
largest worst distance that still prunes, and the special values.  It asserts that a pruned row's distance (summed and
finished in the search kernel's order) is never below the worst distance, that the rows and queries the bound cannot
cover never prune, that L2 code rows are unchanged, and that on U[0,1) and normalised Gaussian data the test rejects
at least half of the rows beyond a median worst distance."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("codes_metric_bound") / "codes_metric_bound_emu")
    r = subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-o", out, os.path.join(EMU, "codes_metric_bound_emu.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_metric_prune_test_never_prunes_an_admissible_row(exe, seed):
    r = subprocess.run([exe, "20000", str(seed)], capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0 and "EMU_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
