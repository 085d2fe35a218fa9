import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")
    config.addinivalue_line("markers", "gpu_unverified: needs an H100 AND exercises code that has not run on one yet "
                                       "(opt in with COZO_RUN_UNVERIFIED=1; never selected by -m gpu)")


@pytest.fixture(scope="session")
def gpu():
    """Initialise the CUDA library; fails loudly (no CPU fallback) when unusable.

    COZO_EMU_LIB=<libcozo_gpu_emu.so> (tests/emu/build_emu_lib.py) points the binding at the CPU-emulated build of the same
    sources instead: a way to run these very tests without a GPU (tests/test_emu_lib_cpu.py does).  The switch lives
    here, in the test fixture, not in the product's loader."""
    from cozo_b200 import capi
    emu = os.environ.get("COZO_EMU_LIB")
    if emu:
        import ctypes
        assert capi._lib is None, "the real library is already loaded in this process"
        capi.LIB_PATH = os.path.abspath(emu)
        # global scope, so that the pybind11 host module (linked against libcozo_gpu.so) binds to these definitions too
        ctypes.CDLL(capi.LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    capi.init(0)
    return capi
