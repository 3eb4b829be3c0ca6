import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the product refuses to load the SIMT-emulated test build of the engine unless the test-suite says so (inherited by
# the subprocesses some tests start)
os.environ["B200NB_TEST_EMULATOR"] = "1"
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _gpu_usable():
    """True on a CUDA box, or when B200NB_LIB points at the SIMT-emulated test build (then `-m gpu` runs on the CPU)."""
    if "libb200nb_emu" in os.path.basename(os.environ.get("B200NB_LIB", "")):
        return True
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """A plain `pytest` on a box without a GPU must end green: gpu-marked tests are skipped there (they are NOT skipped
    on a CUDA box whose engine library is missing -- that has to fail loudly)."""
    if _gpu_usable():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (run on an H100: pytest -m gpu)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure): built on demand from oracle/nbglm_oracle.c."""
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def engine():
    """The product engine (libb200nb.so through the C ABI); fails loudly if missing."""
    import deseq2_b200
    from deseq2_b200 import wrappers
    deseq2_b200.lib()
    return wrappers


@pytest.fixture(scope="module")
def emu(oracle):
    """deseq2_b200.wrappers bound, for the duration of one test module, to the EMULATED engine: the product's CUDA
    sources compiled by g++ against tests/simt_emu/ and executed on CPU fibers (test infrastructure, see
    tests/test_emulated_kernels.py).  The product itself never loads this library."""
    import ctypes as C
    sys.path.insert(0, os.path.join(ROOT, "tests", "simt_emu"))
    import build_emu
    from deseq2_b200 import _lib, wrappers
    lib = C.CDLL(build_emu.build())
    for name, argt in _lib.SIGNATURES.items():
        f = getattr(lib, name)
        f.argtypes = argt
        f.restype = _lib._RESTYPE.get(name, C.c_int)
    saved = _lib._lib
    _lib._lib = lib
    try:
        yield wrappers
    finally:
        _lib._lib = saved


@pytest.fixture(autouse=True, scope="session")
def _emulated_streams():
    """With B200NB_LIB=<emulated engine> the whole `-m gpu` suite runs on the CPU: there is no CUDA stream to pass."""
    from helpers import EMULATED
    if EMULATED:
        import ctypes as C
        from deseq2_b200 import device, device_pipeline
        device._stream = device_pipeline._stream = lambda: C.c_void_p(0)
    yield
