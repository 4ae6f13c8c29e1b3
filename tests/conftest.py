import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    _ensure_built()


def _ensure_built():
    """A fresh checkout has no build artefacts (they are git-ignored): build the
    product library (nvcc cross-compiles for sm_90a without a GPU) and the oracle
    once, exactly as __graft_entry__.build() does."""
    import shutil
    import subprocess
    lib = os.path.join(ROOT, "cfmmrouter.jl_b200", "libcfmm_b200.so")
    if not os.path.exists(lib) and (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")):
        subprocess.run(["make", "-C", os.path.join(ROOT, "cfmmrouter.jl_b200", "csrc")], check=True,
                       capture_output=True)
    if not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)


def _has_gpu():
    try:
        import ctypes
        n = ctypes.c_int(0)
        rt = ctypes.CDLL("libcudart.so")
        return rt.cudaGetDeviceCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        try:
            import torch
            return torch.cuda.is_available()
        except Exception:
            return False


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a device: on a box without one they are skipped, not failed, so a plain
    `pytest tests` stays green on CPU-only CI."""
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def cr():
    import cfmmrouter_b200
    return cfmmrouter_b200


@pytest.fixture(scope="session")
def synth():
    from cfmmrouter_b200 import synth as s
    return s
