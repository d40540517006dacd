import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped when no CUDA device is visible, so a plain `pytest tests/` works
    on the CPU build container as well as `-m "not gpu"`."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def emu():
    """Host emulation of the kernels' arithmetic (tests/emu), built on demand with g++."""
    import ctypes
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu.cpp")
    core = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_core.cuh")
    stale = (not os.path.exists(so)) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core))
    if stale:
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    from helpers import set_emu_sigs
    return set_emu_sigs(ctypes.CDLL(so))
