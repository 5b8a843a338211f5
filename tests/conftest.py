import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def emul():
    """Host emulation of the device arithmetic (test-only library, see tests/emul/emul.cpp)."""
    import ctypes
    d = os.path.join(ROOT, "tests", "emul")
    subprocess.check_call(["make", "-C", d, "-s"])
    return ctypes.CDLL(os.path.join(d, "libibft_emul.so"))


@pytest.fixture(scope="session", params=["thread", "quad", "split", "qsplit"])
def engine(request):
    """Every parity test that takes `engine` runs on ALL FOUR recover kernels: one thread per signature (throughput), four
    lanes per signature, chain + helper warps (mid-size latency) and four-lane chains + helper (small-round latency).  Tests that build their own engine
    exercise the AUTO selection."""
    if not has_gpu():
        pytest.skip("no CUDA device")
    import ibft_b200 as ib
    e = ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 24, max_groups=64, max_table_slots=16, max_validators=16384)
    e.set_recover_path({"thread": ib.Engine.PATH_THREAD, "quad": ib.Engine.PATH_QUAD, "split": ib.Engine.PATH_SPLIT, "qsplit": ib.Engine.PATH_QSPLIT}[request.param])
    yield e
    e.close()
