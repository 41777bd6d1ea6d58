import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def _cuda_available() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def emulated() -> bool:
    """B200_EMU=1: the gpu-marked tests run against the kernels' source compiled for the CPU under the SIMT emulator
    (tests/emu/, test infrastructure; see tests/test_emu_kernels.py) instead of the sm_90a library on a GPU."""
    return os.environ.get("B200_EMU") == "1"


@pytest.fixture(scope="session")
def cuda():
    if emulated():
        sys.path.insert(0, str(ROOT / "tests" / "emu"))
        import build_emu
        # B200_EMU_LIB: an instrumented build of the emulated library (e.g. AddressSanitizer, tests/emu/README.md)
        os.environ["B200_DEMOD_LIB"] = os.environ.get("B200_EMU_LIB") or str(build_emu.build())
        return True
    if not _cuda_available():
        pytest.skip("no CUDA device")
    return True
