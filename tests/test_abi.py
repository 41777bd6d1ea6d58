"""-m "not gpu": the C-ABI library builds for sm_90a, loads, and exports exactly what include/b200_demod.h declares.
No compute is called here (there is no GPU in this container)."""
import ctypes
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib_path():
    from readsb_b200.build import build_demod
    return build_demod()


def declared_functions():
    text = (ROOT / "include" / "b200_demod.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_demod_\w+)\s*\(", text)))


def test_every_declared_symbol_is_exported(lib_path):
    L = ctypes.CDLL(str(lib_path))
    names = declared_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/b200_demod.h but not exported"
    from readsb_b200.demod import EXPORTED_SYMBOLS
    assert sorted(EXPORTED_SYMBOLS) == names
    assert L.b200_demod_abi_version() == 2


def test_no_internal_symbols_leak(lib_path):
    out = subprocess.run(["nm", "-D", "--defined-only", str(lib_path)], capture_output=True, text=True).stdout
    exported = [ln.split()[-1] for ln in out.splitlines() if " T " in ln]
    assert exported and all(s.startswith("b200_demod_") for s in exported), exported


def test_library_is_sm90a_and_has_no_cpu_path(lib_path):
    out = subprocess.run(["cuobjdump", "-lelf", str(lib_path)], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out
    # nothing under oracle/ is linked into the product
    ldd = subprocess.run(["ldd", str(lib_path)], capture_output=True, text=True).stdout
    assert "oracle" not in ldd and "readsb_ref" not in ldd


def test_struct_layouts_match_header():
    from readsb_b200 import abi
    assert ctypes.sizeof(abi.Frame) == 64 and abi.FRAME_DTYPE.itemsize == 64
    assert ctypes.sizeof(abi.BufferResult) == 112
    assert ctypes.sizeof(abi.Config) == 40
    assert ctypes.sizeof(abi.Stats) == 8 * (4 + 2 + 5 + 5 + 3 + 2 + 2)
    for name, _ in abi.Frame._fields_:
        assert getattr(abi.Frame, name).offset == abi.FRAME_DTYPE.fields[name][1]


def test_create_without_gpu_fails_loudly(lib_path):
    """No silent CPU fallback: without a device, create() returns B200_E_NODEV / raises."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from readsb_b200.demod import DemodError, Demodulator
    with pytest.raises(DemodError):
        Demodulator(n_streams=1)


def test_host_lut_matches_oracle(lib_path):
    """The table the device uses is built by the library's own host code; it must equal the oracle's / reference's."""
    from oraclelib import Oracle
    from readsb_b200.demod import uc8_lut
    assert np.array_equal(uc8_lut(), Oracle.lut())


def test_product_does_not_import_oracle():
    for p in (ROOT / "readsb_b200").rglob("*"):
        if p.name == "build.py":      # build() may compile the checker (it never loads it)
            continue
        if p.suffix in (".py", ".cu", ".cuh", ".h", ".c") and p.is_file():
            text = p.read_text()
            assert "oraclelib" not in text and "modes_oracle" not in text and "libreadsb_ref" not in text, p
