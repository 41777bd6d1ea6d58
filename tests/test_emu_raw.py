"""tests/test_gpu_raw.py on the emulated kernels (tests/test_emu_kernels.py): the raw / AVR encoder's source run on the CPU, once
as it is and once with AddressSanitizer redzones around every "device" allocation, so that no record is written past the packed
output and no frame, reply or descriptor is read past its array."""
from pathlib import Path

from test_emu_kernels import _run_gpu_tests_emulated

ROOT = Path(__file__).resolve().parent.parent
# the comparison with the reference program's stdout needs oracle/_ref/readsb_cpu (the reference tree at build time)
SELECT = None if (ROOT / "oracle" / "_ref" / "readsb_cpu").exists() else "not readsb_cpu"


def test_raw_output_on_emulated_kernels():
    _run_gpu_tests_emulated("tests/test_gpu_raw.py", select=SELECT)


def test_raw_output_on_emulated_kernels_under_address_sanitizer():
    _run_gpu_tests_emulated("tests/test_gpu_raw.py", select=SELECT, sanitize="address")
