#!/bin/bash
# Everything that can be checked without a GPU, in one go (about 10 minutes on 8 cores):
#   build (nvcc cross-compile for sm_90a, oracle, reference pair), the not-gpu tier (which includes the emulated kernels under the
#   gpu-marked tests, ASan, UBSan, two random schedules, allocation-fault injection), a fuzz campaign, the instruction model.
set -e
cd "$(dirname "$0")/.."
python __graft_entry__.py
python -m pytest tests -x -q -m "not gpu"
python tools/emu_fuzz.py --seed "${1:-1}" --cases "${2:-500}"
python tools/scan_model.py cfg2 | tail -14
