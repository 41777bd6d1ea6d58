"""Pins the SIMT emulator's definitions (tests/emu/, test infrastructure) against the hardware: tests/emu/selftest/selftest.cu
exercises every primitive the emulator provides — shuffles, ballot, REDUX, popc / ffs / clz / brev, funnel shifts, byte_perm,
prmt in sign-replication mode, dp2a.lo / .hi, mad.wide, cp.async, shared / global atomics, __syncthreads, reconvergence at a
__syncwarp — and is valid CUDA: built by nvcc for sm_90a and run on the GPU it must give the results the emulated build gives
(both are checked against the same numpy expectations, written from the CUDA / PTX definitions)."""
import ctypes
import os
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "emu" / "selftest"))

pytestmark = pytest.mark.gpu


def test_emulator_primitives_match_the_hardware(cuda):
    import run_selftest as st
    inp = st.make_input()
    if os.environ.get("B200_EMU") == "1":
        L = ctypes.CDLL(str(st.build()))
        ow = np.zeros(32 * 16, np.uint32); ob = np.zeros(st.NB * st.NT, np.uint32); cnt = np.zeros(1, np.uint32)
        assert L.b200_emu_selftest(inp.ctypes.data, ow.ctypes.data, ob.ctypes.data, cnt.ctypes.data, st.NB, st.NT) == 0
    else:
        import torch
        try:
            lib = st.build_sm90a()
        except (OSError, FileNotFoundError) as e:           # no nvcc on this box: nothing to compare with
            pytest.skip(f"nvcc not available: {e}")
        L = ctypes.CDLL(str(lib))
        L.b200_emu_selftest.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_uint32] * 2
        d_in = torch.from_numpy(inp.view(np.int32)).cuda()
        d_ow = torch.zeros(32 * 16, dtype=torch.int32, device="cuda")
        d_ob = torch.zeros(st.NB * st.NT, dtype=torch.int32, device="cuda")
        d_cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert L.b200_emu_selftest(d_in.data_ptr(), d_ow.data_ptr(), d_ob.data_ptr(), d_cnt.data_ptr(), st.NB, st.NT) == 0
        torch.cuda.synchronize()
        ow, ob, cnt = (t.cpu().numpy().view(np.uint32) for t in (d_ow, d_ob, d_cnt))
    st.check(inp, ow, ob, cnt)
