"""The kernels' own source, run on the CPU.

tests/emu/ compiles readsb_b200/csrc/*.cu (kernels and the C-ABI host code, rewritten mechanically: launches, dynamic shared
memory, inline PTX) with g++ against a SIMT emulator — one fiber per CUDA thread, warp collectives and block barriers as
rendezvous points — and the gpu-marked parity tests are then run against that library through the same C ABI and the same
Python mirror.  This is TEST INFRASTRUCTURE: it checks the kernels' logic where no GPU is available (this tier runs without
one) and lets a kernel change be tried before GPU minutes are spent on it.  It is not a product path — the product library is
built by nvcc for sm_90a only, has no CPU path (tests/test_abi.py) and never loads the emulated one — and it says nothing
about performance, memory-ordering races between warps, or anything else that only exists on the hardware: the gpu-marked
tests on an H100 remain the parity tests proper.
"""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _run_gpu_tests_emulated(*modules: str, timeout: int = 900, sanitize: str | None = None, select: str | None = None,
                            sched_seed: int | None = None, extra_env: dict | None = None) -> str:
    env = dict(os.environ, B200_EMU="1", **(extra_env or {}))
    if sched_seed is not None:
        env["B200_EMU_SCHED_SEED"] = str(sched_seed)
    env.pop("B200_DEMOD_LIB", None)
    env.pop("B200_EMU_LIB", None)
    cmd = [sys.executable, "-m", "pytest", *modules, "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"]
    if select:
        cmd += ["-k", select]
    if sanitize:
        sys.path.insert(0, str(ROOT / "tests" / "emu"))
        import build_emu
        env["B200_EMU_LIB"] = str(build_emu.build(sanitize=sanitize))
        env["LD_PRELOAD"] = build_emu.sanitizer_runtime(sanitize)
        env["ASAN_OPTIONS"] = "detect_leaks=0:detect_stack_use_after_return=0"      # fibers switch stacks by hand
        env["UBSAN_OPTIONS"] = "halt_on_error=1:print_stacktrace=0"
        cmd += ["-s"]                                                                # a sanitizer report must reach our pipe
    elif extra_env:
        cmd += ["-s"]                                                                # ... and so must what the library prints when asked to
    res = subprocess.run(cmd, cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=timeout)
    tail = (res.stdout + res.stderr)[-3000:]
    assert res.returncode == 0, "gpu-marked tests failed against the emulated kernels:\n" + tail
    assert " passed" in tail and "skipped" not in tail.splitlines()[-1], tail
    return tail


def test_emulated_library_exports_the_whole_abi():
    import ctypes
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu
    from readsb_b200 import demod
    lib = ctypes.CDLL(str(build_emu.build()))
    for sym in demod.EXPORTED_SYMBOLS:
        getattr(lib, sym)


@pytest.mark.parametrize("module", ["tests/test_gpu_parity.py", "tests/test_gpu_edges.py", "tests/test_gpu_fullsize.py", "tests/test_gpu_shim.py",
                                    "tests/test_gpu_fuzz.py", "tests/test_gpu_emu_semantics.py"])
def test_gpu_parity_suite_on_emulated_kernels(module):
    """test_gpu_shim.py: the whole unmodified reference program linked with integration/readsb_shim.c, its libb200demod.so
    resolved to the emulated library (needs oracle/_ref/readsb_{cpu,b200}, i.e. the reference tree at build time)."""
    if module.endswith("test_gpu_shim.py") and not (ROOT / "oracle" / "_ref" / "readsb_b200").exists():
        pytest.skip("oracle/_ref/readsb_b200 not built")
    _run_gpu_tests_emulated(module)


def test_edge_cases_under_address_sanitizer():
    """Ragged / tiny / empty buffers, unequal receivers, fuzzed buffer sizes, the dense slow path and Mode A/C with odd buffer
    lengths, with redzones around every "device" allocation: no kernel reads or writes past a pool, an arena or a result array."""
    _run_gpu_tests_emulated("tests/test_gpu_edges.py", "tests/test_gpu_fullsize.py", "tests/test_gpu_parity.py", sanitize="address",
                            select="edges or dense_tile or golden or modeac_matches or sc16 or beast_output or magnitude_handoff or has_to_be_repeated or noise_floor")


def test_no_undefined_behaviour_where_cpu_and_gpu_semantics_differ():
    """UBSan over the parity tests: no shift by >= 32, no signed overflow, no misaligned vector access in the kernels' source —
    the constructs C++ leaves undefined and PTX defines, i.e. where an emulated run could disagree with the hardware."""
    _run_gpu_tests_emulated("tests/test_gpu_edges.py", "tests/test_gpu_parity.py", sanitize="undefined")


@pytest.mark.parametrize("seed", [7, 8])
def test_parity_does_not_depend_on_the_order_lanes_and_warps_run_in(seed):
    """The emulator's default schedule runs lane 0 first and warp 0 first; here every scheduling round uses a fresh random order
    of the CTA's fibers (lanes within a warp, warps within the CTA) — code that leans on the default order fails."""
    _run_gpu_tests_emulated("tests/test_gpu_parity.py", "tests/test_gpu_edges.py", sched_seed=seed)


def test_pipelined_session_measures_its_sm_partition_on_a_larger_emulated_chip():
    """The host code that measures a pipelined session's SM partition (demod_api.cu tune_partition) only runs on chips with
    at least 16 SMs: a 20-SM emulated device takes the long-session test through its phases - whole chip, 85 %, 82 %, the
    decision, and the new measurement when the size of the runs changes (the periods themselves mean nothing here) - and the
    asynchronous tests through changing scan grids, all still bit-exact."""
    out = _run_gpu_tests_emulated("tests/test_gpu_parity.py", select="long_pipelined or async_pipeline_matches", extra_env={"B200_EMU_SMS": "20", "B200_SCAN_PART": "2"})
    assert "passed" in out and "b200 partition: 15 tiles" in out and "-> scan grid" in out, out


def test_every_allocation_failure_is_reported_not_fatal():
    """tests/emu/fail_alloc_probe.py: the n-th device / pinned allocation fails, for every n the host code reaches."""
    env = dict(os.environ); env.pop("B200_DEMOD_LIB", None); env.pop("B200_EMU_LIB", None)
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "emu" / "fail_alloc_probe.py")], cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "results equal the oracle's" in res.stdout, (res.stdout + res.stderr)[-2000:]


def test_product_never_refers_to_the_emulator():
    for p in list((ROOT / "readsb_b200").rglob("*.py")) + list((ROOT / "readsb_b200" / "csrc").glob("*")) + list((ROOT / "include").glob("*")) \
            + [ROOT / "bench.py", ROOT / "__graft_entry__.py"]:
        if p.is_file() and p.suffix != ".so":
            text = p.read_text(errors="ignore")
            assert "tests/emu" not in text and "B200_EMU" not in text and "build_emu" not in text, p
