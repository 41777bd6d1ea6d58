"""The CUDA library against the reference's own verdicts on the crafted captures of tests/golden/verdicts/verdicts.npz (see
tests/golden/make_verdicts.py and tests/test_verdicts.py): every accept and reject branch of the demodulator, the filter generations,
frames on the skip, on buffer edges and on the kernels' chunk / tile / sub-range boundaries, and exact ties of the pre-check, the
correlator thresholds and the bit slicers.  Frames, signal levels, per-buffer counters and receiver statistics must equal what the
reference returned, on every entry path:

- one receiver through submit_iq + run, whole buffers per run (K = 8) and one buffer per run (K = 1: stage B sub-ranges of a
  65536-sample buffer); Beast bytes, verbatim and corrected, against the oracle's encoder over the reference's frames;
- three receivers with the same capture (the many-receiver stage B);
- submit_mag for the magnitude captures, including a buffer handed over with a zero halo;
- run_device, run_device_async and run_host_async at depth 3;
- run_device_rx with four receivers whose descriptors carry the option sets' thresholds in one step;
- a context with Mode A/C, whose Mode S results must not change.

The gpu-marked tests also run on the emulated kernels in the tier without a GPU (the last two tests of this file)."""
import numpy as np
import pytest

from oraclelib import Oracle
from test_verdicts import CAPTURES, compare, fixture, mag_buffers
from readsb_b200.abi import FORMAT_UC8, RX_CONTINUES, RX_STEP_DTYPE

NFIX_FIXDF = [0, 1, 2, 3]                  # option sets that differ in nfix_crc / fixDF (threshold 58)
THRESHOLDS = [0, 4, 5, 6]                  # option sets with nfix_crc 1, fixDF 1 and thresholds 58, 40, 75, 400


def _demod(cap, o, **kw):
    from readsb_b200.demod import Demodulator
    F = fixture()
    return Demodulator(buf_samples=F.buf(cap), **F.kwargs(cap, o), **kw)


def _with_sigpow(frames, levels):
    """The reference's frames with the exact power sum behind each signal level (the Beast signal byte is taken from it)."""
    f = frames.copy()
    f["sigpow_sum"] = np.rint(levels * 65535.0 * 65535.0 * f["signal_len"]).astype(np.uint64)
    assert np.array_equal(f["sigpow_sum"] / 65535.0 / 65535.0 / f["signal_len"], levels)
    return f


def _check(got_frames, got_bufres, stats, cap, kind, o, what=""):
    problems = compare(np.concatenate(got_frames), np.concatenate(got_bufres), stats, fixture().want(cap, kind, o))
    assert not problems, f"{what}: " + "\n".join(problems)


@pytest.mark.gpu
@pytest.mark.parametrize("o", range(7))
@pytest.mark.parametrize("cap", CAPTURES)
def test_submit_iq_whole_buffers_and_beast_bytes(cuda, cap, o):
    """Eight buffers per run.  Beast records of each run, verbatim and corrected, are the oracle's encoding of the reference's frames."""
    F = fixture()
    K, L = 8, F.buf(cap)
    iq = F.capture(cap, "uc8")
    d = _demod(cap, o, max_buffers_per_run=K)
    fs, bs, beast = [], [], {True: b"", False: b""}
    nb = iq.size // 2 // L
    for b0 in range(0, nb, K):
        for b in range(b0, min(b0 + K, nb)):
            d.submit_iq(0, iq[2 * b * L: 2 * (b + 1) * L], b * L * 5)
        d.run()
        fs.append(d.frames(0)); bs.append(d.buffer_results(0))
        for v in (True, False):
            beast[v] += d.beast(0, verbatim=v)
    _check(fs, bs, d.stats(0), cap, "uc8", o)
    wf, wl = fixture().want(cap, "uc8", o)[:2]
    ref = _with_sigpow(wf, wl)
    assert beast[True] == Oracle.beast(ref, verbatim=True) and beast[False] == Oracle.beast(ref)
    assert len(wf) > 0 and (o != 0 or wf["correctedbits"].any() or cap == "c")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("o", NFIX_FIXDF)
@pytest.mark.parametrize("cap", ["b", "c"])
def test_submit_iq_one_buffer_per_run(cuda, cap, o):
    """One buffer per run: a 65536-sample buffer is resolved in sub-ranges of whole tiles (redone when a skip reaches across)."""
    F = fixture()
    d = _demod(cap, o, max_buffers_per_run=1)
    f, b = d.replay(F.capture(cap, "uc8"))
    _check([f], [b], d.stats(0), cap, "uc8", o)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("o", NFIX_FIXDF)
@pytest.mark.parametrize("cap", ["a", "c"])
def test_three_receivers(cuda, cap, o):
    F = fixture()
    K, L = 4, F.buf(cap)
    iq = F.capture(cap, "uc8")
    d = _demod(cap, o, n_streams=3, max_buffers_per_run=K)
    got = [([], []) for _ in range(3)]
    nb = iq.size // 2 // L
    for b0 in range(0, nb, K):
        for s in range(3):
            for b in range(b0, min(b0 + K, nb)):
                d.submit_iq(s, iq[2 * b * L: 2 * (b + 1) * L], b * L * 5)
        d.run()
        for s in range(3):
            got[s][0].append(d.frames(s)); got[s][1].append(d.buffer_results(s))
    for s in range(3):
        _check(*got[s], d.stats(s), cap, "uc8", o, f"receiver {s}")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("o", range(7))
@pytest.mark.parametrize("cap", CAPTURES)
def test_submit_mag(cuda, cap, o):
    """Magnitudes handed over with their halo (a zero one where the capture restarts): the exact ties reach the kernels unchanged."""
    F = fixture()
    K = 8 if cap != "c" else 2
    d = _demod(cap, o, max_buffers_per_run=K)
    fs, bs, pending = [], [], 0
    bufs = list(mag_buffers(F.capture(cap, "mag"), F.buf(cap), F.restart(cap, "mag")))
    for i, (data, n, ts, sl, sp) in enumerate(bufs):
        d.submit_mag(0, data, n, ts)
        pending += 1
        if pending == K or i == len(bufs) - 1:
            d.run()
            fs.append(d.frames(0)); bs.append(d.buffer_results(0))
            pending = 0
    _check(fs, bs, d.stats(0), cap, "mag", o)
    d.close()


def _device_slab(iq, L, b0, n):
    """A step's buffers in device memory with the 326 samples before them in front (what a continuing step's halo is read from)."""
    import devbuf
    pad = 2048
    dev = devbuf.zeros(pad + n * L * 2)
    if b0 > 0:
        dev[pad - 652: pad] = devbuf.to_dev(np.ascontiguousarray(iq[2 * (b0 * L - 326): 2 * b0 * L]))
    dev[pad: pad + n * L * 2] = devbuf.to_dev(np.ascontiguousarray(iq[2 * b0 * L: 2 * (b0 + n) * L]))
    devbuf.sync()
    return dev, dev.data_ptr() + pad


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "device_async", "host_async"])
@pytest.mark.parametrize("cap", ["a", "c"])
def test_device_and_pipelined_paths(cuda, cap, path):
    F = fixture()
    K, L, depth = (8, F.buf(cap), 3) if cap == "a" else (2, F.buf(cap), 3)
    iq = F.capture(cap, "uc8")
    d = _demod(cap, 0, max_buffers_per_run=K)
    fs, bs, keep, flying = [], [], [], 0
    nb = iq.size // 2 // L

    def harvest():
        if path != "device":
            d.wait()
        fs.append(d.frames(0)); bs.append(d.buffer_results(0))

    for b0 in range(0, nb, K):
        n = min(K, nb - b0)
        if path == "host_async":
            host = np.ascontiguousarray(iq[2 * b0 * L: 2 * (b0 + n) * L]); keep.append(host)
            d.run_host_async(host.ctypes.data, n * L * 2, n, L, b0 > 0, b0 * L * 5)
        else:
            dev, ptr = _device_slab(iq, L, b0, n); keep.append(dev)
            (d.run_device if path == "device" else d.run_device_async)(ptr, n * L * 2, n, L, b0 > 0, b0 * L * 5)
        if path == "device":
            harvest()
        else:
            flying += 1
            if flying == depth:
                harvest(); flying -= 1
    while flying:
        harvest(); flying -= 1
    _check(fs, bs, d.stats(0), cap, "uc8", 0, path)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["a", "c"])
def test_rx_step_thresholds_per_receiver(cuda, cap):
    """run_device_rx: four receivers of one context (threshold 58) carry the thresholds 58, 40, 75 and 400 in their descriptors."""
    import devbuf
    F = fixture()
    K, L = (8, F.buf(cap)) if cap == "a" else (2, F.buf(cap))
    iq = F.capture(cap, "uc8")
    S = len(THRESHOLDS)
    d = _demod(cap, 0, n_streams=S, max_buffers_per_run=K)
    got = [([], []) for _ in range(S)]
    nb = iq.size // 2 // L
    for b0 in range(0, nb, K):
        n = min(K, nb - b0)
        stride = (n * L * 2 + 2048 + 15) & ~15
        pad = 2048
        dev = devbuf.zeros(pad + S * stride)
        for s in range(S):
            lo = pad + s * stride
            if b0 > 0:
                dev[lo - 652: lo] = devbuf.to_dev(np.ascontiguousarray(iq[2 * (b0 * L - 326): 2 * b0 * L]))
            dev[lo: lo + n * L * 2] = devbuf.to_dev(np.ascontiguousarray(iq[2 * b0 * L: 2 * (b0 + n) * L]))
        devbuf.sync()
        rx = np.zeros(S, RX_STEP_DTYPE)
        for s, o in enumerate(THRESHOLDS):
            rx[s] = (b0 * L * 5, n, RX_CONTINUES if b0 > 0 else 0, F.options[o][0], 0)
        d.run_device_rx(FORMAT_UC8, dev.data_ptr() + pad, stride, L, rx)
        for s in range(S):
            got[s][0].append(d.frames(s)); got[s][1].append(d.buffer_results(s))
    for s, o in enumerate(THRESHOLDS):
        _check(*got[s], d.stats(s), cap, "uc8", o, f"threshold {F.options[o][0]}")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["a", "c"])
def test_mode_ac_context_keeps_the_mode_s_verdicts(cuda, cap):
    F = fixture()
    d = _demod(cap, 0, max_buffers_per_run=8 if cap == "a" else 2, mode_ac=True)
    f, b, _ = d.replay(F.capture(cap, "uc8"), want_modeac=True)
    st = d.stats(0)
    _check([f], [b], st, cap, "uc8", 0)
    d.close()


# ---- without a GPU -----------------------------------------------------------------------------------------------------------------
def test_verdicts_on_emulated_kernels():
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_verdicts.py", timeout=1800)


def test_verdicts_on_emulated_kernels_under_address_sanitizer():
    """Redzones around every "device" allocation while the kernels take every accept and reject branch and the boundary cases."""
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_verdicts.py", sanitize="address", timeout=3000)
