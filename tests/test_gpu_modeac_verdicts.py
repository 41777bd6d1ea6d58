"""The CUDA library's Mode A/C path against the reference's own verdicts on the crafted captures of
tests/golden/verdicts/modeac_verdicts.npz (see tests/golden/make_modeac_verdicts.py and tests/test_modeac_verdicts.py): every
accept and reject branch of demodulate2400AC, exact ties of its comparisons, every clock phase, noise floors that wrap or vanish,
and replies on buffer, skip and scan-tile edges.  Replies (timestamp, f1_sample, code, buffer), stats()["demod_modeac"], the Mode S
frames of the same buffers and the Beast bytes (verbatim and corrected) must be the reference's, on every entry path:

- submit_mag with the caller's mean_level / mean_power, and with the buffers' own sums;
- submit_iq + run, eight buffers per run and one; three receivers;
- run_device, run_device_async and run_host_async at depth 3;
- run_device_rx with a receiver that is absent from every other step, and a restart;
- submit_iq_sc16 + run and run_device_sc16 (the noise floor from the converter's float sums).

The gpu-marked tests also run on the emulated kernels in the tier without a GPU (the last two tests of this file)."""
import numpy as np
import pytest

from oraclelib import Oracle
from paritylib import diff_frames
from test_modeac_verdicts import diff_replies, fixture, mag_buffers
from test_verdicts import FRAME_FIELDS
from readsb_b200.abi import FORMAT_UC8, RX_CONTINUES, RX_STEP_DTYPE

HALO = 326
PLACEMENT = ["c65536", "c100", "c300", "c400", "c1000", "c8191", "c20000", "cbig"]
DEVICE_CAPS = ["c65536", "c400", "c1000", "c20000"]        # buffer lengths that are multiples of 8 (what the device paths take)


def _demod(cap, K, **kw):
    from readsb_b200.demod import Demodulator
    return Demodulator(buf_samples=fixture().buf(cap), max_buffers_per_run=K, mode_ac=True, **kw)


def _with_sigpow(frames, levels):
    f = frames.copy()
    f["sigpow_sum"] = np.rint(levels * 65535.0 * 65535.0 * f["signal_len"]).astype(np.uint64)
    assert np.array_equal(f["sigpow_sum"] / 65535.0 / 65535.0 / f["signal_len"], levels)
    return f


class Got:
    """One receiver's results, run by run: replies with a running buffer index, Mode S frames, Beast bytes."""

    def __init__(self):
        self.ac, self.frames, self.beast, self.nbuf = [], [], {True: b"", False: b""}, 0

    def take(self, d, s, n_buffers, beast=True):
        a = d.modeac(s)
        a["buffer_idx"] += self.nbuf
        self.ac.append(a)
        self.frames.append(d.frames(s))
        if beast:
            for v in (True, False):
                self.beast[v] += d.beast(s, verbatim=v)
        self.nbuf += n_buffers

    def check(self, d, s, cap, kind, beast=True, what=""):
        wf, wl, wa, wn = fixture().want(cap, kind)
        ac = np.concatenate(self.ac)
        problems = diff_replies(ac, wa) + diff_frames(np.concatenate(self.frames), wf, fields=FRAME_FIELDS)
        assert not problems, f"{what} {cap}/{kind}: " + "\n".join(problems)
        assert np.array_equal(np.bincount(ac["buffer_idx"].astype(np.int64), minlength=len(wn)), wn)
        assert d.stats(s)["demod_modeac"] == len(wa), what
        if beast:
            ref = _with_sigpow(wf, wl)
            assert self.beast[True] == Oracle.beast(ref, wa, verbatim=True) and self.beast[False] == Oracle.beast(ref, wa), what


def _runs(cap, K):
    """Buffer ranges of the runs: K at a time, and a new run at every buffer that starts with a zero halo."""
    F = fixture()
    nb = F.capture(cap, "uc8").size // 2 // F.buf(cap)
    out, b0 = [], 0
    while b0 < nb:
        b1 = min([b0 + K, nb] + [r for r in F.restart(cap) if b0 < r])
        out.append((b0, b1))
        b0 = b1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["a", "b"])
def test_submit_mag_with_given_levels(cuda, cap):
    """Each buffer with the caller's own mean_level / mean_power: the floors the ties are built on, and those that wrap or are NaN."""
    K = 8
    d = _demod(cap, K)
    g, bufs = Got(), list(mag_buffers(cap, "given"))
    for b0 in range(0, len(bufs), K):
        for data, n, ts, ml, mp in bufs[b0: b0 + K]:
            d.submit_mag(0, data, n, ts, ml, mp)
        d.run()
        g.take(d, 0, len(bufs[b0: b0 + K]))
    g.check(d, 0, cap, "given")
    assert cap != "a" or len(fixture().want(cap, "given")[2]) > 60
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["b"] + PLACEMENT)
def test_submit_mag_with_own_sums(cuda, cap):
    """Magnitudes whose noise floor comes from their own sums; the restart buffer is handed over with a zero halo."""
    K = 8 if cap != "cbig" else 1
    d = _demod(cap, K)
    g, bufs = Got(), list(mag_buffers(cap, "mag"))
    for b0 in range(0, len(bufs), K):
        for data, n, ts, _, _ in bufs[b0: b0 + K]:
            d.submit_mag(0, data, n, ts)
        d.run()
        g.take(d, 0, len(bufs[b0: b0 + K]))
    g.check(d, 0, cap, "mag")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap,K", [(c, k) for c in ["a", "b"] + PLACEMENT for k in (8, 1) if c != "cbig" or k == 1])
def test_submit_iq(cuda, cap, K):
    """uc8 I/Q: K buffers of a run form one segment (tiles over many short buffers), restart_stream before a dropped block."""
    F = fixture()
    L, iq = F.buf(cap), F.capture(cap, "uc8")
    d = _demod(cap, K)
    g = Got()
    for b0, b1 in _runs(cap, K):
        if b0 in F.restart(cap):
            d.restart_stream(0)
        for b in range(b0, b1):
            d.submit_iq(0, iq[2 * b * L: 2 * (b + 1) * L], b * L * 5)
        d.run()
        g.take(d, 0, b1 - b0)
    g.check(d, 0, cap, "uc8")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["a", "c65536", "c1000"])
def test_three_receivers(cuda, cap):
    F = fixture()
    L, iq = F.buf(cap), F.capture(cap, "uc8")
    d = _demod(cap, 4, n_streams=3)
    got = [Got() for _ in range(3)]
    for b0, b1 in _runs(cap, 4):
        for s in range(3):
            if b0 in F.restart(cap):
                d.restart_stream(s)
            for b in range(b0, b1):
                d.submit_iq(s, iq[2 * b * L: 2 * (b + 1) * L], b * L * 5)
        d.run()
        for s in range(3):
            got[s].take(d, s, b1 - b0)
    for s in range(3):
        got[s].check(d, s, cap, "uc8", what=f"receiver {s}")
    d.close()


def _device_slab(iq, L, b0, n, continues):
    import devbuf
    pad = 2048
    dev = devbuf.zeros(pad + n * L * 2)
    if continues:
        dev[pad - 2 * HALO: pad] = devbuf.to_dev(np.ascontiguousarray(iq[2 * (b0 * L - HALO): 2 * b0 * L]))
    dev[pad: pad + n * L * 2] = devbuf.to_dev(np.ascontiguousarray(iq[2 * b0 * L: 2 * (b0 + n) * L]))
    devbuf.sync()
    return dev, dev.data_ptr() + pad


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "device_async", "host_async"])
@pytest.mark.parametrize("cap", DEVICE_CAPS)
def test_device_and_pipelined_paths(cuda, cap, path):
    F = fixture()
    K, L, depth = 3, F.buf(cap), 3
    iq = F.capture(cap, "uc8")
    d = _demod(cap, K)
    g, keep, flying = Got(), [], []

    def harvest():
        if path != "device":
            d.wait()
        g.take(d, 0, flying.pop(0))

    for b0, b1 in _runs(cap, K):
        n, cont = b1 - b0, b0 > 0 and b0 not in F.restart(cap)
        if path == "host_async":
            host = np.ascontiguousarray(iq[2 * b0 * L: 2 * b1 * L]); keep.append(host)
            d.run_host_async(host.ctypes.data, n * L * 2, n, L, cont, b0 * L * 5)
        else:
            dev, ptr = _device_slab(iq, L, b0, n, cont); keep.append(dev)
            (d.run_device if path == "device" else d.run_device_async)(ptr, n * L * 2, n, L, cont, b0 * L * 5)
        flying.append(n)
        if path == "device" or len(flying) == depth:
            harvest()
    while flying:
        harvest()
    g.check(d, 0, cap, "uc8", what=path)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cap", DEVICE_CAPS)
def test_rx_steps_with_an_absent_receiver_and_a_restart(cuda, cap):
    """run_device_rx: receiver 0 takes a run every step, receiver 1 the same runs every other step (absent in between, its state
    untouched); both restart where the capture has a zero halo."""
    import devbuf
    F = fixture()
    K, L = 3, F.buf(cap)
    iq = F.capture(cap, "uc8")
    runs = _runs(cap, K)
    d = _demod(cap, K, n_streams=2)
    got = [Got(), Got()]
    stride = (K * L * 2 + 2048 + 15) & ~15
    pad = 2048
    for step in range(2 * len(runs)):
        todo = {0: runs[step] if step < len(runs) else None, 1: runs[step // 2] if step % 2 == 0 else None}
        rx = np.zeros(2, RX_STEP_DTYPE)
        dev = devbuf.zeros(pad + 2 * stride)
        for s, r in todo.items():
            if r is None:
                continue
            b0, b1 = r
            lo = pad + s * stride
            cont = b0 > 0 and b0 not in F.restart(cap)
            if cont:
                dev[lo - 2 * HALO: lo] = devbuf.to_dev(np.ascontiguousarray(iq[2 * (b0 * L - HALO): 2 * b0 * L]))
            dev[lo: lo + (b1 - b0) * L * 2] = devbuf.to_dev(np.ascontiguousarray(iq[2 * b0 * L: 2 * b1 * L]))
            rx[s] = (b0 * L * 5, b1 - b0, RX_CONTINUES if cont else 0, 0, 0)
        devbuf.sync()
        if not rx["n_buffers"].any():
            continue
        d.run_device_rx(FORMAT_UC8, dev.data_ptr() + pad, stride, L, rx)
        for s in (0, 1):
            if rx[s]["n_buffers"]:
                got[s].take(d, s, int(rx[s]["n_buffers"]))
            else:
                assert len(d.modeac(s)) == 0
    for s in (0, 1):
        got[s].check(d, s, cap, "uc8", what=f"receiver {s}")
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sc16", "sc16q11"])
def test_sc16_float_sums(cuda, kind):
    """Noise floors from the converter's float sums, the last buffer's variance below zero: submit_iq_sc16 + run, and run_device_sc16."""
    import devbuf
    F = fixture()
    L, iq16 = F.buf("b"), F.capture("b", kind)
    q11 = kind == "sc16q11"
    nb = iq16.size // 2 // L
    d = _demod("b", 8)
    g = Got()
    for b0 in range(0, nb, 8):
        for b in range(b0, min(b0 + 8, nb)):
            d.submit_iq_sc16(0, iq16[2 * b * L: 2 * (b + 1) * L], b * L * 5, q11)
        d.run()
        g.take(d, 0, min(b0 + 8, nb) - b0)
    g.check(d, 0, "b", kind, what="submit_iq_sc16")
    d.close()
    d = _demod("b", 8)
    g = Got()
    pad = 4096
    for b0 in range(0, nb, 8):
        n = min(b0 + 8, nb) - b0
        dev = devbuf.zeros(pad + n * L * 4)
        if b0:
            dev[pad - 4 * HALO: pad] = devbuf.to_dev(np.ascontiguousarray(iq16[2 * (b0 * L - HALO): 2 * b0 * L]).view(np.uint8))
        dev[pad: pad + n * L * 4] = devbuf.to_dev(np.ascontiguousarray(iq16[2 * b0 * L: 2 * (b0 + n) * L]).view(np.uint8))
        devbuf.sync()
        d.run_device_sc16(dev.data_ptr() + pad, n * L * 4, n, L, b0 > 0, b0 * L * 5, q11)
        g.take(d, 0, n)
    g.check(d, 0, "b", kind, what="run_device_sc16")
    d.close()


@pytest.mark.gpu
def test_device_steps_of_buffers_shorter_than_the_halo_are_refused(cuda):
    """The buffer after one shorter than the halo starts with a zero halo (what the 100- and 300-sample captures check on the
    submit path); a device step cannot express that, so it takes such buffers one at a time and never continued."""
    import devbuf
    from readsb_b200.demod import DemodError
    d = _demod("c100", 4)
    dev = devbuf.zeros(4096 + 4 * 96 * 2)
    ptr = dev.data_ptr() + 4096
    for n, cont in ((2, False), (1, True), (4, True)):
        with pytest.raises(DemodError):
            d.run_device(ptr, 4 * 96 * 2, n, 96, cont, 0)
    d.run_device(ptr, 96 * 2, 1, 96, False, 0)
    assert len(d.modeac(0)) == 0
    d.close()


# ---- without a GPU -----------------------------------------------------------------------------------------------------------------
def test_modeac_verdicts_on_emulated_kernels():
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_modeac_verdicts.py", timeout=1800)


def test_modeac_verdicts_on_emulated_kernels_under_address_sanitizer():
    """Redzones around every "device" allocation while the Mode A/C kernels take every branch and placement edge."""
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_modeac_verdicts.py", sanitize="address", timeout=3000)
