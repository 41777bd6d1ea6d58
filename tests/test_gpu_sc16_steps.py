"""sc16 / sc16q11 receivers on the device-resident and pipelined paths (b200_demod_run_device_sc16, run_device_sc16_async,
run_host_sc16_async): frames, buffer results (with the reference's float sums as bit patterns), receiver statistics and Mode A/C
replies against the CPU oracle, the same samples through submit_iq_sc16 + run, repeats, and the arguments that are refused.

The gpu-marked tests also run on the emulated kernels in the tier without a GPU (the last two tests of this file)."""
import numpy as np
import pytest

from oraclelib import Oracle
from paritylib import diff_bufres, diff_frames, diff_stats
from test_gpu_parity import _to_sc16
from readsb_b200 import synth
from readsb_b200.abi import BUFRES_DTYPE

GENS = [synth.config2_stream, synth.config5_stream, synth.mixed_stream, synth.mixed_stream]


def _bits(x: np.float32) -> int:
    return int(np.float32(x).view(np.uint32))


class _Ref:
    """One receiver of the reference: sc16 converter, halo carry and demodulate2400 per buffer (sdr_ifile.c:194-259)."""

    def __init__(self, q11: bool, thr: int = 58):
        self.o, self.q11 = Oracle(thr), q11
        self.halo = np.zeros(326, np.uint16)

    def step(self, iq16: np.ndarray, n_buffers: int, buf_len: int, first_ts: int, continues: bool):
        if not continues:
            self.halo = np.zeros(326, np.uint16)
        frames, bufres = [], []
        for b in range(n_buffers):
            mag, sl, sp = Oracle.convert_sc16(iq16[2 * b * buf_len: 2 * (b + 1) * buf_len], self.q11)
            data = np.concatenate([self.halo, mag])
            f, res = self.o.demodulate(data, buf_len, first_ts + b * buf_len * 5)
            r = np.frombuffer(bytearray(res), dtype=BUFRES_DTYPE).copy()
            r["sum_level"], r["sum_power"] = _bits(sl), _bits(sp)
            frames.append(f); bufres.append(r)
            self.halo = data[buf_len: buf_len + 326].copy()
        return np.concatenate(frames), np.concatenate(bufres)


def _check(d, refs, got_f, got_b):
    for s, ref in enumerate(refs):
        fo, bo = ref
        problems = diff_frames(np.concatenate(got_f[s]), fo) + diff_bufres(np.concatenate(got_b[s]), bo)
        assert not problems, f"receiver {s}: " + "\n".join(problems)


def _device_rows(iq16s, pad=2048):
    """Receiver s's int16 samples at dev + pad + s * stride (16-byte aligned, room for the 1304-byte halo in front)."""
    import devbuf
    n = max(a.size for a in iq16s) * 2
    stride = (n + 4096 + 15) & ~15
    dev = devbuf.zeros(pad + len(iq16s) * stride)
    for s, a in enumerate(iq16s):
        dev[pad + s * stride: pad + s * stride + a.size * 2] = devbuf.to_dev(a.view(np.uint8))
    devbuf.sync()
    return dev, stride, pad


@pytest.mark.gpu
@pytest.mark.parametrize("q11", [False, True])
def test_run_device_sc16_matches_oracle_across_continues_and_a_restart(cuda, q11):
    """Four receivers of different kinds, five blocking calls of two buffers; the third starts every receiver over (zero halo)."""
    from readsb_b200.demod import Demodulator
    S, buf, nb, calls = 4, 16384, 2, 5
    total = buf * nb * calls
    iq16 = [_to_sc16(GENS[s](500 + s, total), q11, s) for s in range(S)]
    dev, stride, pad = _device_rows(iq16)
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb)
    refs = [_Ref(q11) for _ in range(S)]
    want_f = [[] for _ in range(S)]; want_b = [[] for _ in range(S)]
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]
    for c in range(calls):
        cont = c not in (0, 2)
        off = c * nb * buf
        d.run_device_sc16(dev.data_ptr() + pad + off * 4, stride, nb, buf, cont, off * 5, q11)
        for s in range(S):
            got_f[s].append(d.frames(s)); got_b[s].append(d.buffer_results(s))
            f, b = refs[s].step(iq16[s][2 * off: 2 * (off + nb * buf)], nb, buf, off * 5, cont)
            want_f[s].append(f); want_b[s].append(b)
    _check(d, [(np.concatenate(want_f[s]), np.concatenate(want_b[s])) for s in range(S)], got_f, got_b)
    assert sum(len(np.concatenate(f)) for f in got_f) > 100
    for s in range(S):
        problems = diff_stats(d.stats(s), refs[s].o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [2, 3])
@pytest.mark.parametrize("q11", [False, True])
def test_run_device_sc16_async_matches_oracle(cuda, depth, q11):
    """Two or three sc16 steps in flight; a fourth is refused, and so is a wait with nothing in flight."""
    from readsb_b200.demod import DemodError, Demodulator
    S, buf, nb, calls = 4, 16384, 2, 5
    total = buf * nb * calls
    iq16 = [_to_sc16(GENS[s](700 + s, total), q11, 10 + s) for s in range(S)]
    dev, stride, pad = _device_rows(iq16)
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb)
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]

    def collect():
        d.wait()
        for s in range(S):
            got_f[s].append(d.frames(s)); got_b[s].append(d.buffer_results(s))
    flying = 0
    for c in range(calls):
        d.run_device_sc16_async(dev.data_ptr() + pad + c * nb * buf * 4, stride, nb, buf, c > 0, c * nb * buf * 5, q11)
        flying += 1
        if depth == 3 and flying == 3:
            with pytest.raises(DemodError):
                d.run_device_sc16_async(dev.data_ptr() + pad, stride, nb, buf, False, 0, q11)
        if flying == depth:
            collect(); flying -= 1
    while flying:
        collect(); flying -= 1
    with pytest.raises(DemodError):
        d.wait()
    refs = []
    for s in range(S):
        r = _Ref(q11)
        refs.append(r.step(iq16[s], nb * calls, buf, 0, False))
        problems = diff_stats(d.stats(s), r.o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    _check(d, refs, got_f, got_b)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("q11", [False, True])
def test_run_host_sc16_async_matches_oracle(cuda, q11):
    """Pinned slabs with the halo carried between the library's input buffers, then pageable memory with a restart; a uc8 step
    does not give an sc16 step its halo."""
    from readsb_b200.demod import DemodError, Demodulator, PinnedBuffer
    S, buf, nb, calls = 3, 16384, 2, 4
    total = buf * nb * calls
    iq16 = [_to_sc16(GENS[s](800 + s, total), q11, 20 + s) for s in range(S)]
    pin = PinnedBuffer(S * 4 * total)
    host = pin.array.view(np.int16).reshape(S, 2 * total)
    for s in range(S):
        host[s] = iq16[s]
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb)
    with pytest.raises(DemodError):      # nothing to continue from yet
        d.run_host_sc16_async(pin.ptr, 4 * total, nb, buf, True, 0, q11)
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]

    def collect():
        d.wait()
        for s in range(S):
            got_f[s].append(d.frames(s)); got_b[s].append(d.buffer_results(s))
    for c in range(calls):
        d.run_host_sc16_async(pin.ptr + c * nb * buf * 4, 4 * total, nb, buf, c > 0, c * nb * buf * 5, q11)
        if c >= 2:
            collect()
    collect(); collect()
    refs = [_Ref(q11) for _ in range(S)]
    _check(d, [refs[s].step(iq16[s], nb * calls, buf, 0, False) for s in range(S)], got_f, got_b)
    d.close()

    # pageable memory: two steps, then the receivers start over a second later
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb)
    plain = np.ascontiguousarray(host.copy())
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]
    restart_ts = 2 * nb * buf * 5 + 12_000_000
    d.run_host_sc16_async(plain.ctypes.data, 4 * total, nb, buf, False, 0, q11)
    d.run_host_sc16_async(plain.ctypes.data + nb * buf * 4, 4 * total, nb, buf, True, nb * buf * 5, q11)
    d.run_host_sc16_async(plain.ctypes.data, 4 * total, nb, buf, False, restart_ts, q11)
    collect(); collect(); collect()
    refs = []
    for s in range(S):
        r = _Ref(q11)
        f1, b1 = r.step(iq16[s], 2 * nb, buf, 0, False)
        f2, b2 = r.step(iq16[s], nb, buf, restart_ts, False)
        refs.append((np.concatenate([f1, f2]), np.concatenate([b1, b2])))
        problems = diff_stats(d.stats(s), r.o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    _check(d, refs, got_f, got_b)

    # a uc8 step, then an sc16 step that claims to continue it
    iq8 = np.full(S * 2 * nb * buf, 127, np.uint8)
    d.run_host_async(iq8.ctypes.data, 2 * nb * buf, nb, buf, False, 0)
    d.wait()
    with pytest.raises(DemodError):
        d.run_host_sc16_async(plain.ctypes.data, 4 * total, nb, buf, True, nb * buf * 5, q11)
    d.close()
    pin.free()


@pytest.mark.gpu
@pytest.mark.parametrize("q11", [False, True])
def test_modeac_on_the_async_sc16_path(cuda, q11):
    """Mode A/C through run_device_sc16_async: the noise floor of each buffer from its float sums (convert.c:243-249 ->
    demod_2400.c:580-581), three steps of two buffers, two in flight."""
    from readsb_b200.demod import Demodulator
    S, B, BUF, steps = 3, 2, 16384, 3
    n = B * BUF * steps
    iq16 = [_to_sc16(synth.generate(n, seed=80 + s, frames_per_sec=2500.0, df_mask=synth.MODEAC | synth.DF17, n_icao=4, amp=(0.4, 0.95)), q11, 30 + s)
            for s in range(S)]
    dev, stride, pad = _device_rows(iq16)
    d = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B, mode_ac=True)
    got_f = [[] for _ in range(S)]; got_a = [[] for _ in range(S)]

    def harvest(k):
        d.wait()
        for s in range(S):
            got_f[s].append(d.frames(s))
            a = d.modeac(s); a["buffer_idx"] += k * B; got_a[s].append(a)
    for k in range(steps):
        d.run_device_sc16_async(dev.data_ptr() + pad + k * B * BUF * 4, stride, B, BUF, k > 0, k * B * BUF * 5, q11)
        if k >= 1:
            harvest(k - 1)
    harvest(steps - 1)
    for s in range(S):
        fo, _ = Oracle().run_stream_sc16(iq16[s], BUF, q11)
        ao = Oracle().run_stream_ac_sc16(iq16[s], BUF, q11)
        ag = np.concatenate(got_a[s])
        assert len(ao) > 10
        assert not diff_frames(np.concatenate(got_f[s]), fo), f"receiver {s}"
        for f in ("timestamp", "f1_sample", "modeac", "buffer_idx"):
            assert len(ag) == len(ao) and np.array_equal(ag[f], ao[f]), f"receiver {s}: modeac {f}"
        assert d.stats(s)["demod_modeac"] == len(ao)
    d.close()


@pytest.mark.gpu
def test_float_sums_are_added_in_sample_order(cuda):
    """A buffer whose float32 sums depend on the order of the adds: numpy's pairwise sum gives other bits than the reference's
    sequential accumulators, and the library must return the sequential ones."""
    from readsb_b200.demod import Demodulator
    buf = 8192
    rng = np.random.default_rng(4)
    iq16 = rng.integers(-32768, 32768, size=2 * buf).astype(np.int16)
    fI, fQ = iq16[0::2].astype(np.float32) / np.float32(32768), iq16[1::2].astype(np.float32) / np.float32(32768)
    magsq = np.minimum(fI * fI + fQ * fQ, np.float32(1))
    mag = np.sqrt(magsq)
    seq_level, seq_power = np.float32(0), np.float32(0)
    for a, b in zip(mag.tolist(), magsq.tolist()):
        seq_level = np.float32(seq_level + np.float32(a)); seq_power = np.float32(seq_power + np.float32(b))
    _, sl, sp = Oracle.convert_sc16(iq16)
    assert (sl, sp) == (seq_level, seq_power)
    assert np.sum(mag, dtype=np.float32) != seq_level and np.sum(magsq, dtype=np.float32) != seq_power
    dev, stride, pad = _device_rows([iq16])
    d = Demodulator(n_streams=1, buf_samples=buf, max_buffers_per_run=1)
    d.run_device_sc16(dev.data_ptr() + pad, stride, 1, buf, False, 0)
    r = d.buffer_results(0)
    assert int(r["sum_level"][0]) == _bits(seq_level) and int(r["sum_power"][0]) == _bits(seq_power)
    d.close()


@pytest.mark.gpu
def test_repeated_sc16_step_converts_again_and_counts_once(cuda):
    """Dense captures at --preamble-threshold=25 make the first of three sc16 steps in flight outgrow the record pool: it and
    the two behind it are repeated (the converter runs again); every result is still the oracle's and nothing is counted twice."""
    from readsb_b200.demod import Demodulator
    S, buf, calls, thr = 12, 65536, 5, 25
    total = buf * calls
    iq16 = [_to_sc16(synth.generate(total, seed=12000 + s, frames_per_sec=20000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP | synth.MODEAC,
                                    n_icao=8, amp=(0.5, 1.0), p_bit_error=0.3), False, 40 + s) for s in range(S)]
    dev, stride, pad = _device_rows(iq16)
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=1, preamble_threshold=thr, mode_ac=True)
    first_pool = 65536          # records each slot starts with for this shape: max(65536, positions / 16)
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]; got_a = [[] for _ in range(S)]
    rec_alloc = []

    def collect(k):
        d.wait()
        for s in range(S):
            got_f[s].append(d.frames(s)); got_b[s].append(d.buffer_results(s))
            a = d.modeac(s); a["buffer_idx"] += k; got_a[s].append(a)
        rec_alloc.append(d.debug_counters()["rec_alloc"])
    for c in range(calls):
        d.run_device_sc16_async(dev.data_ptr() + pad + c * buf * 4, stride, 1, buf, c > 0, c * buf * 5)
        if c >= 2:
            collect(c - 2)
    collect(calls - 2); collect(calls - 1)
    assert rec_alloc[0] > first_pool, rec_alloc        # the first step could only finish in a grown pool
    for s in range(S):
        r = _Ref(False, thr)
        fo, bo = r.step(iq16[s], calls, buf, 0, False)
        problems = diff_frames(np.concatenate(got_f[s]), fo) + diff_bufres(np.concatenate(got_b[s]), bo) + diff_stats(d.stats(s), r.o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
        ao = Oracle(thr).run_stream_ac_sc16(iq16[s], buf)
        ag = np.concatenate(got_a[s])
        assert len(ag) == len(ao) and np.array_equal(ag["timestamp"], ao["timestamp"]) and np.array_equal(ag["buffer_idx"], ao["buffer_idx"])
        assert d.stats(s)["demod_modeac"] == len(ao)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("q11", [False, True])
def test_full_size_step_equals_the_submit_path(cuda, q11):
    """256 receivers x 8 buffers x 65536 samples in one run_device_sc16_async step, array for array equal to the same samples
    fed through submit_iq_sc16 + run; receivers 0-3 also against the oracle."""
    import devbuf
    from readsb_b200.demod import Demodulator
    S, K, BUF = 256, 8, 65536
    n = K * BUF
    kinds = [_to_sc16(GENS[k % 4](900 + k, n), q11, 50 + k) for k in range(8)]      # receiver s gets capture s % 8
    pad, stride = 2048, n * 4 + 4096
    dev = devbuf.zeros(pad + S * stride)
    dk = [devbuf.to_dev(a.view(np.uint8)) for a in kinds]
    for s in range(S):
        dev[pad + s * stride: pad + s * stride + 4 * n] = dk[s % 8]
    devbuf.sync()
    a = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=K)
    a.run_device_sc16_async(dev.data_ptr() + pad, stride, K, BUF, False, 0, q11)
    a.wait()
    b = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=K)
    for k in range(K):
        for s in range(S):
            b.submit_iq_sc16(s, kinds[s % 8][2 * k * BUF: 2 * (k + 1) * BUF], k * BUF * 5, q11)
    b.run()
    for s in range(S):
        fa, fb = a.frames(s), b.frames(s)
        ba, bb = a.buffer_results(s), b.buffer_results(s)
        assert fa.tobytes() == fb.tobytes() and ba.tobytes() == bb.tobytes() and a.stats(s) == b.stats(s), f"receiver {s}"
    for s in range(4):
        r = _Ref(q11)
        fo, bo = r.step(kinds[s], K, BUF, 0, False)
        problems = diff_frames(a.frames(s), fo) + diff_bufres(a.buffer_results(s), bo) + diff_stats(a.stats(s), r.o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    assert sum(len(a.frames(s)) for s in range(8)) > 1000
    a.close(); b.close()


@pytest.mark.gpu
def test_sc16_steps_refuse_bad_arguments(cuda):
    from readsb_b200.demod import DemodError, Demodulator
    S, buf, nb = 2, 8192, 2
    iq16 = [_to_sc16(synth.mixed_stream(60 + s, nb * buf), False, s) for s in range(S)]
    dev, stride, pad = _device_rows(iq16)
    base = dev.data_ptr() + pad
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb)
    bad = [
        (base + 4, stride, nb, buf),               # d_iq not 16-byte aligned
        (base, stride + 4, nb, buf),               # stride not 16-byte aligned
        (base, stride, nb, buf - 4),               # buf_len not a multiple of 8
        (base, stride, nb + 1, buf),               # more buffers than max_buffers_per_run
        (base, stride, 1, buf + 8),                # longer than buf_samples
        (base, nb * buf * 4 - 16, nb, buf),        # rows overlap: 4 bytes per sample
    ]
    for args in bad:
        for call in (d.run_device_sc16, d.run_device_sc16_async):
            with pytest.raises(DemodError):
                call(*args, False, 0)
    host = np.ascontiguousarray(np.stack(iq16))
    with pytest.raises(DemodError):
        d.run_host_sc16_async(host.ctypes.data, 4 * nb * buf, nb, buf - 4, False, 0)
    with pytest.raises(DemodError):
        d.run_host_sc16_async(host.ctypes.data, 4 * nb * buf - 16, nb, buf, False, 0)
    d.submit_iq_sc16(0, iq16[0][: 2 * buf], 0)
    with pytest.raises(DemodError):            # host submits are pending
        d.run_host_sc16_async(host.ctypes.data, 4 * nb * buf, nb, buf, False, 0)
    d.run()
    # after the refusals the context still works
    d.run_host_sc16_async(host.ctypes.data, 4 * nb * buf, nb, buf, False, 0)
    d.wait()
    fo, _ = Oracle().run_stream_sc16(iq16[1], buf)
    assert not diff_frames(d.frames(1), fo)
    d.close()


def test_sc16_steps_on_emulated_kernels():
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_sc16_steps.py", select="not full_size")


def test_sc16_steps_on_emulated_kernels_under_address_sanitizer():
    """Redzones around every "device" allocation: the converter reads no raw sample and writes no magnitude or sum outside
    its receiver's rows."""
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_sc16_steps.py", select="not full_size", sanitize="address")
