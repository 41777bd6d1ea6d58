"""Independent receivers in one step (b200_demod_run_device_rx, run_device_rx_async, run_host_rx_async) and restart_stream on the
host-buffer path: every receiver with its own buffer count (absent ones included), timestamps, restarts after a gap and preamble
threshold, against one CPU oracle per receiver; the uniform calls against the same calls with a uniform descriptor array; the
refused arguments.

The gpu-marked tests also run on the emulated kernels in the tier without a GPU (the last two tests of this file)."""
import ctypes

import numpy as np
import pytest

from oraclelib import Oracle
from paritylib import diff_bufres, diff_frames, diff_stats
from test_gpu_parity import _to_sc16
from readsb_b200 import synth
from readsb_b200.abi import BUFRES_DTYPE, FORMAT_SC16, FORMAT_SC16Q11, FORMAT_UC8, MODEAC_DTYPE, RX_CONTINUES, RX_STEP_DTYPE

GENS = [synth.config2_stream, synth.config5_stream, synth.mixed_stream, synth.modeac_stream]
FORMATS = [FORMAT_UC8, FORMAT_SC16, FORMAT_SC16Q11]
CTX_THR = 58


def _bps(fmt):
    return 2 if fmt == FORMAT_UC8 else 4


def _bits(x) -> int:
    return int(np.float32(x).view(np.uint32))


def _capture(fmt, s, n, seed):
    iq8 = GENS[s % 4](seed + s, n)
    return iq8 if fmt == FORMAT_UC8 else _to_sc16(iq8, fmt == FORMAT_SC16Q11, seed + 100 + s)


class _Rx:
    """One receiver of the reference: its own oracle, halo, clock and threshold; Mode A/C on an oracle of its own (as the
    reference runs demodulate2400AC on the same mag_buf, readsb.c:871-874)."""

    def __init__(self, fmt, ttl):
        self.fmt, self.o, self.oa = fmt, Oracle(CTX_THR, icao_ttl_ms=ttl), Oracle(CTX_THR, icao_ttl_ms=ttl)
        self.halo = np.zeros(326, np.uint16)
        self.frames, self.bufres, self.ac, self.nbuf = [], [], [], 0

    def step(self, raw, n, buf, ts, cont, thr):
        if not cont:
            self.halo = np.zeros(326, np.uint16)
            self.o.restart_stream()
        self.o.set_preamble_threshold(thr or CTX_THR)
        for b in range(n):
            if self.fmt == FORMAT_UC8:
                mag, sl, sp = Oracle.convert(raw[2 * b * buf: 2 * (b + 1) * buf])
            else:
                mag, fl, fp = Oracle.convert_sc16(raw[2 * b * buf: 2 * (b + 1) * buf], self.fmt == FORMAT_SC16Q11)
                sl = sp = 0
            data = np.concatenate([self.halo, mag]).astype(np.uint16)
            f, res = self.o.demodulate(data, buf, ts + b * buf * 5, sl, sp)
            r = np.frombuffer(bytearray(res), dtype=BUFRES_DTYPE).copy()
            if self.fmt == FORMAT_UC8:
                a = self.oa.demodulate_ac(data, buf, ts + b * buf * 5, sl, sp)
            else:
                r["sum_level"], r["sum_power"] = _bits(fl), _bits(fp)
                a = self.oa.demodulate_ac_levels(data, buf, ts + b * buf * 5, float(np.float32(fl) / np.float32(buf)), float(np.float32(fp) / np.float32(buf)))
            a["buffer_idx"] = self.nbuf
            self.frames.append(f); self.bufres.append(r); self.ac.append(a)
            self.nbuf += 1
            self.halo = data[buf: buf + 326].copy()


def _plan(rng, S, K, steps, absent_run=(3, 4, 5, 6)):
    """Per step and receiver: (n_buffers, continues, gap, threshold).  Receiver 3 is absent in steps absent_run and then continues."""
    out, started = [], [False] * S
    for k in range(steps):
        row = []
        for s in range(S):
            n = int(rng.integers(0, K + 1))
            if s == 3:
                n = 0 if k in absent_run else max(n, 1)
            gap = started[s] and rng.random() < 0.2      # dropped samples: the clock jumps, the halo is zero
            row.append((n, started[s] and not gap, gap, int(rng.choice([0, 40, 75]))))
            started[s] = started[s] or n > 0
        out.append(row)
    return out


class _Session:
    """Drives one context through a plan on one entry path and checks every receiver against its own oracle."""

    def __init__(self, path, fmt, S=8, K=3, buf=8192, steps=8, depth=2, ttl=60000, mode_ac=False, pinned=False, seed=1, plan=None):
        from readsb_b200.demod import Demodulator
        self.path, self.fmt, self.S, self.K, self.buf, self.depth, self.pinned = path, fmt, S, K, buf, depth, pinned
        rng = np.random.default_rng(seed)
        self.plan = plan or _plan(rng, S, K, steps)
        need = [sum(r[s][0] for r in self.plan) * buf for s in range(S)]
        self.raw = [_capture(fmt, s, max(n, buf), seed * 10) for s, n in enumerate(need)]
        self.d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K, icao_ttl_ms=ttl, mode_ac=mode_ac, preamble_threshold=CTX_THR)
        self.refs = [_Rx(fmt, ttl) for _ in range(S)]
        self.mode_ac = mode_ac
        self.got = [([], [], []) for _ in range(S)]
        self.keep = []

    def _step_input(self, row, cursors, clock):
        S, buf, bps = self.S, self.buf, _bps(self.fmt)
        rx = np.zeros(S, RX_STEP_DTYPE)
        maxn = max(r[0] for r in row)
        stride = (max(maxn, 1) * buf * bps + 2048 + 15) & ~15
        parts = []
        for s, (n, cont, gap, thr) in enumerate(row):
            if gap:
                clock[s] += 12_000_000 + 4096 * 5      # a second and a dropped block later
            rx[s] = (clock[s], n, RX_CONTINUES if cont else 0, thr, 0)
            parts.append(self.raw[s][2 * cursors[s]: 2 * (cursors[s] + n * buf)])
        return rx, stride, parts

    def run(self):
        S, buf, bps = self.S, self.buf, _bps(self.fmt)
        d = self.d
        cursors, clock = [0] * S, [1000 * s for s in range(S)]
        flying = 0
        for k, row in enumerate(self.plan):
            rx, stride, parts = self._step_input(row, cursors, clock)
            if self.path == "host":
                pitch = max(max(r[0] for r in row), 1) * buf * bps
                if self.pinned:
                    from readsb_b200.demod import PinnedBuffer
                    pb = PinnedBuffer(S * pitch); self.keep.append(pb)
                    host, ptr = pb.array, pb.ptr
                else:
                    host = np.zeros(S * pitch, np.uint8); self.keep.append(host); ptr = host.ctypes.data
                for s, p in enumerate(parts):
                    host[s * pitch: s * pitch + p.nbytes] = p.view(np.uint8)
                d.run_host_rx_async(self.fmt, ptr, pitch, buf, rx)
            else:
                import devbuf
                pad = 2048
                dev = devbuf.zeros(pad + S * stride); self.keep.append(dev)
                junk = np.random.default_rng(k).integers(0, 256, size=326 * bps, dtype=np.uint8)
                for s, p in enumerate(parts):
                    lo = pad + s * stride
                    if row[s][0]:
                        # the halo in front: the receiver's previous samples when it continues, junk after a restart (never read)
                        prev = self.raw[s][2 * (cursors[s] - 326): 2 * cursors[s]].view(np.uint8) if row[s][1] and cursors[s] >= 326 else junk
                        dev[lo - 326 * bps: lo] = devbuf.to_dev(np.ascontiguousarray(prev))
                        dev[lo: lo + p.nbytes] = devbuf.to_dev(np.ascontiguousarray(p.view(np.uint8)))
                devbuf.sync()
                ptr = dev.data_ptr() + pad
                if self.path == "device":
                    d.run_device_rx(self.fmt, ptr, stride, buf, rx)
                    self._harvest(row)
                else:
                    d.run_device_rx_async(self.fmt, ptr, stride, buf, rx)
            for s, (n, cont, gap, thr) in enumerate(row):
                if n:
                    self.refs[s].step(parts[s], n, buf, int(rx[s]["first_sample_timestamp"]), cont, thr)
                    cursors[s] += n * buf
                    clock[s] += n * buf * 5
            if self.path != "device":
                self._rows = getattr(self, "_rows", []) + [row]
                flying += 1
                if flying == self.depth:
                    self._harvest(self._rows.pop(0)); flying -= 1
        while self.path != "device" and flying:
            self._harvest(self._rows.pop(0)); flying -= 1
        return self

    def _harvest(self, row):
        d = self.d
        if self.path != "device":
            d.wait()
        for s in range(self.S):
            f, b = d.frames(s), d.buffer_results(s)
            if row[s][0] == 0:
                assert len(f) == 0 and len(b) == 0, f"absent receiver {s} has results"
            assert len(b) == row[s][0]
            self.got[s][0].append(f); self.got[s][1].append(b)
            if self.mode_ac:
                a = d.modeac(s)
                a["buffer_idx"] += sum(len(x) for x in self.got[s][1][:-1])
                self.got[s][2].append(a)
            if not self.mode_ac and len(f):      # (the frames themselves are checked against the oracle in check())
                assert d.beast(s) == Oracle.beast(f), f"receiver {s}: Beast bytes"

    def check(self, min_frames=50):
        total = 0
        for s in range(self.S):
            ref = self.refs[s]
            fo = np.concatenate(ref.frames) if ref.frames else np.zeros(0, self.got[s][0][0].dtype)
            bo = np.concatenate(ref.bufres) if ref.bufres else np.zeros(0, BUFRES_DTYPE)
            fg, bg = np.concatenate(self.got[s][0]), np.concatenate(self.got[s][1])
            problems = diff_frames(fg, fo) + diff_bufres(bg, bo) + diff_stats(self.d.stats(s), ref.o.stats())
            assert not problems, f"receiver {s}: " + "\n".join(problems)
            if self.mode_ac:
                ag, ao = np.concatenate(self.got[s][2]), (np.concatenate(ref.ac) if ref.ac else np.zeros(0, MODEAC_DTYPE))
                for f in ("timestamp", "f1_sample", "modeac", "buffer_idx"):
                    assert len(ag) == len(ao) and np.array_equal(ag[f], ao[f]), f"receiver {s}: modeac {f}"
            total += len(fg)
        assert total >= min_frames, total
        self.d.close()
        return total


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("path", ["device", "device_async", "host"])
def test_independent_receivers_match_their_oracles(cuda, path, fmt):
    """Eight receivers of different generators: counts 0 .. 3 from step to step, receiver 3 absent for four steps and then
    continuing, clock jumps with a zero halo, thresholds 0 / 40 / 75 mixed within each step."""
    _Session(path, fmt, seed=3 + fmt).run().check()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device_async", "host"])
def test_receivers_flip_their_filters_at_different_buffers(cuda, path):
    """A 10 ms filter period: each receiver's flips follow its own clock."""
    s = _Session(path, FORMAT_UC8, ttl=10, seed=21).run()
    flips = [int(np.concatenate(g[1])["icao_flipped"].sum()) for g in s.got]
    s.check()
    assert min(flips) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [FORMAT_UC8, FORMAT_SC16])
@pytest.mark.parametrize("depth", [2, 3])
@pytest.mark.parametrize("pinned", [False, True])
def test_pipelined_host_rx_steps(cuda, fmt, depth, pinned):
    _Session("host", fmt, depth=depth, pinned=pinned, seed=40 + depth).run().check()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_modeac_with_independent_receivers(cuda, fmt):
    _Session("device_async", fmt, mode_ac=True, seed=60, S=4).run().check()


@pytest.mark.gpu
def test_one_receiver_solo_path(cuda):
    """One receiver (the single-CTA stage B), absent in some steps."""
    plan = [[(1, False, False, 0)], [(0, True, False, 0)], [(2, True, False, 75)], [(1, False, True, 40)], [(0, True, False, 0)], [(1, True, False, 0)]]
    for path in ("device", "device_async", "host"):
        _Session(path, FORMAT_UC8, S=1, K=2, plan=plan, seed=70).run().check(min_frames=1)


@pytest.mark.gpu
def test_dense_rx_step_is_repeated_with_two_behind_it(cuda):
    """Dense captures at threshold 25 make the first of three steps in flight outgrow the record pool: it and the two behind it
    are repeated; every receiver still matches its oracle and nothing is counted twice."""
    from readsb_b200.demod import Demodulator
    S, buf, K = 12, 65536, 2
    counts = [[1 + (s + k) % 2 if (s + k) % 5 else 0 for s in range(S)] for k in range(4)]
    plan = [[(counts[k][s], any(counts[j][s] for j in range(k)), False, 25) for s in range(S)] for k in range(4)]
    sess = _Session.__new__(_Session)
    sess.path, sess.fmt, sess.S, sess.K, sess.buf, sess.depth, sess.pinned, sess.plan, sess.mode_ac = "device_async", FORMAT_UC8, S, K, buf, 3, False, plan, False
    sess.raw = [synth.generate(K * 4 * buf, seed=12000 + s, frames_per_sec=20000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP, n_icao=8,
                               amp=(0.5, 1.0), p_bit_error=0.3) for s in range(S)]
    sess.d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K, preamble_threshold=CTX_THR)
    sess.refs = [_Rx(FORMAT_UC8, 60000) for _ in range(S)]
    sess.got = [([], [], []) for _ in range(S)]
    sess.keep = []
    rec = []
    orig = sess._harvest

    def harvest(row):
        orig(row)
        rec.append(sess.d.debug_counters()["rec_alloc"])
    sess._harvest = harvest
    sess.run()
    assert rec[0] > 65536, rec
    sess.check()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [FORMAT_UC8, FORMAT_SC16])
def test_full_size_rx_step(cuda, fmt):
    """256 receivers x up to 8 x 65536 samples with random counts (some absent) equals the same receivers' buffers through
    submit_* + run; receivers 0 - 3 also against their oracles."""
    import devbuf
    from readsb_b200.demod import Demodulator
    S, K, BUF = 256, 8, 65536
    rng = np.random.default_rng(5)
    counts = rng.choice([0, 7, 8], size=S, p=[0.05, 0.45, 0.5])
    kinds = [_capture(fmt, k, K * BUF, 900) for k in range(8)]
    bps = _bps(fmt)
    pad, stride = 2048, K * BUF * bps + 4096
    dev = devbuf.zeros(pad + S * stride)
    dk = [devbuf.to_dev(a.view(np.uint8)) for a in kinds]
    for s in range(S):
        dev[pad + s * stride: pad + s * stride + K * BUF * bps] = dk[s % 8]
    devbuf.sync()
    rx = np.zeros(S, RX_STEP_DTYPE)
    for s in range(S):
        rx[s] = (7 * s, counts[s], 0, 0, 0)
    a = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=K)
    a.run_device_rx_async(fmt, dev.data_ptr() + pad, stride, BUF, rx)
    a.wait()
    b = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=K)
    for k in range(K):
        for s in range(S):
            if k < counts[s]:
                chunk = kinds[s % 8][2 * k * BUF: 2 * (k + 1) * BUF]
                if fmt == FORMAT_UC8:
                    b.submit_iq(s, chunk, 7 * s + k * BUF * 5)
                else:
                    b.submit_iq_sc16(s, chunk, 7 * s + k * BUF * 5)
    b.run()
    for s in range(S):
        assert a.frames(s).tobytes() == b.frames(s).tobytes() and a.buffer_results(s).tobytes() == b.buffer_results(s).tobytes() \
            and a.stats(s) == b.stats(s), f"receiver {s}"
    for s in range(4):
        r = _Rx(fmt, 60000)
        r.step(kinds[s], int(counts[s]), BUF, 7 * s, False, 0)
        fo = np.concatenate(r.frames) if r.frames else a.frames(s)[:0]
        problems = diff_frames(a.frames(s), fo) + diff_stats(a.stats(s), r.o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    a.close(); b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("path", ["device", "device_async", "host"])
def test_uniform_descriptors_equal_the_uniform_calls(cuda, path, fmt):
    """A descriptor array with one entry repeated gives what the existing call gives, array for array."""
    import devbuf
    from readsb_b200.demod import Demodulator
    S, K, buf, steps = 4, 2, 8192, 3
    bps = _bps(fmt)
    caps = [_capture(fmt, s, K * buf * steps, 300) for s in range(S)]
    host = np.ascontiguousarray(np.stack([c.view(np.uint8) for c in caps]))
    row = K * buf * bps * steps
    pad = 2048
    dev = devbuf.zeros(pad + S * row + 4096)
    for s in range(S):
        dev[pad + s * row: pad + (s + 1) * row] = devbuf.to_dev(host[s])
    devbuf.sync()
    out = []
    for use_rx in (False, True):
        d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K)
        res = []
        for k in range(steps):
            cont, ts, off = k > 0, k * K * buf * 5, k * K * buf * bps
            rx = np.zeros(S, RX_STEP_DTYPE)
            rx[:] = (ts, K, RX_CONTINUES if cont else 0, 0, 0)
            q11 = fmt == FORMAT_SC16Q11
            if path == "host":
                if use_rx:
                    d.run_host_rx_async(fmt, host.ctypes.data + off, row, buf, rx)
                elif fmt == FORMAT_UC8:
                    d.run_host_async(host.ctypes.data + off, row, K, buf, cont, ts)
                else:
                    d.run_host_sc16_async(host.ctypes.data + off, row, K, buf, cont, ts, q11)
            else:
                ptr = dev.data_ptr() + pad + off
                if use_rx:
                    (d.run_device_rx if path == "device" else d.run_device_rx_async)(fmt, ptr, row, buf, rx)
                elif fmt == FORMAT_UC8:
                    (d.run_device if path == "device" else d.run_device_async)(ptr, row, K, buf, cont, ts)
                else:
                    (d.run_device_sc16 if path == "device" else d.run_device_sc16_async)(ptr, row, K, buf, cont, ts, q11)
            if path != "device":
                d.wait()
            res.append([(d.frames(s).tobytes(), d.buffer_results(s).tobytes()) for s in range(S)])
        res.append([str(d.stats(s)) for s in range(S)])
        out.append(res)
        d.close()
    assert out[0] == out[1]
    assert sum(len(f) for f, _ in out[0][1]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [FORMAT_UC8, FORMAT_SC16])
def test_restart_stream_on_the_submit_path(cuda, fmt):
    """restart_stream before a buffer: that buffer starts with a zero halo, also between two buffers pending in one run."""
    from readsb_b200.demod import Demodulator
    buf, n = 8192, 6
    cap = _capture(fmt, 2, n * buf, 500)
    d = Demodulator(n_streams=2, buf_samples=buf, max_buffers_per_run=3)
    ref = _Rx(fmt, 60000)
    restarts = {2, 4}                  # buffer 2 in the middle of a run of three, buffer 4 at ...
    got_f, got_b = [], []
    for run in range(2):
        for b in range(3 * run, 3 * run + 3):
            if b in restarts:
                d.restart_stream(0)
            chunk = cap[2 * b * buf: 2 * (b + 1) * buf]
            if fmt == FORMAT_UC8:
                d.submit_iq(0, chunk, b * buf * 5)
            else:
                d.submit_iq_sc16(0, chunk, b * buf * 5)
            ref.step(chunk, 1, buf, b * buf * 5, b not in restarts and b > 0, 0)
        d.run()
        got_f.append(d.frames(0)); got_b.append(d.buffer_results(0))
    d.restart_stream(1)                # no effect on a magnitude hand-off
    d.submit_mag(1, np.zeros(326 + buf, np.uint16), buf, 0)
    d.run()
    problems = diff_frames(np.concatenate(got_f), np.concatenate(ref.frames)) + diff_bufres(np.concatenate(got_b), np.concatenate(ref.bufres)) \
        + diff_stats(d.stats(0), ref.o.stats())
    assert not problems, "\n".join(problems)
    assert sum(len(f) for f in got_f) > 10
    d.close()


@pytest.mark.gpu
def test_rx_steps_refuse_bad_arguments(cuda):
    """Every refused argument is refused before anything is enqueued; the next valid step still matches the oracle."""
    from readsb_b200.demod import DemodError, Demodulator
    S, buf, K = 3, 8192, 2
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K)
    caps = [_capture(FORMAT_UC8, s, 2 * K * buf, 600) for s in range(S)]
    host = np.ascontiguousarray(np.stack([c.view(np.uint8) for c in caps]))
    row = host.shape[1]
    good = np.zeros(S, RX_STEP_DTYPE)
    good[:] = (0, K, 0, 0, 0)

    def variant(**kw):
        r = good.copy()
        for k, v in kw.items():
            r[k][1] = v
        return r
    bad = [(FORMAT_UC8 + 7, good, row), (FORMAT_UC8, variant(n_buffers=K + 1), row), (FORMAT_UC8, variant(preamble_threshold=-1), row),
           (FORMAT_UC8, variant(reserved_=1), row), (FORMAT_UC8, variant(flags=2), row), (FORMAT_UC8, good, K * buf * 2 - 16),
           (FORMAT_SC16, good, K * buf * 4 - 16)]            # 4 bytes per sample
    for fmt, rx, stride in bad:
        for call in (d.run_device_rx, d.run_device_rx_async, d.run_host_rx_async):
            with pytest.raises(DemodError):
                call(fmt, host.ctypes.data, stride, buf, rx)
    with pytest.raises(DemodError):        # a host-path receiver with no stored halo of this width cannot continue
        d.run_host_rx_async(FORMAT_UC8, host.ctypes.data, row, buf, variant(flags=RX_CONTINUES))
    with pytest.raises(DemodError):
        d.run_device_rx(FORMAT_UC8, host.ctypes.data, row, buf - 4, good)
    with pytest.raises(DemodError):
        d.restart_stream(S)
    with pytest.raises(AssertionError):
        d.run_host_rx_async(FORMAT_UC8, host.ctypes.data, row, buf, good[:2])
    # nothing was enqueued or stored: the first step is the one that fills the pipeline and starts the halo store
    refs = [_Rx(FORMAT_UC8, 60000) for _ in range(S)]
    d.run_host_rx_async(FORMAT_UC8, host.ctypes.data, row, buf, good)
    sc = np.ascontiguousarray(np.stack([_to_sc16(c, False, 1).view(np.uint8) for c in caps]))
    with pytest.raises(DemodError):        # an sc16 step cannot continue a uc8 one
        d.run_host_rx_async(FORMAT_SC16, sc.ctypes.data, sc.shape[1], buf, variant(flags=RX_CONTINUES))
    d.wait()
    cont = good.copy(); cont["flags"] = RX_CONTINUES; cont["first_sample_timestamp"] = K * buf * 5
    d.run_host_rx_async(FORMAT_UC8, host.ctypes.data + K * buf * 2, row, buf, cont)
    fr = [d.frames(s) for s in range(S)]
    d.wait()
    for s in range(S):
        refs[s].step(caps[s], 2 * K, buf, 0, False, 0)
        got = np.concatenate([fr[s], d.frames(s)])
        problems = diff_frames(got, np.concatenate(refs[s].frames)) + diff_stats(d.stats(s), refs[s].o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
    d.close()


def test_rx_step_dtype_matches_the_header():
    """RX_STEP_DTYPE is the header's b200_rx_step: 24 bytes, same offsets."""
    import re
    from pathlib import Path
    text = (Path(__file__).resolve().parent.parent / "include" / "b200_demod.h").read_text()
    body = re.search(r"typedef struct b200_rx_step \{(.*?)\} b200_rx_step;", text, re.S).group(1)
    ctypes_of = {"int64_t": ctypes.c_int64, "uint32_t": ctypes.c_uint32, "int32_t": ctypes.c_int32}
    fields = [(m.group(2), ctypes_of[m.group(1)]) for m in re.finditer(r"^\s*(\w+)\s+(\w+);", body, re.M)]
    S = type("S", (ctypes.Structure,), {"_fields_": fields})
    assert ctypes.sizeof(S) == RX_STEP_DTYPE.itemsize == 24
    assert [n for n, _ in fields] == list(RX_STEP_DTYPE.names)
    for n, _ in fields:
        assert getattr(S, n).offset == RX_STEP_DTYPE.fields[n][1], n
    assert re.search(r"#define B200_RX_CONTINUES 0x1u", text) and RX_CONTINUES == 1
    assert re.search(r"B200_FORMAT_UC8 = 0, B200_FORMAT_SC16 = 1, B200_FORMAT_SC16Q11 = 2", text)
    assert (FORMAT_UC8, FORMAT_SC16, FORMAT_SC16Q11) == (0, 1, 2)


def test_rx_steps_on_emulated_kernels():
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_rx_steps.py", select="not full_size and not dense_rx")


def test_rx_steps_on_emulated_kernels_under_address_sanitizer():
    """Redzones around every "device" allocation: the halo store, the converter and the absent receivers' rows are never read or
    written out of bounds."""
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_rx_steps.py", select="not full_size and not dense_rx", sanitize="address")
