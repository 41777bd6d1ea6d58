"""-m gpu: b200_demod_fetch_raw, the raw / AVR records encoded on the device, byte for byte.

Network records (modesSendRawOutput, net_io.c:1837-1863) and the --raw stdout line (displayModesMessage, mode_s.c:1835-1841)
against the oracle's frames and replies through rawlib.raw_records, against the bytes the reference program itself sent to a raw_out
client (tests/golden/raw/raw_stream.npz), and against the reference program's own --mlat --raw output; on the host-buffer,
device-resident, pipelined, sc16 and independent-receiver paths; with 12 MHz clocks past 2^48, negative, and exactly 0.

The gpu-marked tests also run on the emulated kernels in the tier without a GPU (tests/test_emu_raw.py)."""
import ctypes as C
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oraclelib import Oracle
from rawlib import raw_records
from readsb_b200 import synth
from readsb_b200.abi import FORMAT_SC16, FORMAT_UC8, RX_STEP_DTYPE
from test_gpu_parity import _device_streams
from test_gpu_rx_steps import _Session

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
READSB_CPU = ROOT / "oracle" / "_ref" / "readsb_cpu"
# every valid (mlat, verbatim, stdout): the stdout line always prints the corrected frame
COMBOS = [(m, v, o) for m in (False, True) for v in (False, True) for o in (False, True) if not (v and o)]
E_INVAL, E_OVERFLOW = -1, -6


def _kw(combo):
    return dict(mlat=combo[0], verbatim=combo[1], stdout=combo[2])


def _traffic(n, seed, rate=3000.0):
    return synth.generate(n, seed=seed, frames_per_sec=rate, df_mask=synth.MODEAC | synth.DF17 | synth.DF11 | synth.AP | synth.DF18,
                          n_icao=5, amp=(0.35, 0.95), p_bit_error=0.4)


def _run_records(d, s, mode_ac):
    """The library's own frames and replies of receiver s's last run, the frames' buffer number made per-run like the replies'."""
    f, b = d.frames(s).copy(), d.buffer_results(s)
    if len(b):
        f["buffer_seq"] -= b["buffer_seq"][0]
    return f, (d.modeac(s) if mode_ac else None)


@pytest.mark.parametrize("mode_ac", [False, True])
def test_raw_output_matches_oracle(cuda, mode_ac):
    """Every flag combination: several streams, several buffers per run, runs concatenated; a second call gives the same bytes,
    and Beast calls in between (the same one-run cache, another format) change neither."""
    from readsb_b200.demod import Demodulator
    S, buf, K, runs = 3, 32768, 3, 2
    n = buf * K * runs
    iqs = [_traffic(n, 90 + s, [3000.0, 9000.0, 500.0][s]) for s in range(S)]
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K, mode_ac=mode_ac)
    got = {c: [b"" for _ in range(S)] for c in COMBOS}
    beast = [b"" for _ in range(S)]
    for r in range(runs):
        for b in range(K):
            k = r * K + b
            for s in range(S):
                d.submit_iq(s, iqs[s][2 * k * buf: 2 * (k + 1) * buf], k * buf * 5)
        d.run()
        for s in range(S):
            for c in COMBOS:
                first = d.raw(s, **_kw(c))
                beast[s] += d.beast(s) if c == COMBOS[0] else b""
                assert d.raw(s, **_kw(c)) == first, f"run {r} stream {s} {c}: second call"
                got[c][s] += first
    for s in range(S):
        fo, _ = Oracle().run_stream(iqs[s], buf)
        ao = Oracle().run_stream_ac(iqs[s], buf) if mode_ac else None
        assert len(fo) > 10 and (not mode_ac or s != 0 or len(ao) > 3)
        assert beast[s] == Oracle.beast(fo, ao), f"stream {s}: Beast bytes"
        for c in COMBOS:
            want = raw_records(fo, ao, **_kw(c))
            assert got[c][s] == want, f"stream {s} {c}: {len(got[c][s])} vs {len(want)} bytes"
    assert got[(False, True, False)] != got[(False, False, False)]      # some frames were repaired: the bytes as received differ
    d.close()


@pytest.mark.parametrize("mlat", [False, True])
def test_raw_golden_stream_from_reference_program(cuda, mlat):
    """The bytes the reference program sent to a raw_out client with --net-verbatim --modeac (tests/golden/make_raw_golden.py)."""
    from readsb_b200.demod import Demodulator
    z = np.load(ROOT / "tests" / "golden" / "beast_stream.npz")
    want = bytes(np.load(ROOT / "tests" / "golden" / "raw" / "raw_stream.npz")["raw_mlat" if mlat else "raw"])
    meta = json.loads(bytes(z["meta"]).decode())
    iq = np.concatenate([np.full(2 * meta["silence_samples"], 127, np.uint8), z["traffic"]])
    d = Demodulator(n_streams=1, buf_samples=131072, max_buffers_per_run=4, mode_ac=True)
    got, off, nsamples = b"", 0, iq.size // 2
    while off < nsamples:
        for _ in range(4):
            if off >= nsamples:
                break
            m = min(131072, nsamples - off)
            d.submit_iq(0, iq[2 * off: 2 * (off + m)], off * 5); off += m
        d.run(); got += d.raw(0, mlat=mlat, verbatim=True)
    assert len(want) > 1000 and got == want
    d.close()


@pytest.mark.skipif(not READSB_CPU.exists(), reason="oracle/_ref/readsb_cpu not built")
@pytest.mark.parametrize("extra,buf", [([], 131072), (["--sdr-buffer-size=128"], 65536)])
def test_stdout_lines_equal_readsb_cpu(cuda, tmp_path, extra, buf):
    """`readsb --device-type ifile --mlat --raw --modeac` prints one line per accepted frame and reply (displayModesMessage): the
    library's B200_RAW_STDOUT | B200_RAW_MLAT records of the same buffers are those lines."""
    from readsb_b200.demod import Demodulator
    nsamples = 1_200_000 + 4321                                   # a partial last buffer
    iq = synth.generate(nsamples, seed=2025, frames_per_sec=4000.0, df_mask=synth.MODEAC | synth.DF17 | synth.DF11 | synth.AP,
                        n_icao=12, amp=(0.3, 0.9), p_bit_error=0.3)
    cap = tmp_path / "cap.bin"
    iq.tofile(cap)
    res = subprocess.run([str(READSB_CPU), "--device-type", "ifile", "--ifile", str(cap), "--mlat", "--raw", "--modeac"] + extra,
                         capture_output=True, text=True, timeout=180)
    assert res.returncode == 0, res.stderr[-2000:]
    want = [l for l in res.stdout.splitlines() if l.startswith("@") or l.startswith("*")]
    d = Demodulator(n_streams=1, buf_samples=buf, max_buffers_per_run=4, mode_ac=True)
    got, off = b"", 0
    while off < nsamples:
        for _ in range(4):
            if off >= nsamples:
                break
            m = min(buf, nsamples - off)
            d.submit_iq(0, iq[2 * off: 2 * (off + m)], off * 5); off += m
        d.run(); got += d.raw(0, mlat=True, stdout=True)
    lines = got.decode().splitlines()
    assert len(want) > 200 and any(len(l) == 1 + 12 + 4 + 1 for l in want)     # Mode A/C replies among them
    assert lines == want, f"first difference at line {next((i for i, (a, b) in enumerate(zip(want, lines)) if a != b), min(len(want), len(lines)))}"
    d.close()


def test_device_async_steps_fetched_while_the_next_is_in_flight(cuda):
    from readsb_b200.demod import Demodulator
    S, buf, nb, calls = 2, 32768, 2, 3
    total = buf * nb * calls
    iqs = [_traffic(total, 40 + s, 4000.0) for s in range(S)]
    dev, stride, pad = _device_streams(iqs, total)
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=nb, mode_ac=True)
    got = {c: [b"" for _ in range(S)] for c in COMBOS}
    for c in range(calls):
        d.run_device_async(dev.data_ptr() + pad + c * nb * buf * 2, stride, nb, buf, continues=c > 0, first_sample_timestamp=c * nb * buf * 5)
        if c >= 1:
            d.wait()
            for s in range(S):                        # the next step is in flight in the other slot
                for k in COMBOS:
                    got[k][s] += d.raw(s, **_kw(k))
    d.wait()
    for s in range(S):
        for k in COMBOS:
            got[k][s] += d.raw(s, **_kw(k))
    for s in range(S):
        fo, _ = Oracle().run_stream(iqs[s], buf)
        ao = Oracle().run_stream_ac(iqs[s], buf)
        assert len(fo) > 20
        for k in COMBOS:
            assert got[k][s] == raw_records(fo, ao, **_kw(k)), f"stream {s} {k}"
    d.close()


class _RawSession(_Session):
    """An independent-receiver session that also fetches every receiver's raw records after each step."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.raw_got = {c: [b"" for _ in range(self.S)] for c in COMBOS}

    def _harvest(self, row):
        super()._harvest(row)
        for s in range(self.S):
            for c in COMBOS:
                r = self.d.raw(s, **_kw(c))
                assert row[s][0] or r == b"", f"absent receiver {s} has raw records"
                self.raw_got[c][s] += r

    def check(self, min_frames=50):
        want = {}
        for s in range(self.S):
            ref = self.refs[s]
            fo = np.concatenate(ref.frames) if ref.frames else np.zeros(0, self.got[s][0][0].dtype)
            ao = np.concatenate(ref.ac) if (self.mode_ac and ref.ac) else None
            for c in COMBOS:
                want[c, s] = raw_records(fo, ao, **_kw(c))
        super().check(min_frames)
        for (c, s), w in want.items():
            assert self.raw_got[c][s] == w, f"receiver {s} {c}: {len(self.raw_got[c][s])} vs {len(w)} bytes"


# receiver 1 absent in steps 1 and 2 and then continuing; receiver 2 restarted after a gap in step 2 (its clock jumps, zero halo)
_PLAN = [[(2, False, False, 0), (1, False, False, 0), (2, False, False, 0)],
         [(1, True, False, 0), (0, True, False, 0), (2, True, False, 40)],
         [(2, True, False, 0), (0, True, False, 0), (1, False, True, 0)],
         [(1, True, False, 75), (2, True, False, 0), (2, True, False, 0)]]


@pytest.mark.parametrize("path,fmt", [("host", FORMAT_UC8), ("device", FORMAT_SC16), ("device_async", FORMAT_UC8)])
def test_independent_receivers(cuda, path, fmt):
    """run_host_rx_async (pipelined), an sc16 run_device_rx step and run_device_rx_async: an absent receiver has no records, a
    receiver restarted after a gap goes on in order, Mode A/C replies included."""
    _RawSession(path, fmt, S=3, K=2, buf=16384, mode_ac=True, plan=_PLAN, seed=7).run().check(min_frames=30)


def _rx_results(clocks, iq, buf, K):
    """One run_device_rx step of len(clocks) receivers over the same capture, receiver s's clock starting at clocks[s]."""
    from readsb_b200.demod import Demodulator
    S = len(clocks)
    dev, stride, pad = _device_streams([iq] * S, K * buf)
    rx = np.zeros(S, RX_STEP_DTYPE)
    for s, t in enumerate(clocks):
        rx[s] = (t, K, 0, 0, 0)
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K, mode_ac=True)
    d.run_device_rx(FORMAT_UC8, dev.data_ptr() + pad, stride, buf, rx)
    return d


def test_clocks_past_2_48_negative_and_zero(cuda):
    """Through b200_rx_step.first_sample_timestamp (the ABI takes any int64 clock): a receiver whose clock crosses 2^48 - the
    network record keeps the first 12 of the 13 digits, the stdout line prints all 13 - and receivers whose clocks start negative
    so that one frame and one Mode A/C reply fall exactly on 0 - those records start with '*' even with MLAT, and the negative
    ones print PRIX64 of the unsigned value (16 digits on stdout, the first 12 of them on the network)."""
    buf, K = 65536, 3
    iq = synth.modeac_stream(31, K * buf)
    probe = _rx_results([0], iq, buf, K)
    f0, a0 = probe.frames(0), probe.modeac(0)
    probe.close()
    df17 = f0[(f0["msgtype"] == 17) & (f0["crc"] == 0)]
    assert len(df17) > 4 and len(a0) > 4
    t_frame, t_ac, t_mid = int(df17["timestamp"][len(df17) // 2]), int(a0["timestamp"][len(a0) // 2]), int(f0["timestamp"][len(f0) // 2])
    clocks = [(1 << 48) - t_mid, -t_frame, -t_ac]
    d = _rx_results(clocks, iq, buf, K)
    for s in range(3):
        f, a = _run_records(d, s, True)
        for c in COMBOS:
            assert d.raw(s, **_kw(c)) == raw_records(f, a, **_kw(c)), f"receiver {s} {c}"
    net = [d.raw(s, mlat=True).decode().splitlines() for s in range(3)]
    out = [d.raw(s, mlat=True, stdout=True).decode().splitlines() for s in range(3)]
    assert all(len(net[s]) == len(out[s]) > 10 for s in range(3))
    # past 2^48: 13 digits on stdout, the first 12 of them on the network; before it 12 in both
    late = [(n, o) for n, o in zip(net[0], out[0]) if len(o) == len(n) + 1]
    assert late and all(o.startswith("@1000000") and n[:13] == o[:13] and n[13:] == o[14:].upper() for n, o in late)
    assert any(len(o) == len(n) and n[13:] == o[13:].upper() for n, o in zip(net[0], out[0]))
    # exactly 0: '*' even with MLAT; negative: PRIX64 of the unsigned value, 16 digits on stdout, the first 12 on the network
    for s, rec_len in ((1, 1 + 28 + 1), (2, 1 + 4 + 1)):              # a DF17 frame on 0, a Mode A/C reply on 0
        stars = [(n, o) for n, o in zip(net[s], out[s]) if o.startswith("*")]
        assert len(stars) == 1 and len(stars[0][1]) == rec_len and stars[0][0] == stars[0][1].upper()
        neg = [(n, o) for n, o in zip(net[s], out[s]) if len(o) == len(n) + 4]
        assert neg and all(o.startswith("@FFFFFFFFFF") and n[:13] == o[:13] and n[13:] == o[17:].upper() for n, o in neg)
    d.close()


def test_overflow_and_bad_flags(cuda):
    from readsb_b200.demod import RAW_MLAT, RAW_STDOUT, RAW_VERBATIM, Demodulator
    iq = _traffic(65536, 5, 6000.0)
    d = Demodulator(n_streams=2, buf_samples=65536, max_buffers_per_run=1, mode_ac=True)
    d.submit_iq(0, iq, 0)
    d.run()
    whole = d.raw(0, mlat=True)
    assert len(whole) > 100
    n = C.c_uint32(7)
    buf = (C.c_uint8 * len(whole))(*([0xAA] * len(whole)))
    assert d.L.b200_demod_fetch_raw(d.h, 0, RAW_MLAT, buf, len(whole) - 1, C.byref(n)) == E_OVERFLOW
    assert n.value == len(whole) and bytes(buf) == b"\xaa" * len(whole)      # nothing copied
    assert d.L.b200_demod_fetch_raw(d.h, 0, RAW_MLAT, buf, len(whole), C.byref(n)) == 0 and bytes(buf) == whole
    for bad in (0x8, 0x80000000, RAW_STDOUT | RAW_VERBATIM, RAW_STDOUT | RAW_VERBATIM | RAW_MLAT):
        assert d.L.b200_demod_fetch_raw(d.h, 0, bad, buf, len(whole), C.byref(n)) == E_INVAL, hex(bad)
    assert d.L.b200_demod_fetch_raw(d.h, 2, RAW_MLAT, buf, len(whole), C.byref(n)) == E_INVAL      # no such stream
    assert d.L.b200_demod_fetch_raw(d.h, 1, 0, None, 0, C.byref(n)) == 0 and n.value == 0          # nothing submitted for it
    assert d.raw(0, mlat=True) == whole
    d.close()
