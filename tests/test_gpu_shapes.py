"""The launch shapes where the kernels change their schedule, every receiver against an oracle of its own:

- the scan kernel's three regimes (b200_launch_scan, scan_kernel.cu): one CTA per tile (static tiles, each shared by four warps), a
  spread grid with dynamic claims, and the persistent grid; at the chip's own SM count and on small forced grids;
- stage B's work units (resolve_stream): whole buffers, or sub-ranges of whole tiles of each buffer;
- stage B CTAs in several waves (more receivers than the chip holds at two CTAs per SM), with grown filter tables at receiver 0
  and past the first 256 receivers;
- one receiver with grown filter tables (resolve_solo_kernel's grown-table instantiation, the drop-in's shape);
- the result copy around FIRST_COPY_FRAMES (16) frames.

Before it compares anything, each test asserts that it reached the shape it is named for, from what the library reports
(debug_counters, timing()["launches"], icao_test).  The gpu-marked tests also run on the emulated kernels of a 20-SM chip in the
tier without a GPU (the last tests of this file)."""
import os
import re
from pathlib import Path

import numpy as np
import pytest

from oraclelib import Oracle
from paritylib import diff_bufres, diff_frames, diff_stats
from test_gpu_parity import _to_sc16
from test_gpu_rx_steps import _Rx, _Session
from readsb_b200 import synth
from readsb_b200.abi import FORMAT_SC16, FORMAT_UC8

ROOT = Path(__file__).resolve().parent.parent
SCAN_SRC = ROOT / "readsb_b200" / "csrc" / "scan_kernel.cu"
RESOLVE_SRC = ROOT / "readsb_b200" / "csrc" / "resolve_kernel.cu"
SCAN_TILE = 2048
# Device-resident and pipelined steps: d_iq is 16-byte aligned and the 326-sample halo lies 652 bytes in front of it (sc16: the
# converter's slab, 2 samples of padding), so a segment's base is 4 bytes past a 16-byte boundary: 2 dummy positions in its first tile.
LEAD = 2
# Buffers of 2040 samples: a receiver with n buffers (n <= 255) has exactly n tiles, since 2 + 2040 n <= 2048 n < 2 + 2040 n + 2048.
TILE_BUF = 2040
ICAO_DEFAULT_GEN = 2048        # addresses one generation of the default tables holds (4096 slots at load <= 1/2)
ICAO_ADDED = 0x01              # B200_FRAME_ICAO_ADDED


def _sc_warps() -> int:
    return int(re.search(r"#define SC_WARPS (\d+)", SCAN_SRC.read_text()).group(1))


SC_WARPS = _sc_warps()


def _regime(n_tiles: int, grid: int) -> str:
    """b200_launch_scan's rule (test_regime_rule_is_the_launchers pins it to the source)."""
    if n_tiles >= grid * SC_WARPS:
        return "persistent"
    return "static" if n_tiles <= grid else "spread"


def _target(where: str, grid: int):
    """Tile count at a regime boundary and the regime it has to land in."""
    return {"grid-1": (grid - 1, "static"), "grid": (grid, "static"), "grid+1": (grid + 1, "spread"),
            "28grid-1": (SC_WARPS * grid - 1, "spread"), "28grid": (SC_WARPS * grid, "persistent"),
            "28grid+1": (SC_WARPS * grid + 1, "persistent")}[where]


WHERES = ["grid-1", "grid", "grid+1", "28grid-1", "28grid", "28grid+1"]


def _sms() -> int:
    if os.environ.get("B200_EMU") == "1":
        return int(os.environ.get("B200_EMU_SMS", "2"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(npos: int, lead: int = LEAD) -> int:
    return (lead + npos + SCAN_TILE - 1) // SCAN_TILE if npos else 0


def _nsplit(n_bufs: int, buf_len: int) -> int:
    """Work units per buffer in resolve_stream: whole buffers from 8 buffers on, else sub-ranges of whole tiles (at most 8 units)."""
    if n_bufs >= 8:
        return 1
    return max(1, min(8 // max(n_bufs, 1), (buf_len + 4 * SCAN_TILE - 1) // (4 * SCAN_TILE)))


def _sub_len(n_bufs: int, buf_len: int) -> int:
    ns = _nsplit(n_bufs, buf_len)
    return buf_len if ns == 1 else ((-(-buf_len // ns) + SCAN_TILE - 1) & ~(SCAN_TILE - 1))


def _dense(s: int, n: int, seed: int):
    """Dense traffic: the 10 000 frames/s stress, or strong overlapping frames near clipping."""
    if s % 2 == 1:
        return synth.generate(n, seed=seed + s, frames_per_sec=8000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP | synth.MODEAC, n_icao=8,
                              amp=(0.7, 1.0), p_bit_error=0.3)
    return synth.config5_stream(seed + s, n)


def _record(sess):
    """debug_counters() and timing() after every step the session collects."""
    seen = []
    orig = sess._harvest

    def harvest(row):
        orig(row)
        seen.append((sess.d.debug_counters(), sess.d.timing()))
    sess._harvest = harvest
    return seen


def _uniform_plan(counts, steps):
    return [[(n, k > 0, False, 0) for n in counts] for k in range(steps)]


def _forward(d, ref: Oracle, s: int, addrs):
    for a in addrs:
        d.icao_add(s, int(a)); ref.icao_add(int(a))


# ---- 1. scan regimes at the chip's SM count ------------------------------------------------------------------------------------
def _regime_session(path, T, fmt=FORMAT_UC8, mode_ac=False, seed=1):
    """T tiles per step in TILE_BUF buffers, spread over receivers of up to 60 buffers; three steps (depth 3 when pipelined)."""
    S = max(8, -(-T // 60))
    base, extra = divmod(T, S)
    counts = [base + (s < extra) for s in range(S)]
    steps = 3 if path != "device" else 2
    sess = _Session(path, fmt, S=S, K=max(counts), buf=TILE_BUF, depth=3, mode_ac=mode_ac, seed=seed, plan=_uniform_plan(counts, steps))
    # dense traffic: every tile has preambles and records, so a tile scanned twice or not at all shows in the results
    raw8 = [_dense(s, max(n, 1) * TILE_BUF * steps, 100 * seed) for s, n in enumerate(counts)]
    sess.raw = raw8 if fmt == FORMAT_UC8 else [_to_sc16(r, False, seed + s) for s, r in enumerate(raw8)]
    return sess, counts


def _check_regime(path, where, grid, fmt=FORMAT_UC8, mode_ac=False, seed=1):
    T, want = _target(where, grid)
    assert _regime(T, grid) == want, (where, T, grid)
    sess, counts = _regime_session(path, T, fmt, mode_ac, seed)
    seen = _record(sess)
    sess.run()
    present = sum(1 for n in counts if n)
    for c, _ in seen:
        assert (c["tiles"], c["segments"], c["buffers"]) == (T, present, sum(counts)), c
        assert sum(_tiles(n * TILE_BUF) for n in counts) == T
    sess.check(min_frames=1)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "device_async"])
@pytest.mark.parametrize("where", WHERES)
def test_scan_regimes_at_the_chips_sm_count(cuda, monkeypatch, path, where):
    """Tile counts one below, at and one above each regime boundary of a grid of the chip's SMs, blocking and three steps in flight."""
    monkeypatch.delenv("B200_SCAN_SMS", raising=False)
    monkeypatch.setenv("B200_SCAN_PART", "0")      # pipelined steps keep the whole chip (no measured partition moving the boundary)
    _check_regime(path, where, _sms(), seed=3 + WHERES.index(where))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,where", [("modeac", "grid"), ("modeac", "28grid"), ("sc16", "grid+1"), ("sc16", "28grid-1")])
def test_scan_regimes_with_modeac_and_sc16(cuda, monkeypatch, kind, where):
    """The scan kernel that keeps its magnitudes for Mode A/C, and sc16 input (magnitude segments over the converter's slab)."""
    monkeypatch.delenv("B200_SCAN_SMS", raising=False)
    monkeypatch.setenv("B200_SCAN_PART", "0")
    _check_regime("device_async", where, _sms(), fmt=FORMAT_SC16 if kind == "sc16" else FORMAT_UC8, mode_ac=kind == "modeac", seed=20)


# ---- 2. small forced grids -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("grid", [1, 3, 7])
def test_scan_regimes_on_forced_small_grids(cuda, monkeypatch, grid):
    assert grid <= _sms()
    monkeypatch.setenv("B200_SCAN_SMS", str(grid))          # read by create: the scan grid of blocking and pipelined runs
    for i, where in enumerate(WHERES):
        if _target(where, grid)[0] == 0:
            continue
        for path in ("device", "device_async"):
            _check_regime(path, where, grid, seed=30 + grid + i)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [3, 7])
def test_tiles_shared_between_warps(cuda, monkeypatch, grid):
    """n_tiles == grid: CTA b takes tile b, and its first four warps share it, one chunk each."""
    monkeypatch.setenv("B200_SCAN_SMS", str(grid))
    for path in ("device", "device_async"):
        _check_regime(path, "grid", grid, seed=41)


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [1, 3])
def test_claims_cross_many_short_segments(cuda, monkeypatch, grid):
    """Receivers of 1, 2, 3, 5 and 9 tiles in one run: claims of up to 8 tiles cut through several segments, quads end partway."""
    monkeypatch.setenv("B200_SCAN_SMS", str(grid))
    counts = [1, 2, 3, 5, 9] * 12
    T = sum(counts)
    assert _regime(T, grid) == "persistent" and min(-(-T // (grid * SC_WARPS)), 8) >= 3      # the first claims take 8 or 3 tiles
    for path in ("device", "device_async"):
        sess = _Session(path, FORMAT_UC8, S=len(counts), K=9, buf=TILE_BUF, depth=3, seed=50 + grid, plan=_uniform_plan(counts, 2))
        seen = _record(sess)
        sess.run()
        for c, _ in seen:
            assert (c["tiles"], c["segments"], c["buffers"]) == (T, len(counts), T), c
        sess.check()


# ---- 3. stage B work units -------------------------------------------------------------------------------------------------------
KS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 16]
SPLIT_LENGTHS = {         # buffer length -> buffer counts of consecutive runs
    2040: KS,             # 1 tile per buffer (tiles straddle buffer boundaries)
    4088: KS,             # 2
    14328: KS,            # 7
    16376: KS,            # 8
    18424: KS,            # 9
    10000: KS,            # not a multiple of 2048
    65528: [1, 2, 3, 4, 5, 8, 9],     # 32 tiles: 8, 4 and 2 sub-ranges
}


def _edge_frames(ref: _Rx, Ks, buf):
    """Oracle frames whose skip (the 2 x msgbits positions after an accepted frame, demod_2400.c:468) reaches over a sub-range edge of
    their buffer: stage B has to redo the unit after the edge."""
    n, b = 0, 0
    for K in Ks:
        sub = _sub_len(K, buf)
        edges = np.arange(sub, buf, sub) if _nsplit(K, buf) > 1 else np.zeros(0, np.int64)
        for _ in range(K):
            f = ref.frames[b]
            if len(edges) and len(f):
                j = f["j"].astype(np.int64)[:, None]
                n += int(((j < edges[None, :]) & (edges[None, :] <= j + 2 * f["msgbits"].astype(np.int64)[:, None])).any(axis=1).sum())
            b += 1
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("path", ["device", "device_async", "host"])
@pytest.mark.parametrize("buf", list(SPLIT_LENGTHS))
def test_stage_b_work_units(cuda, path, S, buf):
    """Dense traffic in consecutive runs of 1 - 9 and 16 buffers per receiver: whole buffers from 8 on, below that every buffer cut
    into sub-ranges of whole tiles.  One receiver (resolve_solo_kernel) and three (resolve_kernel)."""
    Ks = SPLIT_LENGTHS[buf]
    plan = [[(K, k > 0, False, 0)] * S for k, K in enumerate(Ks)]
    sess = _Session(path, FORMAT_UC8, S=S, K=max(Ks), buf=buf, depth=2, seed=60, plan=plan)
    sess.raw = [_dense(s, sum(Ks) * buf, 600 + buf) for s in range(S)]
    seen = _record(sess)
    sess.run()
    for (c, _), K in zip(seen, Ks):
        assert (c["tiles"], c["segments"], c["buffers"]) == (S * _tiles(K * buf), S, S * K), (K, c)
    if buf > 4 * SCAN_TILE:
        assert {_nsplit(K, buf) for K in Ks} - {1}
        assert sum(_edge_frames(r, Ks, buf) for r in sess.refs) > 0
    sess.check()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("buf", [2040, 16376, 18424, 10000, 65528, 12345])
def test_stage_b_work_units_on_the_submit_path(cuda, S, buf):
    """The same through submit_iq + run: a run of full buffers with contiguous timestamps is one segment (the arena's regions are
    256-byte aligned: no dummy positions)."""
    from readsb_b200.demod import Demodulator
    Ks = SPLIT_LENGTHS.get(buf, [1, 2, 3, 4, 5, 8, 9, 16])
    raws = [_dense(s, sum(Ks) * buf, 600 + buf) for s in range(S)]
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=max(Ks))
    refs = [_Rx(FORMAT_UC8, 60000) for _ in range(S)]
    got = [([], []) for _ in range(S)]
    cur = 0
    for k, K in enumerate(Ks):
        for s in range(S):
            for b in range(K):
                off = cur + b * buf
                d.submit_iq(s, raws[s][2 * off: 2 * (off + buf)], off * 5)
        d.run()
        c = d.debug_counters()
        assert (c["tiles"], c["segments"], c["buffers"]) == (S * _tiles(K * buf, lead=0), S, S * K), (K, c)
        for s in range(S):
            refs[s].step(raws[s][2 * cur: 2 * (cur + K * buf)], K, buf, cur * 5, k > 0, 0)
            f = d.frames(s)
            got[s][0].append(f); got[s][1].append(d.buffer_results(s))
            assert d.beast(s) == Oracle.beast(f), f"receiver {s}: Beast bytes"
        cur += K * buf
    if buf > 4 * SCAN_TILE:
        assert sum(_edge_frames(r, Ks, buf) for r in refs) > 0
    total = 0
    for s in range(S):
        fg, bg = np.concatenate(got[s][0]), np.concatenate(got[s][1])
        problems = diff_frames(fg, np.concatenate(refs[s].frames)) + diff_bufres(bg, np.concatenate(refs[s].bufres)) + diff_stats(d.stats(s), refs[s].o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
        total += len(fg)
    assert total > 50
    d.close()


# ---- 4. stage B CTA waves ----------------------------------------------------------------------------------------------------------
def _wave_receivers(case: str, sms: int) -> int:
    # resolve_kernel runs one CTA per receiver, two per SM by its __launch_bounds__(256, RS_MIN_CTAS = 2) - an occupancy set at compile
    # time, not queried from the device here: S against 2 x SMs says how many CTAs wait for a later wave.  The last case has at least
    # 259 receivers, so that receivers past the first 256 (one pass of the capacity check's 256 threads) have grown tables.
    return {"2sm-1": 2 * sms - 1, "2sm": 2 * sms, "2sm+1": 2 * sms + 1, "4sm+3": max(4 * sms + 3, 259)}[case]


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "device_async"])
@pytest.mark.parametrize("case", ["2sm-1", "2sm", "2sm+1", "4sm+3"])
def test_stage_b_ctas_in_several_waves(cuda, path, case):
    """Receivers of one or two 4096-sample buffers, more than one wave of stage B CTAs.  With 2 x SMs + 1 and 4 x SMs + 3 receivers,
    receivers 0 and S - 1 have grown tables (2 100 forwarded addresses), so the grown-table launch runs in several waves too; with
    4 x SMs + 3, receiver S - 2 (past the first 256) holds 2 046 forwarded addresses and learns at least three more from its own traffic
    in the first run: the capacity check asks for larger tables, the library grows them and repeats the run."""
    sms = _sms()
    S = _wave_receivers(case, sms)
    rng = np.random.default_rng(S)
    counts = [[int(rng.integers(1, 3)) for _ in range(S)] for _ in range(2)]
    grown = [0, S - 1] if case in ("2sm+1", "4sm+3") else []
    in_run = S - 2 if case == "4sm+3" else None
    if in_run is not None:
        counts[0][in_run] = 1              # its first buffer teaches the generation the forwarded addresses are in
    plan = [[(counts[k][s], k > 0, False, 0) for s in range(S)] for k in range(2)]
    sess = _Session(path, FORMAT_UC8, S=S, K=2, buf=4096, depth=2, seed=70, plan=plan)
    addrs = np.random.default_rng(71).choice(1 << 24, size=2 * 2100 + 2046, replace=False)
    for i, s in enumerate(grown):
        _forward(sess.d, sess.refs[s].o, s, addrs[i * 2100: (i + 1) * 2100])
    if in_run is not None:
        assert in_run >= 256
        fwd = addrs[2 * 2100:]
        _forward(sess.d, sess.refs[in_run].o, in_run, fwd)
        n = sum(r[in_run][0] for r in plan) * 4096
        sess.raw[in_run] = synth.generate(n, seed=73, frames_per_sec=6000.0, df_mask=synth.DF17, n_icao=400, amp=(0.5, 1.0))
    seen = _record(sess)
    sess.run()
    for (c, t), row in zip(seen, plan):
        assert (c["segments"], c["buffers"]) == (S, sum(r[0] for r in row)), c
        assert t["launches"] == (3 if grown else 2), t          # scan, stage B (+ stage B for grown tables)
    if in_run is not None:
        ref = sess.refs[in_run]
        first = ref.frames[0]
        learned = {int(a) & 0xFFFFFF for a, fl in zip(first["addr"], first["flags"]) if fl & ICAO_ADDED}
        assert len(learned - set(int(a) for a in fwd)) >= 3, learned     # more than 2 048 - 2 046 new addresses in the first buffer
        probe = sorted(set(int(a) for a in fwd) | learned)
        present = [sess.d.icao_test(in_run, a) for a in probe]
        assert present == [ref.o.icao_test(a) for a in probe]
        assert sum(present) > ICAO_DEFAULT_GEN, sum(present)   # one generation holds them all: the tables grew in the run
    sess.check()


# ---- 5. one receiver with grown tables -------------------------------------------------------------------------------------------
def _probe_filter(d, o, addrs):
    assert [d.icao_test(0, int(a)) for a in addrs] == [o.icao_test(int(a)) for a in addrs]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["submit", "device"])
@pytest.mark.parametrize("mode_ac", [False, True])
def test_one_receiver_with_forwarded_addresses(cuda, entry, mode_ac):
    """5 000 addresses forwarded through icao_add (a readsb fed by an aggregator), then a capture one buffer per run, through
    submit_iq + run and through run_device; then icao_expire and icao_test against the oracle."""
    import devbuf
    from readsb_b200.demod import Demodulator
    BUF = 65536
    d = Demodulator(n_streams=1, buf_samples=BUF, max_buffers_per_run=1, mode_ac=mode_ac)
    o, oa = Oracle(), Oracle()
    rng = np.random.default_rng(80)
    fwd = rng.choice(1 << 24, size=5000, replace=False)
    _forward(d, o, 0, fwd)
    held = sum(d.icao_test(0, int(a)) for a in fwd[:2500])
    assert held == 2500 > ICAO_DEFAULT_GEN            # one generation (no flip yet) holds more than the default tables
    iq = synth.generate(900_000, seed=40, frames_per_sec=2000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP | synth.MODEAC, n_icao=30)
    fo, bo = o.run_stream(iq, BUF)
    ao = oa.run_stream_ac(iq, BUF) if mode_ac else None
    if entry == "submit":
        out = d.replay(iq, want_modeac=mode_ac)
        fg, bg = out[0], out[1]
        ag = out[2] if mode_ac else None
    else:
        n = iq.size // 2
        dev = devbuf.zeros(1024 + iq.size)
        dev[1024:] = devbuf.to_dev(iq)
        devbuf.sync()
        fs, bs, acs = [], [], []
        for k, off in enumerate(range(0, n, BUF)):
            m = min(BUF, n - off)
            d.run_device(dev.data_ptr() + 1024 + 2 * off, 2 * BUF, 1, m, off > 0, off * 5)
            c, t = d.debug_counters(), d.timing()
            assert (c["tiles"], c["segments"], c["buffers"]) == (_tiles(m), 1, 1)
            if not mode_ac:
                assert t["launches"] == 2, t             # scan + the one-receiver stage B (its grown-table path is in the same kernel)
            f = d.frames(0)
            fs.append(f); bs.append(d.buffer_results(0))
            a = d.modeac(0) if mode_ac else None
            if mode_ac:
                a["buffer_idx"] += k
                acs.append(a)
            assert d.beast(0) == Oracle.beast(f, a), f"run {k}: Beast bytes"
        fg, bg = np.concatenate(fs), np.concatenate(bs)
        ag = np.concatenate(acs) if mode_ac else None
    problems = diff_frames(fg, fo) + diff_bufres(bg, bo) + diff_stats(d.stats(0), o.stats())
    assert not problems, "\n".join(problems)
    assert len(fo) > 300
    if mode_ac:
        assert len(ao) > 0
        for f in ("timestamp", "f1_sample", "modeac", "buffer_idx"):
            assert len(ag) == len(ao) and np.array_equal(ag[f], ao[f]), f"modeac {f}"
    learned = sorted({int(a) & 0xFFFFFF for a, fl in zip(fo["addr"], fo["flags"]) if fl & ICAO_ADDED})
    probe = list(fwd[::50]) + learned + list(rng.choice(1 << 24, size=100))
    _probe_filter(d, o, probe)
    for _ in range(2):                                   # the older generation goes, then the one that held the forwarded addresses
        d.icao_expire(0); o.icao_expire()
        _probe_filter(d, o, probe)
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 4])
def test_one_receiver_grows_its_tables_during_a_replay(cuda, K):
    """A capture of 9 000 aircraft: the one-receiver kernel's capacity check refuses a run, the library grows the tables and repeats
    it (with the halo carry of the refused attempt not made), and the runs after it use the grown tables."""
    from readsb_b200.demod import Demodulator
    iq = synth.generate(6_000_000, seed=41, frames_per_sec=4000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP, n_icao=9000, amp=(0.5, 0.9))
    o = Oracle()
    fo, bo = o.run_stream(iq, 65536)
    d = Demodulator(n_streams=1, buf_samples=65536, max_buffers_per_run=K)
    fg, bg = d.replay(iq)
    problems = diff_frames(fg, fo) + diff_bufres(bg, bo) + diff_stats(d.stats(0), o.stats())
    assert not problems, "\n".join(problems)
    # The filter flips once, at the end of buffer 0 (the first flip is due at once); everything taught after it is in one generation
    # (the capture is far shorter than the 60 s period).  More than 2 048 of them present: that generation outgrew the default tables.
    late = fo[fo["buffer_seq"] >= 1]
    taught = sorted({int(a) & 0xFFFFFF for a, fl in zip(late["addr"], late["flags"]) if fl & ICAO_ADDED})
    present = [d.icao_test(0, a) for a in taught]
    assert present == [o.icao_test(a) for a in taught]
    assert sum(present) > ICAO_DEFAULT_GEN, sum(present)
    d.icao_expire(0); o.icao_expire()
    _probe_filter(d, o, taught[::7])
    d.close()


# ---- 6. the result copy around FIRST_COPY_FRAMES -----------------------------------------------------------------------------------
def _prefix_with_frames(iq, want: int) -> int:
    """A length (a multiple of 8) whose single buffer gives `want` frames on a fresh oracle: the shortest one for want > 0, the
    longest one for want == 0."""
    def count(n):
        return len(Oracle().run_stream(iq[: 2 * n], 65536)[0]) if n else 0
    lo, hi = 1, iq.size // 2 // 8
    while lo < hi:
        mid = (lo + hi) // 2
        if count(8 * mid) >= max(want, 1):
            hi = mid
        else:
            lo = mid + 1
    n = 8 * lo if want else 8 * (lo - 1)
    assert n > 0 and count(n) == want, (want, n, count(n))
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("mode_ac", [False, True])
@pytest.mark.parametrize("total", [0, 16, 17])
def test_result_copy_edges(cuda, mode_ac, total):
    """Two receivers with 0, exactly 16 and exactly 17 frames in total: the first result copy carries 16 frames, a 17th takes the
    second copy.  Receiver 1 has Mode A/C replies only (their copy is a third one)."""
    from readsb_b200.demod import Demodulator
    BUF = 65536
    ac_only = synth.generate(40_000, seed=90, frames_per_sec=3000.0, df_mask=synth.MODEAC, amp=(0.3, 0.9))
    mixed = synth.mixed_stream(91, BUF)
    assert len(Oracle().run_stream(ac_only, BUF)[0]) == 0
    L = _prefix_with_frames(mixed, total)
    caps = [mixed[: 2 * L], ac_only]
    d = Demodulator(n_streams=2, buf_samples=BUF, max_buffers_per_run=1, mode_ac=mode_ac)
    for s, c in enumerate(caps):
        d.submit_iq(s, c, 0)
    d.run()
    assert d.debug_counters()["frames"] == d.total_frames() == total
    for s, c in enumerate(caps):
        o = Oracle()
        fo, bo = o.run_stream(c, BUF)
        f = d.frames(s)
        problems = diff_frames(f, fo) + diff_bufres(d.buffer_results(s), bo) + diff_stats(d.stats(s), o.stats())
        assert not problems, f"receiver {s}: " + "\n".join(problems)
        ao = None
        if mode_ac:
            ao, ag = Oracle().run_stream_ac(c, BUF), d.modeac(s)
            if s == 1:
                assert len(ao) > 0
            for fld in ("timestamp", "f1_sample", "modeac", "buffer_idx"):
                assert len(ag) == len(ao) and np.array_equal(ag[fld], ao[fld]), f"receiver {s}: modeac {fld}"
        assert d.beast(s) == Oracle.beast(f, ao), f"receiver {s}: Beast bytes"
    d.close()


# ---- without a GPU -----------------------------------------------------------------------------------------------------------------
def test_regime_rule_is_the_launchers():
    """The tests above choose their tile counts from _regime and their sub-ranges from _nsplit: both must be the kernels' rules, so
    that a change of a rule fails here instead of moving the tests off the boundaries they are named for."""
    src = SCAN_SRC.read_text()
    body = re.search(r'extern "C" int b200_launch_scan\(.*?\n\}', src, re.S).group(0)
    assert "uint32_t grid = (uint32_t)n_sm;" in body
    assert "if (q.n_tiles < grid * SC_WARPS) {" in body
    assert "if (grid > q.n_tiles) grid = q.n_tiles;" in body
    assert "q.warps_per_cta = (q.n_tiles + grid - 1) / grid;" in body
    assert "const bool shared = grid == q.n_tiles;" in body
    assert "if (shared) q.warps_per_cta = TILE_CHUNKS;" in body and "if (shared) { if (q.mag_copy) scan_kernel<true, true><<<" in body
    assert "q.warps_per_cta = SC_WARPS;" in body and "<<<grid, SC_WARPS * 32, smem, stream>>>" in body and SC_WARPS == 28
    assert [_regime(t, 132) for t in (131, 132, 133, 3695, 3696, 3697)] == ["static", "static", "spread", "spread", "persistent", "persistent"]
    res = RESOLVE_SRC.read_text()
    assert "const uint32_t nsplit = seg.n_bufs >= RS_WARPS ? 1u : max(1u, min((uint32_t)RS_WARPS / max(seg.n_bufs, 1u), " \
           "(seg.buf_len + 4 * SCAN_TILE - 1) / (4 * SCAN_TILE)));" in res
    assert "#define RS_WARPS 8 " in res
    assert re.search(r"#define RS_MIN_CTAS 2 ", res) and "__launch_bounds__(RS_WARPS * 32, RS_MIN_CTAS) resolve_kernel" in res
    assert [_nsplit(k, 65528) for k in (1, 2, 3, 4, 5, 8, 16)] == [8, 4, 2, 2, 1, 1, 1]
    assert _sub_len(5, 18424) == 18424 and _sub_len(3, 18424) == 10240 and _sub_len(1, 18424) == 6144
    assert _tiles(TILE_BUF) == 1 and _tiles(TILE_BUF * 255) == 255 and _tiles(TILE_BUF * 255, lead=0) == 255


def test_shapes_on_emulated_kernels():
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_shapes.py", extra_env={"B200_EMU_SMS": "20"}, timeout=1800)


def test_shapes_on_emulated_kernels_under_address_sanitizer():
    """Redzones around every "device" allocation, on the same shapes: no kernel reads or writes past a pool, a table or a result array
    at any regime boundary, work-unit split or wave."""
    from test_emu_kernels import _run_gpu_tests_emulated
    _run_gpu_tests_emulated("tests/test_gpu_shapes.py", extra_env={"B200_EMU_SMS": "20"}, sanitize="address", timeout=3000)
