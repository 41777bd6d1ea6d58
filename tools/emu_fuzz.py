"""Randomised parity runs of the kernels' source on the CPU (tests/emu/) against the oracle.  TEST TOOLING.

    python tools/emu_fuzz.py [--seed S] [--cases N] [--minutes M] [--sanitize address]

Each case draws: receivers, buffer length (odd sizes included), buffers per run, input kind (the synthetic workloads, plus
saturated / sawtooth / constant / uniformly random bytes), preamble threshold, --no-fix / --no-fix-df, Mode A/C on or off, the
ICAO filter's flip period (down to a few ms of stream time: flips inside a run), a ragged tail, and one of the entry paths
(host submits, magnitude hand-off, sc16 / sc16q11 input, device-resident blocking, device-resident pipelined, pipelined host
slab, or independent receivers through the _rx calls with their own counts, restarts and thresholds).  Frames, per-buffer results, counters, Mode A/C replies and (sometimes) the Beast byte stream must equal the oracle's.
Prints the failing case's parameters (re-run it alone with --only K).  The same script works on a GPU (without B200_EMU).
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def make_input(rng, kind: str, n: int, seed: int):
    import numpy as np
    from readsb_b200 import synth
    if kind == "cfg2":
        return synth.config2_stream(seed, n)
    if kind == "cfg5":
        return synth.config5_stream(seed, n)
    if kind == "mixed":
        return synth.mixed_stream(seed, n, frames_per_sec=float(rng.choice([500, 2000, 6000])))
    if kind == "modeac":
        return synth.modeac_stream(seed, n)
    if kind == "loud":      # strong overlapping traffic close to clipping
        return synth.generate(n, seed=seed, frames_per_sec=8000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP | synth.MODEAC, n_icao=8,
                              amp=(0.7, 1.0), p_bit_error=0.3)
    if kind == "synthrand":     # the generator with every knob drawn at random
        mask = 0
        for bit in (synth.DF17, synth.DF11, synth.AP, synth.DF18, synth.DF11_IID, synth.MODEAC):
            if rng.random() < 0.5:
                mask |= bit
        lo = float(rng.uniform(0.02, 0.6))
        return synth.generate(n, seed=seed, frames_per_sec=float(10 ** rng.uniform(1.5, 4.3)), df_mask=mask or synth.DF17, n_icao=int(rng.integers(1, 200)),
                              amp=(lo, float(rng.uniform(lo, 1.0))), noise_sigma=float(rng.uniform(0.2, 12.0)), p_bit_error=float(rng.uniform(0, 0.6)),
                              p_two_bit_error=float(rng.uniform(0, 0.2)))
    if kind == "random":
        return rng.integers(0, 256, size=2 * n, dtype=np.uint8)
    if kind == "sawtooth":
        return (np.arange(2 * n, dtype=np.uint32) * int(rng.integers(1, 9)) % 256).astype(np.uint8)
    if kind == "constant":
        return np.full(2 * n, int(rng.choice([0, 127, 128, 255])), dtype=np.uint8)
    if kind == "burst":     # quiet, then a block of saturated samples, then traffic
        iq = synth.mixed_stream(seed, n)
        a = int(rng.integers(0, max(1, n - 5000)))
        iq[2 * a: 2 * (a + int(rng.integers(10, 5000)))] = rng.integers(0, 2, dtype=np.uint8) * 255
        return iq
    raise ValueError(kind)


def to_sc16(iq8, q11: bool, seed: int):
    """The uc8 capture as a 16-bit frontend would deliver it (plus sub-LSB dither)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    scale = 16 if q11 else 256
    v = (iq8.astype(np.int32) - 128) * scale + rng.integers(0, scale, size=iq8.size)
    return np.clip(v, -2048 if q11 else -32768, 2047 if q11 else 32767).astype(np.int16)


def run_case(k: int, seed: int, verbose: bool, only_path: str | None = None):
    import numpy as np
    import devbuf
    from oraclelib import Oracle
    from paritylib import diff_bufres, diff_frames, diff_stats
    from readsb_b200.demod import Demodulator
    rng = np.random.default_rng([seed, k])
    S = int(rng.choice([1, 1, 2, 3, 5]))
    buf = int(rng.choice([1000, 4096, 8191, 8192, 20000, 32768, 65536, 65536, 131072, int(rng.integers(700, 70000))]))
    path = str(rng.choice(["host", "host", "mag", "device", "device_async", "host_async", "sc16", "host_var", "mixed", "host_ops", "rx"]))
    path = only_path or path
    if path in ("device", "device_async", "host_async"):
        buf = max(8, buf & ~7)                                   # those entry points want multiples of 8
    K = int(rng.choice([1, 2, 3, 4, 8]))
    steps = int(rng.choice([1, 2, 3, 5]))
    kind = str(rng.choice(["cfg2", "cfg5", "mixed", "mixed", "modeac", "loud", "random", "sawtooth", "constant", "burst", "synthrand", "synthrand"]))
    thr = int(rng.choice([58, 58, 58, 40, 75, 120, 33, 400]))
    nfix, fixdf = int(rng.random() < 0.8), int(rng.random() < 0.8)
    mode_ac = bool(rng.random() < 0.4)
    ragged = path in ("host", "mag", "sc16", "mixed") and rng.random() < 0.5
    ttl = int(rng.choice([60000, 60000, 60000, 300, 40, 7]))          # ms of stream time between ICAO filter flips
    q11 = bool(rng.random() < 0.5)
    beast = bool(rng.random() < 0.35)
    verbatim = bool(rng.random() < 0.5)
    total = K * steps * buf - (int(rng.integers(1, buf)) if ragged else 0)
    params = dict(case=k, S=S, buf=buf, K=K, steps=steps, kind=kind, thr=thr, nfix=nfix, fixdf=fixdf, mode_ac=mode_ac, path=path, total=total, ttl=ttl, q11=q11,
                  beast=beast, verbatim=verbatim)
    if verbose:
        print(params, flush=True)
    # device / pipelined paths: at one step the receivers start over (continues = 0: the samples before are not a halo)
    restart_at = int(rng.integers(1, steps)) if path in ("device", "device_async", "host_async") and steps > 1 and rng.random() < 0.35 else -1
    params["restart_at"] = restart_at
    iqs = [make_input(rng, kind, total, 1000 * k + s) for s in range(S)]
    iq16 = [to_sc16(iqs[s], q11, k + s) for s in range(S)] if path == "sc16" else None
    d = Demodulator(n_streams=S, buf_samples=buf, max_buffers_per_run=K, preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, mode_ac=mode_ac,
                    icao_ttl_ms=ttl)
    got_f = [[] for _ in range(S)]; got_b = [[] for _ in range(S)]; got_a = [[] for _ in range(S)]; got_beast = [b"" for _ in range(S)]
    nb_done = [0] * S

    def harvest():
        for s in range(S):
            got_f[s].append(d.frames(s)); b = d.buffer_results(s); got_b[s].append(b)
            if mode_ac:
                a = d.modeac(s); a["buffer_idx"] += nb_done[s]; got_a[s].append(a)
            nb_done[s] += len(b)
            if beast:
                got_beast[s] += d.beast(s, verbatim=verbatim)

    if path == "host_var":      # buffers of random lengths (empty, shorter than the halo, odd), like a frontend that delivers what it has
        import test_gpu_edges as E
        cuts, pos = [], 0
        while pos < total and len(cuts) < 150:
            n = int(min(total - pos, rng.integers(0, buf + 1) if rng.random() < 0.5 else buf))
            if rng.random() < 0.1:
                n = int(min(total - pos, rng.choice([0, 1, 7, 325, 326, 327])))
            cuts.append((pos, pos + n)); pos += n
        problems = []
        for s_ in range(S):
            o = Oracle(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=ttl)
            fo, bo = E._oracle_buffers(o, iqs[s_], cuts, lambda b, lo: lo * 5)
            fgl, bgl, agl, nb0 = [], [], [], 0
            for i in range(0, len(cuts), K):
                part = cuts[i:i + K]
                for lo, hi in part:
                    d.submit_iq(s_, iqs[s_][2 * lo: 2 * hi], lo * 5)
                d.run()
                fgl.append(d.frames(s_)); bgl.append(d.buffer_results(s_))
                if mode_ac:
                    a_ = d.modeac(s_); a_["buffer_idx"] += nb0; agl.append(a_)
                nb0 += len(part)
            problems += [f"stream {s_}: {p}" for p in diff_frames(np.concatenate(fgl), fo) + diff_bufres(np.concatenate(bgl), bo) + diff_stats(d.stats(s_), o.stats())]
            if mode_ac:
                oa, halo, want = Oracle(), np.zeros(326, np.uint16), []
                for b_, (lo, hi) in enumerate(cuts):
                    mag, sl, sp = Oracle.convert(iqs[s_][2 * lo: 2 * hi]) if hi > lo else (np.zeros(0, np.uint16), 0, 0)
                    data = np.concatenate([halo, mag]).astype(np.uint16)
                    a_ = oa.demodulate_ac(data, hi - lo, lo * 5, sl, sp); a_["buffer_idx"] = b_; want.append(a_)
                    halo = data[hi - lo: hi - lo + 326].copy() if hi - lo >= 326 else np.zeros(326, np.uint16)
                ao, ag = np.concatenate(want), np.concatenate(agl)
                if len(ag) != len(ao) or any(not np.array_equal(ag[f], ao[f]) for f in ("timestamp", "f1_sample", "modeac", "buffer_idx")):
                    problems.append(f"stream {s_}: Mode A/C replies differ ({len(ag)} vs {len(ao)})")
        d.close()
        return params, problems, 0
    if path == "host_ops":      # between runs: addresses added to / expired from the filter through the API, the threshold changed
        oracles = [Oracle(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=ttl) for _ in range(S)]
        gf = [[] for _ in range(S)]; of = [[] for _ in range(S)]
        seen = [0x123456]
        nrun = (total + K * buf - 1) // (K * buf)
        for r_ in range(nrun):
            lo, hi = r_ * K * buf, min(total, (r_ + 1) * K * buf)
            for s_ in range(S):
                for o_ in range(lo, hi, buf):
                    d.submit_iq(s_, iqs[s_][2 * o_: 2 * min(hi, o_ + buf)], o_ * 5)
            d.run()
            for s_ in range(S):
                f_ = d.frames(s_); gf[s_].append(f_)
                of[s_].append(oracles[s_].run_stream(iqs[s_][2 * lo: 2 * hi], buf, first_ts=lo * 5)[0])
                seen += [int(a) for a in f_["addr"][:4]]
            for s_ in range(S):
                op = rng.random()
                if op < 0.35:
                    a_ = int(rng.choice(seen)) if rng.random() < 0.7 else int(rng.integers(0, 1 << 24))
                    d.icao_add(s_, a_); oracles[s_].icao_add(a_)
                    if d.icao_test(s_, a_) != oracles[s_].icao_test(a_):
                        return params, [f"stream {s_}: icao_test differs after add"], 0
                elif op < 0.5:
                    d.icao_expire(s_); oracles[s_].icao_expire()
            if rng.random() < 0.3:
                t2 = int(rng.choice([40, 58, 75, 120, 400]))
                d.set_preamble_threshold(t2)
                for o in oracles:
                    o.set_preamble_threshold(t2)
        problems = []
        for s_ in range(S):
            problems += [f"stream {s_}: {p}" for p in diff_frames(np.concatenate(gf[s_]), np.concatenate(of[s_])) + diff_stats(d.stats(s_), oracles[s_].stats())]
        d.close()
        return params, problems, sum(len(np.concatenate(x)) for x in gf)
    if path == "rx":            # independent receivers: per-receiver counts (0 included), clock gaps with restarts, thresholds 0 / 40 / 75
        from test_gpu_rx_steps import FORMATS, _Session
        d.close()
        sess = _Session(str(rng.choice(["device", "device_async", "host"])), int(rng.choice(FORMATS)), S=S, K=K, buf=max(8, buf & ~7), steps=max(steps, 2),
                        depth=int(rng.choice([2, 3])), ttl=ttl, mode_ac=mode_ac, seed=int(rng.integers(1 << 30)))
        params.update(rx_path=sess.path, fmt=sess.fmt, plan=sess.plan)
        try:
            return params, [], sess.run().check(min_frames=0)
        except AssertionError as e:
            return params, [str(e)[:2000]], 0
    if path == "mixed":         # every receiver its own entry point and its own amount of data, all in the same runs
        kinds = [str(rng.choice(["host", "mag", "sc16"])) for _ in range(S)]
        tot = [int(max(1, total * rng.uniform(0.2, 1.0))) for _ in range(S)]
        tot[int(rng.integers(0, S))] = total
        iq16m = [to_sc16(iqs[s_], q11, k + s_) if kinds[s_] == "sc16" else None for s_ in range(S)]
        halos = [np.zeros(326, np.uint16) for _ in range(S)]
        offs = [0] * S
        gf = [[] for _ in range(S)]; gb = [[] for _ in range(S)]; ga = [[] for _ in range(S)]; nbd = [0] * S
        while any(offs[s_] < tot[s_] for s_ in range(S)):
            for _ in range(K):
                for s_ in range(S):
                    if offs[s_] >= tot[s_]:
                        continue
                    m = min(buf, tot[s_] - offs[s_]); o_ = offs[s_]
                    if kinds[s_] == "host":
                        d.submit_iq(s_, iqs[s_][2 * o_: 2 * (o_ + m)], o_ * 5)
                    elif kinds[s_] == "sc16":
                        d.submit_iq_sc16(s_, iq16m[s_][2 * o_: 2 * (o_ + m)], o_ * 5, q11)
                    else:
                        mag, _, _ = Oracle.convert(iqs[s_][2 * o_: 2 * (o_ + m)])
                        data = np.concatenate([halos[s_], mag]).astype(np.uint16)
                        d.submit_mag(s_, data, m, o_ * 5)
                        halos[s_] = data[m: m + 326].copy() if m >= 326 else np.zeros(326, np.uint16)
                    offs[s_] += m
            d.run()
            for s_ in range(S):
                gf[s_].append(d.frames(s_)); b_ = d.buffer_results(s_); gb[s_].append(b_)
                if mode_ac:
                    a_ = d.modeac(s_); a_["buffer_idx"] += nbd[s_]; ga[s_].append(a_)
                nbd[s_] += len(b_)
        problems = []
        for s_ in range(S):
            o = Oracle(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=ttl)
            fgc, bgc = np.concatenate(gf[s_]), np.concatenate(gb[s_])
            if kinds[s_] == "sc16":
                fo, sums = o.run_stream_sc16(iq16m[s_][:2 * tot[s_]], buf, q11)
                problems += [f"stream {s_} ({kinds[s_]}): {p}" for p in diff_frames(fgc, fo)]
                if len(bgc) != len(sums) or any(r["length"] != m or np.uint32(r["sum_level"]).view(np.float32) != sl or np.uint32(r["sum_power"]).view(np.float32) != sp
                                                for r, (m, sl, sp) in zip(bgc, sums)):
                    problems.append(f"stream {s_}: sc16 float sums differ")
                ao = Oracle().run_stream_ac_sc16(iq16m[s_][:2 * tot[s_]], buf, q11) if mode_ac else None
            else:
                fo, bo = o.run_stream(iqs[s_][:2 * tot[s_]], buf)
                problems += [f"stream {s_} ({kinds[s_]}): {p}" for p in diff_frames(fgc, fo) + diff_bufres(bgc, bo)]
                ao = Oracle().run_stream_ac(iqs[s_][:2 * tot[s_]], buf) if mode_ac else None
            problems += [f"stream {s_} ({kinds[s_]}): {p}" for p in diff_stats(d.stats(s_), o.stats())]
            if mode_ac:
                ag = np.concatenate(ga[s_])
                if len(ag) != len(ao) or any(not np.array_equal(ag[f], ao[f]) for f in ("timestamp", "f1_sample", "modeac", "buffer_idx")):
                    problems.append(f"stream {s_} ({kinds[s_]}): Mode A/C replies differ ({len(ag)} vs {len(ao)})")
        d.close()
        return params, problems, sum(len(np.concatenate(x)) for x in gf)
    if path == "sc16":
        off = 0
        while off < total:
            for _ in range(K):
                if off >= total:
                    break
                m = min(buf, total - off)
                for s in range(S):
                    d.submit_iq_sc16(s, iq16[s][2 * off: 2 * (off + m)], off * 5, q11)
                off += m
            d.run(); harvest()
    elif path in ("host", "mag"):
        halos = [np.zeros(326, np.uint16) for _ in range(S)]
        off = 0
        use_strided = path == "host" and rng.random() < 0.4
        mag_levels = path == "mag" and mode_ac and rng.random() < 0.6
        level_scale = (float(rng.uniform(0.5, 2.0)), float(rng.uniform(0.5, 3.0)))
        given = [[] for _ in range(S)]
        slab = np.stack(iqs) if use_strided else None             # [S, 2 * total]: receiver s at slab + s * row stride
        while off < total:
            if use_strided:                                        # all receivers in one strided DMA: K full buffers, or the partial tail
                nfull = min(K, (total - off) // buf)
                nb_, bl_ = (nfull, buf) if nfull else (1, total - off)
                d.submit_iq_strided(0, S, slab.ctypes.data + 2 * off, slab.strides[0], nb_, bl_, off * 5)
                off += nb_ * bl_
                d.run(); harvest()
                continue
            for _ in range(K):
                if off >= total:
                    break
                m = min(buf, total - off)
                for s in range(S):
                    if path == "host":
                        d.submit_iq(s, iqs[s][2 * off: 2 * (off + m)], off * 5)
                    else:
                        mag, sl_, sp_ = Oracle.convert(iqs[s][2 * off: 2 * (off + m)])
                        data = np.concatenate([halos[s], mag]).astype(np.uint16)
                        if mag_levels and m:        # the mag_buf's own mean_level / mean_power: exact ones, or (receiver 0) distorted ones
                            ml, mp = sl_ / 65536.0 / m, sp_ / 65535.0 / 65535.0 / m
                            if s == 0:
                                ml, mp = ml * level_scale[0], mp * level_scale[1]
                            d.submit_mag(s, data, m, off * 5, ml, mp)
                            given[s].append((data.copy(), m, off * 5, ml, mp))
                        else:
                            d.submit_mag(s, data, m, off * 5)
                            given[s].append((data.copy(), m, off * 5, None, None))
                        halos[s] = data[m: m + 326].copy() if m >= 326 else np.zeros(326, np.uint16)
                off += m
            d.run(); harvest()
    elif path in ("device", "device_async"):
        pad, stride = 1024, 2 * total + 4096
        dev = devbuf.zeros(pad + S * stride)
        for s in range(S):
            dev[pad + s * stride: pad + s * stride + 2 * total] = devbuf.to_dev(iqs[s])
        devbuf.sync()
        flying = 0
        for c in range(steps):
            args = (dev.data_ptr() + pad + c * K * buf * 2, stride, K, buf)
            if path == "device":
                d.run_device(*args, continues=c > 0 and c != restart_at, first_sample_timestamp=c * K * buf * 5); harvest()
            else:
                d.run_device_async(*args, continues=c > 0 and c != restart_at, first_sample_timestamp=c * K * buf * 5); flying += 1
                if flying == 3:
                    d.wait(); harvest(); flying -= 1
        while path == "device_async" and flying:
            d.wait(); harvest(); flying -= 1
    else:   # host_async
        from readsb_b200.demod import PinnedBuffer
        row = 2 * K * buf
        slabs = [PinnedBuffer(S * row) for _ in range(3)]
        flying = 0
        for c in range(steps):
            sl = slabs[c % 3]
            for s in range(S):
                sl.array[s * row: (s + 1) * row] = iqs[s][c * row: (c + 1) * row]
            d.run_host_async(sl.ptr, row, K, buf, continues=c > 0 and c != restart_at, first_sample_timestamp=c * K * buf * 5); flying += 1
            if flying == 3:
                d.wait(); harvest(); flying -= 1
        while flying:
            d.wait(); harvest(); flying -= 1
        for sl in slabs:
            sl.free()

    problems = []
    for s in range(S):
        o = Oracle(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=ttl)
        ao = None
        if path == "sc16":
            fo, sums = o.run_stream_sc16(iq16[s], buf, q11)
            bg = np.concatenate(got_b[s])
            problems += [f"stream {s}: {p}" for p in diff_frames(np.concatenate(got_f[s]), fo)]
            if len(bg) != len(sums) or any(r["length"] != m or np.uint32(r["sum_level"]).view(np.float32) != sl or np.uint32(r["sum_power"]).view(np.float32) != sp
                                           for r, (m, sl, sp) in zip(bg, sums)):
                problems.append(f"stream {s}: sc16 float sums differ")
        elif restart_at > 0:
            cut = restart_at * K * buf
            f1, b1 = o.run_stream(iqs[s][:2 * cut], buf)
            o.restart_stream()
            f2, b2 = o.run_stream(iqs[s][2 * cut:], buf, first_ts=cut * 5)
            fo, bo = np.concatenate([f1, f2]), np.concatenate([b1, b2])
            problems += [f"stream {s}: {p}" for p in diff_frames(np.concatenate(got_f[s]), fo) + diff_bufres(np.concatenate(got_b[s]), bo)]
        else:
            fo, bo = o.run_stream(iqs[s], buf)
            problems += [f"stream {s}: {p}" for p in diff_frames(np.concatenate(got_f[s]), fo) + diff_bufres(np.concatenate(got_b[s]), bo)]
        st = d.stats(s)
        if mode_ac:
            if path == "mag" and mag_levels:
                oa, parts = Oracle(), []
                for b_, (data_, m_, ts_, ml_, mp_) in enumerate(given[s]):
                    if ml_ is None:
                        a_ = oa.demodulate_ac(data_, m_, ts_, int(data_[326:326 + m_].astype(np.uint64).sum()), int((data_[326:326 + m_].astype(np.uint64) ** 2).sum()))
                    else:
                        a_ = oa.demodulate_ac_levels(data_, m_, ts_, ml_, mp_)
                    a_["buffer_idx"] = b_; parts.append(a_)
                ao = np.concatenate(parts)
            elif restart_at > 0:
                cut = restart_at * K * buf
                a1 = Oracle().run_stream_ac(iqs[s][:2 * cut], buf)
                a2 = Oracle().run_stream_ac(iqs[s][2 * cut:], buf, first_ts=cut * 5); a2["buffer_idx"] += restart_at * K
                ao = np.concatenate([a1, a2])
            else:
                ao = Oracle().run_stream_ac_sc16(iq16[s], buf, q11) if path == "sc16" else Oracle().run_stream_ac(iqs[s], buf)
            ag = np.concatenate(got_a[s])
            if len(ag) != len(ao) or any(not np.array_equal(ag[f], ao[f]) for f in ("timestamp", "f1_sample", "modeac", "buffer_idx")):
                problems.append(f"stream {s}: Mode A/C replies differ ({len(ag)} vs {len(ao)})")
            if st["demod_modeac"] != len(ao):
                problems.append(f"stream {s}: demod_modeac {st['demod_modeac']} vs {len(ao)}")
        problems += [f"stream {s}: {p}" for p in diff_stats(st, o.stats())]
        if beast and got_beast[s] != Oracle.beast(fo, ao, verbatim=verbatim):
            problems.append(f"stream {s}: Beast output differs")
    nframes = sum(len(np.concatenate(x)) for x in got_f)
    d.close()
    return params, problems, nframes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--cases", type=int, default=50)
    ap.add_argument("--minutes", type=float, default=0.0, help="stop after this many minutes (0 = run all cases)")
    ap.add_argument("--only", type=int, default=-1)
    ap.add_argument("--emu", type=int, default=1, help="1: the emulated library (default), 0: the sm_90a library on a GPU")
    ap.add_argument("--path", help="every case on this entry path (the other draws stay as they are)")
    ap.add_argument("-v", action="store_true")
    a = ap.parse_args()
    if a.emu:
        os.environ["B200_EMU"] = "1"
        sys.path.insert(0, str(ROOT / "tests" / "emu"))
        import build_emu
        os.environ["B200_DEMOD_LIB"] = os.environ.get("B200_EMU_LIB") or str(build_emu.build())
    t0, bad, frames = time.time(), 0, 0
    ks = [a.only] if a.only >= 0 else range(a.cases)
    for k in ks:
        params, problems, nf = run_case(k, a.seed, a.v, a.path)
        frames += nf
        if problems:
            bad += 1
            print("FAIL", params)
            for p in problems[:8]:
                print("   ", p)
        if a.minutes and time.time() - t0 > a.minutes * 60:
            print(f"time limit after case {k}")
            break
    print(f"{len(list(ks))} cases requested, {bad} failed, {frames} frames compared, {time.time() - t0:.0f} s")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
