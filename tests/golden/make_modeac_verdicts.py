"""Generates tests/golden/verdicts/modeac_verdicts.npz: crafted captures for the Mode A/C demodulator (demodulate2400AC,
demod_2400.c:575-761) and what the REFERENCE ITSELF (oracle/_ref/libreadsb_ref.so, built from the reference tree by
oracle/Makefile) returned for them.  Only runs where the reference library can be built; the committed fixture is the
authority elsewhere.

    python tests/golden/make_modeac_verdicts.py

Replies are drawn sample by sample, because the comparisons they are made to tie are on exact sample values.  A reply whose F1
pulse starts at f1_sample j is fixed by its F1 pair (a0, a1) = (m[j], m[j + 1]): they set the clock phase
f1_clock = (unsigned)(25 * (j + fraction^2) + 0.5), computed here in float32 exactly as the C expression does, and bit k of
the reply is read from the cell m[s], m[s + 1], m[s + 2] at s = (f1_clock + 87 k) / 25 (s + 2: the quiet sample).  `decide`
restates the reference's test of one position and `scan` its walk over a buffer; the generator asserts that the reference
agrees with both, and that every case meets the class it was drawn for.

Captures (magnitudes, and uc8 I/Q whose table magnitudes are the nearest to those; ties only mean something in magnitudes):
  a    verdicts and ties: one case per 1024-sample buffer, each with its own caller-given noise floor (mean_level /
       mean_power, as b200_demod_submit_mag_u16_levels takes them);
  b    noise floors: the same reply under floors at level / 2 and level / 2 + 1, in [2^31, 2^32) (the 32-bit wrap of
       noise * 2 and of noise * f1f2_level), at and beyond 2^32, NaN and inf; also fed with the buffers' own sums, and as sc16 /
       sc16q11 I/Q through the reference's float-accumulating converters, with one near-constant buffer whose float variance
       is negative;
  c*   placement: buffers of 65536, 100, 300, 400, 1000, 8191 and 20000 samples, and one of 2^20 + 333: f1_sample 0 / 1 / 2, the
       last positions of buffers, the skip at 69 / 70 / 71 positions, replies across 2048-position scan tiles and into the
       look-ahead, tiles over many buffers with different noise floors, a densest-packed buffer, a chunk with more than 32
       front-test survivors, a buffer with a zero halo, clock phases at j past 2^17 and 2^20, and DF17 frames next to replies.
"""
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from readsb_b200.abi import MODEAC_DTYPE  # noqa: E402

OUT = HERE / "verdicts" / "modeac_verdicts.npz"
HALO = 326
LA = 1024
BG = 100                      # background magnitude of the crafted captures
SQRT2 = 1.41421356237309504880
FRAMING, QUIET = 0x80020, 0x0101B
# reply bit (1 << (19 - k) for bit cell k) -> Mode A/C code bit (demod_2400.c:716-731)
CODE_MAP = {0x40000: 0x0010, 0x20000: 0x1000, 0x10000: 0x0020, 0x08000: 0x2000, 0x04000: 0x0040, 0x02000: 0x4000,
            0x00800: 0x0100, 0x00400: 0x0001, 0x00200: 0x0200, 0x00100: 0x0002, 0x00080: 0x0400, 0x00040: 0x0004,
            0x00004: 0x0080}
QUIET_BITS = (0x01000, 0x00010, 0x00008, 0x00002, 0x00001)
CONDITIONS = ("edge1", "quiet1", "level1", "edge2", "quiet2", "level2", "framing", "quiet_bits", "noisy", "uncertain")
C_BUFS = {"c65536": 65536, "c100": 100, "c300": 300, "c400": 400, "c1000": 1000, "c8191": 8191, "c20000": 20000, "cbig": (1 << 20) + 333}


# ---- the reference's arithmetic ----------------------------------------------------------------------------------------
def u32_x86(x: float) -> int:
    """(unsigned)x of a double as the x86-64 build evaluates it (a 64-bit cvttsd2si, truncated): 0 for NaN and >= 2^63."""
    return int(x) & 0xFFFFFFFF if (x == x and 0 <= x < 2.0 ** 63) else 0


def noise_floor(ml: float, mp: float) -> int:
    """demod_2400.c:580-581."""
    with np.errstate(invalid="ignore"):
        sd = np.sqrt(np.float64(mp) - np.float64(ml) * np.float64(ml))
    return u32_x86(float((np.float64(mp) + sd) * 65535 + 0.5))


def sums_levels(new: np.ndarray):
    """mean_level / mean_power of the uc8 converter from a buffer's exact integer sums (convert.c:100-106)."""
    n = new.size
    sl, sp = int(new.astype(np.uint64).sum()), int((new.astype(np.uint64) ** 2).sum())
    return float(np.float64(sl) / 65536.0 / n), float(np.float64(sp) / 65535.0 / 65535.0 / n)


def clock_x(j: int, a0: int, a1: int) -> np.float32:
    """25 * (f1_sample + fraction^2), the float the reference rounds (demod_2400.c:651-654)."""
    fa, fb = np.float32(a0) * np.float32(a0), np.float32(a1) * np.float32(a1)
    fr = fb / (fa + fb)
    return np.float32(25) * (np.float32(j) + fr * fr)


def f1_clock(j: int, a0: int, a1: int) -> int:
    return u32_x86(float(np.float64(clock_x(j, a0, a1)) + 0.5))


def thresholds(noise: int, f1f2: int):
    mid = np.sqrt(np.float32((noise * f1f2) & 0xFFFFFFFF))
    return u32_x86(float(np.float64(mid) * SQRT2 + 0.5)), u32_x86(float(np.float64(mid) / SQRT2 + 0.5))


def decide(m, j: int, noise: int) -> dict:
    """Every condition of demodulate2400AC at f1_sample j, each evaluated on its own (True: passes), with the clock and code."""
    v = lambda k: int(m[k])                                                      # noqa: E731
    a0, a1, a2 = v(j), v(j + 1), v(j + 2)
    c = {"edge1": v(j - 1) < a0, "quiet1": a2 <= a0 and a2 <= a1}
    f1l = (a0 + a1) // 2
    c["level1"] = not ((noise * 2) & 0xFFFFFFFF) > f1l
    clock = f1_clock(j, a0, a1) if a0 or a1 else 25 * j
    f2 = (clock + 87 * 14) // 25
    b0, b1, b2 = v(f2), v(f2 + 1), v(f2 + 2)
    c["edge2"], c["quiet2"] = v(f2 - 1) < b0, b2 <= b0 and b2 <= b1
    f2l = (b0 + b1) // 2
    c["level2"] = not ((noise * 2) & 0xFFFFFFFF) > f2l
    sig, noi = thresholds(noise, max(f1l, f2l))
    bits = noisy = unc = 0
    for bit in range(20):
        s = (clock + 87 * bit) // 25
        bits, noisy, unc = bits << 1, noisy << 1, unc << 1
        if v(s + 2) >= sig:
            noisy |= 1
        if v(s) >= sig or v(s + 1) >= sig:
            bits |= 1
        elif v(s) > noi and v(s + 1) > noi:
            unc |= 1
    c.update(framing=(bits & FRAMING) == FRAMING, quiet_bits=(bits & QUIET) == 0, noisy=noisy == 0, uncertain=unc == 0)
    code = 0
    for b, cb in CODE_MAP.items():
        if bits & b:
            code |= cb
    return dict(ok=all(c[k] for k in CONDITIONS), cond=c, clock=clock, code=code, bits=bits, sig=sig, noi=noi, f1f2=max(f1l, f2l))


def scan(data: np.ndarray, mlen: int, noise: int) -> list:
    """demodulate2400AC's walk over one mag_buf: [(f1_sample, f1_clock, code)]."""
    d = data.astype(np.int64)
    # the positions that pass the first test at all (a rising edge whose third sample is quiet)
    j = np.arange(1, mlen)
    cand = set(j[(d[j - 1] < d[j]) & (d[j + 2] <= d[j]) & (d[j + 2] <= d[j + 1])].tolist())
    out, k = [], 1
    while k < mlen:
        if k in cand:
            r = decide(d, k, noise)
            if r["ok"]:
                out.append((k, r["clock"], r["code"]))
                k += 20 * 87 // 25
        k += 1
    return out


# ---- drawing -----------------------------------------------------------------------------------------------------------------
def word_of(code: int) -> int:
    """The reply bits (F1 and F2 on) that carry Mode A/C code `code`."""
    w = FRAMING
    for b, cb in CODE_MAP.items():
        if code & cb:
            w |= b
    return w


def cells(j: int, clock: int) -> list:
    return [(clock + 87 * k) // 25 - j for k in range(20)]


def draw(m: np.ndarray, base: int, j: int, a0: int, a1: int, word: int, hi: int = 5000, f2=None, lo: int = BG) -> int:
    """A reply at f1_sample j of the buffer whose data index 0 is m[base]: F1 pair (a0, a1), on-cells (hi, hi, lo), off-cells
    lo, F2 pair f2 (default (hi, hi)).  Returns its f1_clock."""
    clock = f1_clock(j, a0, a1)
    g = base + j
    m[g - 1: g + 72] = lo
    for k, s in enumerate(cells(j, clock)):
        if k and word & (1 << (19 - k)):              # (cell 0 is F1 itself: a0, a1 and a quiet m[j + 2])
            m[g + s], m[g + s + 1] = hi, hi
    s14 = cells(j, clock)[14]
    if f2 is not None:
        m[g + s14], m[g + s14 + 1] = f2
    m[g], m[g + 1] = a0, a1
    return clock


def given_levels(noise: int):
    """(mean_level, mean_power) whose floor before the 32-bit conversion is exactly `noise`: mean_level 0, so the floor is
    (mp + sqrt(mp)) * 65535 + 0.5, and mean_power is bisected to the smallest double that reaches it."""
    raw = lambda mp: int((np.float64(mp) + np.sqrt(np.float64(mp))) * 65535 + 0.5)      # noqa: E731
    lo, hi = 0.0, noise / 65535.0 + 1.0
    while True:
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            break
        lo, hi = (lo, mid) if raw(mid) >= noise else (mid, hi)
    assert raw(hi) == noise, noise
    return 0.0, hi


def phase_pairs(j: int) -> dict:
    """For every clock phase offset f1_clock - 25 j in 0..25, an F1 pair (a0, a1) that gives it at f1_sample j."""
    out = {}
    for a1 in range(200, 6001, 100):
        for a0 in (6000, 3000, 1500, 600, 300, 150):
            if a0 <= BG or max(a0, a1) < 3000:
                continue
            o = f1_clock(j, a0, a1) - 25 * j
            out.setdefault(o, (a0, a1))
    assert sorted(out) == list(range(26)), sorted(out)
    return out


def strong_pairs(j: int) -> list:
    """F1 pairs for every phase offset 0..25 (index = offset) with a level of at least 8000: above the floors that busy
    buffers' own sums give (capture c)."""
    out = {}
    for a1 in range(500, 65001, 250):
        for a0 in (30000, 20000, 12000, 8000, 6000, 4000, 3000):
            if (a0 + a1) // 2 >= 8000:
                out.setdefault(f1_clock(j, a0, a1) - 25 * j, (a0, a1))
    assert sorted(out) == list(range(26)), sorted(out)
    return [out[o] for o in range(26)]


def half_ties(j: int, limit: int = 4000, count: int = 6) -> list:
    """F1 pairs whose 25 * (j + fraction^2) is exactly k + 0.5 in float32 (round_half_up's tie), both F2 offsets included."""
    a = np.arange(BG + 1, limit, dtype=np.float32)
    found = []
    for a0 in range(3000, 3000 + 4 * count * 50, 50):
        fa = np.float32(a0) * np.float32(a0)
        fb = a * a
        fr = fb / (fa + fb)
        x = np.float32(25) * (np.float32(j) + fr * fr)
        hit = np.nonzero((x - np.floor(x)) == np.float32(0.5))[0]
        for i in hit[:2]:
            found.append((a0, int(a[i])))
        if len(found) >= count:
            break
    return found


# ---- capture a: verdicts and ties ---------------------------------------------------------------------------------------------
class Cases:
    """Capture a's cases: name, expected class ("accepted:<code>" or "rejected:<the condition it fails>"), the buffer's noise
    floor, and the function that draws the case into its buffer."""

    def __init__(self):
        self.cases, self.noise, self.build = [], [], []

    def add(self, name, expect, noise, build, **info):
        self.cases.append(dict(name=name, expect=expect, **info))
        self.noise.append(noise)
        self.build.append(build)


def capture_a():
    """One reply per 1024-sample buffer at f1_sample J_A, each buffer with its own given noise floor."""
    J = 400
    T = Cases()
    std = dict(a0=5000, a1=5000)

    def reply(word, a0=5000, a1=5000, hi=5000, f2=None, edit=None):
        def build(m, base):
            clock = draw(m, base, J, a0, a1, word, hi=hi, f2=f2)
            if edit:
                edit(m, base + J, cells(J, clock), clock)
        return build

    N = 400                                   # floor of the plain cases: signal threshold 2000, noise threshold 1000 at level 5000
    # codes: none, every code bit alone, all of them
    T.add("code_none", "accepted:0000", N, reply(word_of(0)))
    for b, cb in CODE_MAP.items():
        T.add(f"code_bit_{cb:04x}", f"accepted:{cb:04x}", N, reply(word_of(cb)))
    allc = sum(CODE_MAP.values())
    T.add("code_all", f"accepted:{allc:04x}", N, reply(word_of(allc)))
    # every clock phase offset (F2 48 samples on for offsets 0..6, 49 for 7..25), with a code that changes with the phase
    for o, (a0, a1) in sorted(phase_pairs(J).items()):
        code = (0x1234 + 0x111 * o) & allc
        T.add(f"phase_{o}", f"accepted:{code:04x}", N, reply(word_of(code), a0, a1), phase=o)
    for a0, a1 in half_ties(J):
        T.add(f"phase_half_tie_{a0}_{a1}", "accepted:0605", N, reply(word_of(0x0605), a0, a1), phase=f1_clock(J, a0, a1) - 25 * J)
    # F1 / F2 rising edge: m[-1] < m[0] (a tie fails)
    def set_at(off_fn, val_fn):
        def edit(m, g, cs, clock):
            m[g + off_fn(cs)] = val_fn(m, g, cs)
        return edit
    # (m[j - 2] a little lower than the tie, so that j - 1 is no candidate whose quiet sample passes and j + 1 no rising edge)
    for tag, cls, d in (("tie", "rejected:edge1", 0), ("below", "accepted:0102", 1)):
        T.add(f"edge1_{tag}", cls, N, reply(word_of(0x0102), 6000, 3000, edit=lambda m, g, cs, c, d=d: _pair(m, g, -2, 5990, 6000 - d)))
    # F2 edge just below the signal threshold (m[f2 - 1] may be the quiet sample of bit 13): F1 at 6000 fixes f1f2 = 6000, signal
    # threshold 2191
    sig6 = thresholds(N, 6000)[0]
    T.add("edge2_tie", "rejected:edge2", N, reply(word_of(0x0040), 6000, 6000, f2=(sig6 - 1, 5000),
                                                   edit=set_at(lambda cs: cs[14] - 1, lambda m, g, cs: m[g + cs[14]])))
    T.add("edge2_below", "accepted:0040", N, reply(word_of(0x0040), 6000, 6000, f2=(sig6 - 1, 5000),
                                                   edit=set_at(lambda cs: cs[14] - 1, lambda m, g, cs: m[g + cs[14]] - 1)))
    # quiet third sample of F1 / F2: <= each of the first two (the smaller one below the signal threshold 2000)
    for tag, (a0, a1) in (("a0", (1500, 6000)), ("a1", (6000, 1500))):
        small = min(a0, a1)
        # (a0 < a1: the gap sample m[j + 3] just above m[j + 2], so that j + 1 fails its own quiet test rather than taking the reply)
        for d, cls in ((0, "accepted:0200"), (1, "rejected:quiet1")):
            T.add(f"quiet1_{'tie' if d == 0 else 'above'}_{tag}", cls, N,
                  reply(word_of(0x0200), a0, a1, edit=lambda m, g, cs, c, v=small + d, g3=a0 < a1: _pair(m, g, 2, v, 1502 if g3 else BG)))
    for tag, pair in (("b0", (1500, 5000)), ("b1", (5000, 1500))):
        small = min(pair)
        T.add(f"quiet2_tie_{tag}", "accepted:0004", N, reply(word_of(0x0004), f2=pair, edit=set_at(lambda cs: cs[14] + 2, lambda m, g, cs: small)))
        T.add(f"quiet2_above_{tag}", "rejected:quiet2", N, reply(word_of(0x0004), f2=pair, edit=set_at(lambda cs: cs[14] + 2, lambda m, g, cs: small + 1)))
    # levels 6 dB above the floor: noise * 2 > level fails on a tie.  Floor 1000, F1 and F2 at level 2000 (threshold 2000)
    NL = 1000
    T.add("level1_tie", "accepted:1000", NL, reply(word_of(0x1000), 2000, 2000, f2=(2000, 2000)))
    T.add("level1_below", "rejected:level1", NL, reply(word_of(0x1000), 2000, 1999, f2=(2000, 2000)))
    T.add("level2_tie", "accepted:1000", NL, reply(word_of(0x1000), 2000, 2000, f2=(2000, 2000), hi=2001))
    T.add("level2_below", "rejected:level2", NL, reply(word_of(0x1000), 2000, 2000, f2=(2000, 1999)))
    # bit decision at the signal threshold (s0 or s1 >= it: on), quiet sample at it (noisy), and the uncertain band (both > the
    # noise threshold 1000)
    sig, noi = thresholds(N, 5000)
    k_a1 = 2                                    # bit cell of A1 (reply bit 0x20000)

    def cell_edit(k, q, val):
        return set_at(lambda cs: cs[k] + q, lambda m, g, cs: val)
    for q in (0, 1):
        T.add(f"bit_s{q}_at_signal_threshold", "accepted:1000", N, reply(word_of(0), edit=lambda m, g, cs, c, q=q: _cell(m, g, cs[k_a1], q, sig)))
        T.add(f"bit_s{q}_below_signal_threshold", "accepted:0000", N, reply(word_of(0), edit=lambda m, g, cs, c, q=q: _cell(m, g, cs[k_a1], q, sig - 1)))
    for k in (3, 13, 19):
        T.add(f"quiet_sample_{k}_at_signal_threshold", "rejected:noisy", N, reply(word_of(0x0010), edit=cell_edit(k, 2, sig)))
        T.add(f"quiet_sample_{k}_below_signal_threshold", "accepted:0010", N, reply(word_of(0x0010), edit=cell_edit(k, 2, sig - 1)))
    for k in (4, 11):
        T.add(f"uncertain_{k}_at_noise_threshold", "accepted:0000", N, reply(word_of(0), edit=lambda m, g, cs, c, k=k: _pair(m, g, cs[k], noi, noi)))
        T.add(f"uncertain_{k}_above_noise_threshold", "rejected:uncertain", N, reply(word_of(0), edit=lambda m, g, cs, c, k=k: _pair(m, g, cs[k], noi + 1, noi + 1)))
        T.add(f"uncertain_{k}_s0_above", "accepted:0000", N, reply(word_of(0), edit=lambda m, g, cs, c, k=k: _pair(m, g, cs[k], noi + 1, noi)))
        T.add(f"uncertain_{k}_s1_above", "accepted:0000", N, reply(word_of(0), edit=lambda m, g, cs, c, k=k: _pair(m, g, cs[k], noi, noi + 1)))
    # framing pulses missing one at a time, quiet bits set one at a time
    sigh = thresholds(N, 8000)
    T.add("framing_f1_off", "rejected:framing", N, reply(word_of(0x0001), sigh[0] - 30, sigh[1] - 5, f2=(8000, 8000), hi=8000))
    T.add("framing_f2_off", "rejected:framing", N, reply(word_of(0x0001), 8000, 8000, f2=(sigh[0] - 30, sigh[1] - 5), hi=8000))
    for qb in QUIET_BITS:
        T.add(f"quiet_bit_{qb:05x}_set", "rejected:quiet_bits", N, reply(word_of(0x0400) | qb))
    T.add("noisy_only", "rejected:noisy", N, reply(word_of(0x0400), edit=cell_edit(8, 2, 5000)))
    T.add("uncertain_only", "rejected:uncertain", N, reply(word_of(0x0400), edit=lambda m, g, cs, c: _pair(m, g, cs[9], (sig + noi) // 2, (sig + noi) // 2)))
    # magnitudes 0 and 65535
    T.add("extremes", f"accepted:{0x7777 & allc:04x}", N, lambda m, base: draw(m, base, J, 65535, 65535, word_of(0x7777 & allc), hi=65535, lo=0))
    n = len(T.cases)
    m = np.full(n * LA, BG, np.uint16)
    for i, build in enumerate(T.build):
        base = i * LA - HALO
        build(m, base)
        T.cases[i].update(buffer=i, j=J, noise=T.noise[i])
    levels = np.array([given_levels(N_) for N_ in T.noise], np.float64)
    return T.cases, m, levels


def _cell(m, g, s, q, val):
    m[g + s + q] = val


def _pair(m, g, s, v0, v1):
    m[g + s], m[g + s + 1] = v0, v1


# ---- capture b: noise floors --------------------------------------------------------------------------------------------------
def capture_b():
    """The same kind of reply (level 5000, or 5001 where the product has to be odd) under given floors: (name, floor before the
    32-bit conversion, level, class).  Then mean levels whose floor is NaN (a variance below zero) or inf; both convert to 0, and a
    floor of 0 makes every sample a noisy quiet sample."""
    J = 400
    cases, lv = [], []
    plan = [("half_level", 2500, 5000, "accepted"), ("half_level_plus1", 2501, 5000, "rejected:level1"),
            ("quarter_level", 1250, 5000, "accepted"),
            ("wrap2_even", (1 << 31) + 400, 5000, "accepted"), ("wrap2_even_high", (1 << 31) + 2600, 5000, "rejected:level1"),
            ("wrap2_odd", (1 << 31) + 400, 5001, "any"), ("wrap2_top", 0xFFFFFFFF, 5000, "any"),
            ("beyond_2_32", (1 << 32) + 1000, 5000, "accepted"), ("beyond_2_32_high", (1 << 32) + 2600, 5000, "rejected:level1"),
            ("far_beyond", (1 << 40) + 300, 5000, "accepted"), ("huge", None, 5000, "rejected:noisy")]
    special = {"nan": (0.5, 0.2), "inf": (0.0, float("inf")), "neg_var_tiny": (0.01, 0.0001 * (1 - 1e-15))}
    rows = []
    for name, N, level, cls in plan:
        if N is None:
            rows.append((name, (0.0, 2.0 ** 70), level, cls))      # (mp + sqrt(mp)) * 65535 beyond 2^63: 0 on x86-64
        else:
            rows.append((name, given_levels(N), level, cls))
    for name, (ml, mp) in special.items():
        rows.append((name, (ml, mp), 5000, "rejected:noisy"))
    L = LA
    m = np.full(len(rows) * L, BG, np.uint16)
    for i, (name, (ml, mp), level, cls) in enumerate(rows):
        base = i * L - HALO
        draw(m, base, J, level, level, word_of(0x0652), hi=level, f2=(level, level))
        noise = noise_floor(ml, mp)
        cases.append(dict(name=name, expect=cls if cls != "accepted" else "accepted:0652", buffer=i, j=J, noise=noise))
        lv.append((ml, mp))
    return cases, m, np.array(lv, np.float64)


def sc16_of(mag: np.ndarray, q11: bool) -> np.ndarray:
    """int16 I/Q (Q = 0) whose converted magnitude is the nearest to each magnitude."""
    from oraclelib import Oracle
    top = 2047 if q11 else 32767
    i = np.arange(0, top + 1, dtype=np.int16)
    iq = np.zeros(2 * i.size, np.int16)
    iq[0::2] = i
    table, _, _ = Oracle.convert_sc16(iq, q11)
    pick = np.clip(np.searchsorted(table, mag), 1, table.size - 1)
    pick = np.where(np.abs(table[pick - 1].astype(np.int64) - mag) <= np.abs(table[pick].astype(np.int64) - mag), pick - 1, pick)
    out = np.zeros(2 * mag.size, np.int16)
    out[0::2] = i[pick]
    return out


def negative_variance_buffer(ref, q11: bool, L: int):
    """A constant sc16 buffer whose float mean_power falls below mean_level^2: a NaN noise floor (0 after the conversion)."""
    for c in range(300, 30000, 37):
        iq = sc16_of(np.full(L, c, np.uint16), q11)
        _, ml, mp = ref.convert_sc16(iq, q11)
        if mp - ml * ml < 0:
            return iq
    raise AssertionError("no negative float variance found")


# ---- capture c: placement -----------------------------------------------------------------------------------------------------
def capture_c(name: str, rng):
    """Buffers of C_BUFS[name] samples with replies placed on the edges named in their tags; the reference decides each of them
    (tests/test_modeac_verdicts.py asserts which it must accept).  Returns (buffer length, magnitudes, placed, restart buffers)."""
    L = C_BUFS[name]
    nb = {"c65536": 8, "c100": 60, "c300": 40, "c400": 30, "c1000": 30, "c8191": 10, "c20000": 5, "cbig": 1}[name]
    n = nb * L
    m = np.full(n + 256, BG, np.uint16)
    placed = []                                        # (global f1 position, name)
    restart = []
    pairs = strong_pairs(400)
    busy = np.zeros(n + 256, bool)

    def put(g, tag, k=0, word=None, force=False, pair=None):
        b = (g + HALO) // L
        j = g - b * L + HALO
        a0, a1 = pair or pairs[k % len(pairs)]
        if not force and (g < 1 or busy[max(g - 1, 0): g + 73].any() or g + 80 > n + HALO):
            return False
        draw(m, g - j, j, a0, a1, word if word is not None else word_of((0x0101 * (k + 1) + len(placed)) & 0x7FF7), hi=max(a0, a1), lo=BG)
        busy[max(g - 1, 0): g + 73] = True
        placed.append((g, tag))
        return True

    g_of = lambda b, j: b * L - HALO + j                                           # noqa: E731
    if name == "c65536":
        # (one feature per buffer boundary: a reply at j = 0 .. 2 reads its predecessor's last samples)
        for b, j in ((4, 0), (2, 1), (5, 2)):
            put(g_of(b, j), f"f1_sample_{j}_buf{b}", k=j)
        for b, j in ((5, L - 1), (2, L - 70)):
            put(g_of(b, j), f"last_{j}_buf{b}", k=b)
        # a densest-packed buffer: replies at j = 1 + 70 k
        # (F1 and F2 only, at 30000: the buffer's own floor is high)
        for j in range(1, L, 70):
            put(g_of(7, j), "dense", word=FRAMING, pair=(30000, 30000), force=True)
        # pairs at the skip: the second reply 69 (hidden), 70 and 71 positions after the first
        for i, d in enumerate((69, 70, 71)):
            g = g_of(1, 5000 + 1000 * i)
            put(g, f"skip_first_{d}", k=0, force=True)
            put(g + d, f"skip_second_{d}", k=3, force=True)
        # the skip of a reply near the end of a buffer does not hide the next buffer's positions
        put(g_of(0, L - 40), "skip_into_next_first", k=0, force=True)
        put(g_of(0, L - 40) + 69, "skip_into_next_second_69", k=3, force=True)
        # F1 / F2 / bit cells across scan tiles and into the 64-position look-ahead (tile coordinate = data index of the segment)
        for i, t in enumerate(range(2, 190, 3)):
            dx = (-49, -48, -47, -25, -2, -1, 0, 1)[i % 8]
            put(t * 2048 + dx - HALO, f"tile_{dx:+d}_phase{(0, 6, 7, 25)[(i // 8) % 4]}", k=(0, 6, 7, 25)[(i // 8) % 4])
        # a chunk with more than 32 front-test survivors: a train of F1-like pulses, every 4 positions, then a reply
        g0 = g_of(5, 9000)
        for p in range(g0, g0 + 440, 4):
            m[p - 1], m[p], m[p + 1], m[p + 2] = BG, 6000, 6000, BG
        busy[g0 - 1: g0 + 520] = True
        put(g0 + 460, "after_survivor_train", k=6, force=True)
        # a zero halo: buffer 3 of the magnitude capture is handed over without its predecessor's samples
        restart.append(3)
        put(g_of(3, 200), "in_zero_halo", k=1)
        put(g_of(3, 330), "after_zero_halo", k=2)
        # DF17 frames next to replies
        from make_verdicts import df17, render
        frames = []
        for i in range(4):
            g = g_of(i + 1, 30000 + 10 * i)
            frames.append((5 * g + 4 + i, df17(0x4840D6, rng), 6000))
            put(g - 120, f"before_df17_{i}", k=i)
            put(g + 1400, f"after_df17_{i}", k=i + 1)
        m[:n] = np.maximum(m[:n], render(n, frames, floor=0))
        for b in range(nb):                                     # the rest: sparse replies at every phase
            for i in range(12):
                put(g_of(b, 2000 + 5000 * i + 37 * b), f"filler_{b}_{i}", k=i + b)
    elif name in ("c100", "c300", "c400", "c1000"):
        # tiles over many buffers: every third buffer is loud (a high noise floor from its own sums), the others hold replies.
        # (Buffers shorter than the halo give the next one a zero halo, sdr_ifile.c:207-212, and their positions all lie in that
        # halo: at 100 and 300 samples the reference finds nothing, and the library must not either.)
        for b in range(nb):
            if b % 3 == 1:
                seg = slice(b * L, (b + 1) * L)
                m[seg] = rng.integers(0, 40000, L).astype(np.uint16)
                busy[seg] = True
        for b in range(nb):
            if b % 3 == 1:
                continue
            # (at 400 samples a tile holds five buffers: replies beyond the halo, in the buffers the tile reaches past the loud one)
            for j in (range(1 + (b * 7) % 29, L, 150) if L != 400 else (330 + b % 7,)):
                put(g_of(b, j), f"j{j}_buf{b}", k=j + b)
            put(g_of(b, L - 1), f"last_buf{b}", k=b)
    elif name == "c8191":
        # buffer starts that are not multiples of 32 positions: replies at the first and the last positions of buffers
        for b in range(1, nb):
            j = (1, 2, 3, 4, 5, 1, 2, 3, 4, 5)[b]
            put(g_of(b, j), f"first_{j}_buf{b}", k=j + b)
            for i in range(1, 20):
                put(g_of(b, 400 * i + b), f"mid_{i}_buf{b}", k=i + b)
            if b < 4:                                   # (later buffers keep their successor's first positions free)
                j = (L - 1, L - 3, L - 31, L - 70)[b % 4]
                put(g_of(b, j), f"last_{j}_buf{b}", k=j + b)
    elif name == "c20000":
        for b in range(nb):
            for i in range(40):
                put(g_of(b, 5 + 487 * i + b), f"r{i}_buf{b}", k=i)
    elif name == "cbig":
        # clock phases where float32 rounds j + fraction^2: past 2^17 and past 2^20
        for base in (1000, (1 << 17) - 100, 1 << 17, (1 << 18) + 5, (1 << 20) - 200, 1 << 20, (1 << 20) + 150):
            for i in range(4):
                put(base + 90 * i - HALO, f"j{base + 90 * i}", k=(7 * i + base) % 26)
    assert placed
    return L, m[:n], placed, restart


# ---- the reference's verdicts -------------------------------------------------------------------------------------------------
def to_uc8(mag, lut):
    from make_verdicts import to_uc8 as f
    return f(mag, lut)


def buffers(mag: np.ndarray, L: int, restart=()):
    """(buffer, mag_buf data) with the halo as sdr_ifile.c:207-212 carries it: zero after a buffer shorter than the halo."""
    for b in range(mag.size // L):
        halo = mag[b * L - HALO: b * L] if b > 0 and b not in restart and L >= HALO else np.zeros(HALO, np.uint16)
        yield b, np.ascontiguousarray(np.concatenate([halo, mag[b * L: (b + 1) * L]]))


def run_ref(mk_data, L: int, nb: int, levels_of, model_noise=True):
    """The reference on a capture: for each buffer Mode S (demodulate2400) then Mode A/C (demodulate2400AC), readsb.c:871-874.
    mk_data(b) -> the buffer's mag_buf data (halo + samples); levels_of(b, data) -> (mean_level, mean_power).
    Returns (Mode S frames, their signal levels, replies, per-buffer reply count), checked against the oracle and `scan`."""
    from oraclelib import Oracle, Reference
    ref, orc = Reference(), Oracle()
    frames, flv, acs, counts = [], [], [], []
    for b in range(nb):
        data = mk_data(b)
        ml, mp = levels_of(b, data)
        f, lv, _ = ref.demodulate(data, L, b * L * 5, ml, mp)
        frames.append(f); flv.append(lv)
        import ctypes as C
        out = np.zeros(4096, MODEAC_DTYPE)
        cnt = C.c_uint(0)
        assert ref.L.ref_demodulate2400AC(data.ctypes.data, L, b * L * 5, C.c_double(ml), C.c_double(mp), out.ctypes.data, 4096, C.byref(cnt)) == 0
        a = out[: cnt.value].copy()
        o = orc.demodulate_ac_levels(data, L, b * L * 5, ml, mp)
        assert np.array_equal(a["timestamp"], o["timestamp"]) and np.array_equal(a["modeac"], o["modeac"]), b
        want = scan(data, L, noise_floor(ml, mp))
        assert [(r[0], b * L * 5 + (r[1] + 87 * 14) // 5, r[2]) for r in want] == \
            [(int(x["f1_sample"]), int(x["timestamp"]), int(x["modeac"])) for x in o], (b, want, o)
        a["f1_sample"] = o["f1_sample"]                    # the harness does not see it; the oracle does, at the same timestamps
        a["buffer_idx"] = b
        acs.append(a); counts.append(len(a))
    assert ref.modeac_count() == sum(counts)
    return np.concatenate(frames), np.concatenate(flv), np.concatenate(acs), np.array(counts, np.uint32)


def mag_runner(mag, L, restart=(), levels=None):
    nb = mag.size // L
    datas = dict(buffers(mag, L, restart))
    if levels is None:
        lv = lambda b, d: sums_levels(d[HALO: HALO + L])                                # noqa: E731
    else:
        lv = lambda b, d: (float(levels[b, 0]), float(levels[b, 1]))                     # noqa: E731
    return run_ref(lambda b: datas[b], L, nb, lv)


def uc8_runner(iq, L, restart=()):
    """The reference's uc8 converter, halo carried (a zero one for the `restart` buffers)."""
    from oraclelib import Reference
    conv = Reference()
    nb = iq.size // 2 // L
    datas, lvs, halo = {}, {}, np.zeros(HALO, np.uint16)
    for b in range(nb):
        mag, ml, mp = conv.convert(np.ascontiguousarray(iq[2 * b * L: 2 * (b + 1) * L]))
        if b in restart:
            halo = np.zeros(HALO, np.uint16)
        datas[b] = np.ascontiguousarray(np.concatenate([halo, mag]))
        lvs[b] = (ml, mp)
        halo = datas[b][L: L + HALO].copy() if L >= HALO else np.zeros(HALO, np.uint16)
    return run_ref(lambda b: datas[b], L, nb, lambda b, d: lvs[b])


def sc16_runner(iq16, L, q11):
    from oraclelib import Reference
    conv = Reference()
    nb = iq16.size // 2 // L
    datas, lvs, halo = {}, {}, np.zeros(HALO, np.uint16)
    for b in range(nb):
        mag, ml, mp = conv.convert_sc16(np.ascontiguousarray(iq16[2 * b * L: 2 * (b + 1) * L]), q11)
        datas[b] = np.ascontiguousarray(np.concatenate([halo, mag]))
        lvs[b] = (ml, mp)
        halo = datas[b][L: L + HALO].copy()
    return run_ref(lambda b: datas[b], L, nb, lambda b, d: lvs[b])


def check_expectations(cases, acs, L):
    """Every case meets the class it was drawn for: accepted at its position with its code, or no reply in its buffer."""
    for c in cases:
        got = acs[acs["buffer_idx"] == c["buffer"]]
        cls = c["expect"]
        if cls.startswith("accepted"):
            code = int(cls.split(":")[1], 16) if ":" in cls else None
            hit = got[got["f1_sample"] == c["j"]]
            assert len(hit) == 1 and (code is None or int(hit["modeac"][0]) == code), (c, got)
        elif cls.startswith("rejected"):
            assert len(got) == 0, (c, got)


def generate() -> dict:
    from oraclelib import Reference
    rng = np.random.default_rng(2027)
    ref = Reference()
    lut = ref.lut()
    out, meta = {}, {"buf": {}, "restart": {}, "cases": {}, "kinds": {}}

    def record(cap, kind, res):
        f, flv, a, cnt = res
        out[f"frames_{cap}_{kind}"], out[f"flevels_{cap}_{kind}"], out[f"ac_{cap}_{kind}"], out[f"acn_{cap}_{kind}"] = f, flv, a, cnt
        meta["kinds"].setdefault(cap, []).append(kind)

    # a
    cases, mag, lv = capture_a()
    for c in cases:
        r = decide(dict(buffers(mag, LA))[c["buffer"]], c["j"], c["noise"])
        c["cond"] = [k for k in CONDITIONS if not r["cond"][k]]
        c["phase"] = r["clock"] - 25 * c["j"]
    out["mag_a"], out["lv_a"], out["uc8_a"] = mag, lv, to_uc8(mag, lut)
    meta["buf"]["a"], meta["cases"]["a"] = LA, cases
    res = mag_runner(mag, LA, levels=lv)
    check_expectations(cases, res[2], LA)
    record("a", "given", res)
    record("a", "uc8", uc8_runner(out["uc8_a"], LA))
    # b
    cases, mag, lv = capture_b()
    for c in cases:
        r = decide(dict(buffers(mag, LA))[c["buffer"]], c["j"], c["noise"])
        c["cond"] = [k for k in CONDITIONS if not r["cond"][k]]
    out["mag_b"], out["lv_b"], out["uc8_b"] = mag, lv, to_uc8(mag, lut)
    meta["buf"]["b"], meta["cases"]["b"] = LA, cases
    res = mag_runner(mag, LA, levels=lv)
    check_expectations(cases, res[2], LA)
    record("b", "given", res)
    record("b", "mag", mag_runner(mag, LA))
    record("b", "uc8", uc8_runner(out["uc8_b"], LA))
    for q11 in (False, True):
        kind = "sc16q11" if q11 else "sc16"
        iq = np.concatenate([sc16_of(mag, q11), negative_variance_buffer(ref, q11, LA)])
        out[f"{kind}_b"] = iq
        record("b", kind, sc16_runner(iq, LA, q11))
    # c
    for cap in C_BUFS:
        L, mag, placed, restart = capture_c(cap, rng)
        out[f"mag_{cap}"], out[f"uc8_{cap}"] = mag, to_uc8(mag, lut)
        meta["buf"][cap], meta["restart"][cap] = L, restart
        meta["cases"][cap] = [dict(name=t, g=int(g), buffer=int((g + HALO) // L), j=int(g + HALO - (g + HALO) // L * L)) for g, t in placed]
        record(cap, "mag", mag_runner(mag, L, restart))
        record(cap, "uc8", uc8_runner(out[f"uc8_{cap}"], L, restart))
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    return out


def main():
    out = generate()
    OUT.parent.mkdir(exist_ok=True)
    np.savez_compressed(OUT, **out)
    meta = json.loads(bytes(out["meta"]).decode())
    print(OUT.name, OUT.stat().st_size, "bytes;", {k: len(v) for k, v in meta["cases"].items()}, "cases;",
          {k[3:]: len(v) for k, v in out.items() if k.startswith("ac_")}, "replies")


if __name__ == "__main__":
    main()
