"""Generates tests/golden/verdicts/verdicts.npz: crafted captures, one decision of demodulate2400() per case, and what the
REFERENCE ITSELF (oracle/_ref/libreadsb_ref.so, built from the reference tree by oracle/Makefile) returned for them under every
option set.  Only runs where the reference library can be built; the committed fixture is the authority elsewhere.

    python tests/golden/make_verdicts.py

The captures are drawn by a small magnitude-domain encoder (render): a Mode S pulse is 6 ticks of the 12 MHz clock (0.5 us), a
sample covers 5 ticks, and a sample's magnitude is the floor plus the pulse amplitude times the share of its 5 ticks a pulse
covers.  A frame starting at tick T = 5 pa + phase (phase 4..8) is the one demod_2400.c's position pa and try_phase look for:
preamble pulses at ticks 0/12/42/54, bit k at tick 96 + 12 k (first half for a one, second half for a zero).

Captures (each exists as magnitudes, fed to demodulate2400 buffer by buffer with the halo carried, and as uc8 I/Q whose table
magnitudes are the nearest to those, fed through the reference's converter):
  a  verdicts and exact ties: 1024-sample buffers, one case per buffer (families A and D);
  b  filter generations: 1024-sample buffers, a 30 ms filter TTL (family B);
  c  placement: 65536-sample buffers, frames at the skip, the buffer edges and the kernels' chunk / tile / sub-range
     boundaries (family C).
Family D (exact ties of the pre-check, the correlator thresholds and the bit slicers; magnitudes 0 and 65535; signal levels
around -3 dBFS) only means something in magnitudes: its uc8 buffers are merely more traffic.
"""
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from readsb_b200.abi import BUFRES_DTYPE  # noqa: E402

OUT = HERE / "verdicts" / "verdicts.npz"
HALO = 326
LA, LC = 1024, 65536
FLOOR, AMP = 300, 6000
KNOWN = 0x4840D6
# (preamble threshold, nfix_crc, fix_df): readsb's default, the repairs off one by one and together, and the threshold's clamp range
OPTIONS = [(58, 1, 1), (58, 0, 1), (58, 1, 0), (58, 0, 0), (40, 1, 1), (75, 1, 1), (400, 1, 1)]
TTL = {"a": 60000, "b": 30, "c": 60000}
LONG_OK = (1 << 16) | (1 << 17) | (1 << 18) | (1 << 20) | (1 << 21) | (1 << 1) | (1 << 25) | (1 << 19)   # with the DF17 repair
SHORT_OK = (1 << 0) | (1 << 4) | (1 << 5) | (1 << 11)
AP_TYPES = (0, 4, 5, 16, 20, 21)


# ---- encoder ---------------------------------------------------------------------------------------------------------------
def msg_bits(msg: bytes) -> list:
    return [(msg[i >> 3] >> (7 - (i & 7))) & 1 for i in range(8 * len(msg))]


def pulses(msg: bytes) -> list:
    return [0, 12, 42, 54] + [96 + 12 * k + (0 if b else 6) for k, b in enumerate(msg_bits(msg))]


def render(n: int, frames, floor=FLOOR) -> np.ndarray:
    """frames: (start tick, message bytes, amplitude above the floor[, floor of the frame's own span]).  Pulses add."""
    cov = np.zeros(n, np.int64)
    base = np.full(n, floor, np.int64)
    for f in frames:
        t, msg, amp = f[:3]
        if len(f) > 3:
            s0, s1 = t // 5 - 20, (t + 96 + 12 * 8 * len(msg)) // 5 + 40
            base[max(s0, 0): min(s1, n)] = f[3]
        for p in pulses(msg):
            t0, t1 = t + p, t + p + 6
            for s in range(t0 // 5, (t1 - 1) // 5 + 1):
                if 0 <= s < n:
                    cov[s] += (min(t1, 5 * s + 5) - max(t0, 5 * s)) * amp
    return np.clip(base + (cov + 2) // 5, 0, 65535).astype(np.uint16)


_ORACLE = []


def crc24(msg: bytes) -> int:
    from oraclelib import Oracle
    if not _ORACLE:
        _ORACLE.append(Oracle())                 # the oracle's CRC tables are set up with its first context
    return Oracle.crc24(msg)


def with_parity(head: bytes, overlay: int = 0) -> bytes:
    """head + the 24 parity bits that make the frame's syndrome `overlay` (0: clean DF11 IID 0 / DF17 / DF18; the address of an
    address/parity reply; the IID of a DF11)."""
    rem = crc24(head + b"\0\0\0")
    return head + int(rem ^ overlay).to_bytes(3, "big")


def flip(msg: bytes, *bits) -> bytes:
    m = bytearray(msg)
    for b in bits:
        m[b >> 3] ^= 1 << (7 - (b & 7))
    return bytes(m)


def df17(addr: int, rng, df=17, ca=5) -> bytes:
    return with_parity(bytes([(df << 3) | ca]) + addr.to_bytes(3, "big") + rng.integers(0, 256, 7, dtype=np.uint8).tobytes())


def df11(addr: int, iid=0, ca=5) -> bytes:
    return with_parity(bytes([(11 << 3) | ca]) + addr.to_bytes(3, "big"), iid)


def ap(df: int, addr: int, rng, overlay=0) -> bytes:
    n = 14 if df >= 16 else 7
    return with_parity(bytes([(df << 3) | int(rng.integers(0, 8))]) + rng.integers(0, 256, n - 4, dtype=np.uint8).tobytes(), addr ^ overlay)


# ---- the reference's decision, predicted from the frame alone (default options) ------------------------------------------
def diagnose1(syn: int, bits: int) -> int:
    from oraclelib import Oracle
    crc24(b"")
    return Oracle.diagnose1(syn, bits)


def expect(msg: bytes, known: set) -> str:
    """Outcome class of a frame sliced without errors, under readsb's defaults (nfix_crc 1, fixDF 1): accepted[c] (accepted with c
    corrected bits), rejected_unknown (score or decode -1), rejected_bad (-2)."""
    df = msg[0] >> 3
    aa = int.from_bytes(msg[1:4], "big")
    if df >= 16 or (LONG_OK >> df) & 1:
        if not (LONG_OK >> df) & 1:
            return "rejected_bad"
        if df in (1, 25, 21, 19, 16) and crc24(bytes([(msg[0] & 7) | (17 << 3)]) + msg[1:]) == 0:
            return "accepted[1]"                                             # fixDF17msgtype
        if df in (1, 19, 25):
            return "rejected_bad"
        syn = crc24(msg)
        if df in (16, 20, 21):
            return "accepted[0]" if syn in known else "rejected_unknown"
        if syn == 0:
            return "accepted[0]"
        b = diagnose1(syn, 112)
        if b < 0:
            return "rejected_bad"
        if 8 <= b <= 31 and (aa ^ (1 << (31 - b))) not in known:
            return "rejected_unknown"                                        # positive score, decodeModesMessage says -1
        return "accepted[1]"
    if not (SHORT_OK >> df) & 1:
        return "rejected_bad"
    if msg[:7] == bytes(7):
        return "rejected_bad"
    syn = crc24(msg[:7])
    if df != 11:
        return "accepted[0]" if syn in known else "rejected_unknown"
    if syn & 0xFFFF80:
        b = diagnose1(syn, 56)
        if b < 0:
            return "rejected_bad"
        a2 = aa ^ (1 << (31 - b)) if 8 <= b <= 31 else aa
        return "accepted[1]" if a2 in known else "rejected_unknown"
    if syn == 0:
        return "accepted[0]"
    return "accepted[0]" if aa in known else "rejected_unknown"


def adds(msg: bytes, cls: str) -> int | None:
    """The address a frame of class `cls` adds to the filter (mode_s.c:766-779), or None."""
    df = msg[0] >> 3
    if cls != "accepted[0]":
        return None
    if df == 17 or (df == 11 and crc24(msg[:7]) == 0):
        return int.from_bytes(msg[1:4], "big")
    return None


# ---- capture a: one case per buffer ---------------------------------------------------------------------------------------
class Table:
    def __init__(self, capture, L):
        self.capture, self.L = capture, L
        self.cases, self.frames, self.restart = [], [], []

    def add(self, name, family, cls, buf, msgs, extra=None):
        self.cases.append(dict(name=name, family=family, expect=cls, buffer=buf, msg=msgs[0].hex() if msgs else "", **(extra or {})))


def capture_a(rng):
    T = Table("a", LA)
    known = {KNOWN}
    fresh = iter(range(0x700001, 0x7FFFFF, 0x111))
    cases = []                                                  # (name, family, msg, expected class or None)

    def frame_case(name, msg, family="A", cls=None):
        cases.append((name, family, msg, cls))

    frame_case("teach_df17_known", df17(KNOWN, rng))
    for d in (17, 18):
        for kn in (True, False):
            tag = "known" if kn else "unknown"
            frame_case(f"df{d}_{tag}_clean", df17(KNOWN if kn else next(fresh), rng, df=d, ca=int(rng.integers(0, 8))))
            for b in range(112):
                frame_case(f"df{d}_{tag}_flip{b}", flip(df17(KNOWN if kn else next(fresh), rng, df=d, ca=int(rng.integers(0, 8))), b))
    for iid in (0, 3):
        for kn in (True, False):
            tag = "known" if kn else "unknown"
            frame_case(f"df11_iid{iid}_{tag}_clean", df11(KNOWN if kn else next(fresh), iid))
            for b in range(56):
                frame_case(f"df11_iid{iid}_{tag}_flip{b}", flip(df11(KNOWN if kn else next(fresh), iid), b))
    # a DF17 / DF18 / DF11 whose syndrome is the single-bit syndrome of a DF bit (a clean frame of the neighbouring DF with that
    # bit flipped): modesChecksumDiagnose never repairs bits 0..4 (crc.c), so these are -2 however the filter stands
    for d in (17, 18, 11):
        for b in range(5):
            src = d ^ (1 << (4 - b))
            head = bytes([(src << 3) | 5]) + KNOWN.to_bytes(3, "big")
            clean = with_parity(head + (rng.integers(0, 256, 7, dtype=np.uint8).tobytes() if d != 11 else b""))
            frame_case(f"df{d}_syndrome_of_df_bit{b}", flip(clean, b))
    for b0, b1 in ((10, 50), (40, 41), (5, 100), (0, 1), (30, 111), (60, 90)):
        frame_case(f"df17_known_flip{b0}+{b1}", flip(df17(KNOWN, rng), b0, b1))
    for b0, b1 in ((10, 20), (30, 31), (5, 40), (12, 52)):
        frame_case(f"df11_known_flip{b0}+{b1}", flip(df11(KNOWN), b0, b1))
    for d in range(32):
        if d in AP_TYPES:
            frame_case(f"df{d}_known", ap(d, KNOWN, rng))
            frame_case(f"df{d}_unknown", ap(d, next(fresh), rng))
        elif d in (11, 17, 18):
            frame_case(f"df{d}_any", df11(next(fresh)) if d == 11 else df17(next(fresh), rng, df=d))
        else:
            n = 14 if d >= 16 else 7
            frame_case(f"df{d}_any", bytes([(d << 3) | int(rng.integers(0, 8))]) + rng.integers(0, 256, n - 1, dtype=np.uint8).tobytes())
    for d in (20, 21):
        for bds in (0x10, 0x40):
            frame_case(f"df{d}_known_bds{bds:02x}", ap(d, KNOWN, rng, overlay=bds << 16))
    frame_case("df0_all_zero", bytes(7))
    frame_case("df17_all_zero_head", with_parity(bytes([17 << 3]) + bytes(10)))

    # family A: frames drawn at a rotating phase, 60 samples into their buffer; their expected classes follow the filter they meet
    buf = 0
    for name, family, msg, cls in cases:
        phase = 4 + buf % 5
        pa = buf * LA + 60
        if cls is None:
            cls = expect(msg, known)
            a = adds(msg, cls)
            if a is not None:
                known.add(a)
        T.frames.append((5 * pa + phase, msg, AMP))
        T.add(name, family, cls, buf, [msg], dict(pa=pa, phase=phase))
        buf += 1
    nbuf_a = buf
    mag = np.zeros(0, np.uint16)
    extra = []                     # (buffer, magnitude block) for the family D buffers, edited after drawing
    # family D
    for phase in range(4, 9):
        for which, (i, j) in enumerate(((1, 7), (12, 14), (12, 15))):
            for d_ in (0, 1):
                extra.append(("tie", f"precheck_phase{phase}_pa{i}_pa{j}_{'equal' if d_ == 0 else 'plus1'}", phase, (i, j, d_)))
    for thr in sorted({o[0] for o in OPTIONS}):
        for corr, phase in ((0, 4), (1, 6), (2, 8)):
            for d_ in (0, -1):
                extra.append(("thr", f"corr{corr}_thr{thr}_{'at' if d_ == 0 else 'below'}_ref_level", phase, (thr, corr, d_)))
    for phase in range(4, 9):
        for k in (20, 57, 90):
            extra.append(("zero", f"zero_cell_phase{phase}_bit{k}", phase, (k,)))
    extra.append(("ext", "floor0_amp65535", 4, (0, 65535)))
    extra.append(("ext", "floor0_amp65535_phase7", 7, (0, 65535)))
    extra.append(("ext", "saturated", 6, (65535, 65535)))
    for phase in range(4, 9):
        for floor in (25000, 20000):
            extra.append(("strong", f"level_floor{floor}_phase{phase}", phase, (floor, 65535)))

    n = (nbuf_a + len(extra)) * LA
    mag = render(n, T.frames)
    for e, (kind, name, phase, arg) in enumerate(extra):
        buf = nbuf_a + e
        pa = buf * LA + 60
        seg = slice(buf * LA, (buf + 1) * LA)
        msg = df17(KNOWN, rng, ca=int(rng.integers(0, 8)))
        floor, amp = FLOOR, AMP
        if kind in ("ext", "strong"):
            floor, amp = arg[0], arg[1] - arg[0]
        local = render(LA + 400, [(5 * 60 + phase, msg, amp)], floor=floor)
        mag[seg] = local[:LA]
        info = dict(pa=pa, phase=phase)
        cls = None
        if kind == "tie":
            i, j, d_ = arg
            mag[pa + j] = min(int(mag[pa + i]) - d_, 65535) if int(mag[pa + i]) - d_ >= 0 else 0
        elif kind == "thr":
            thr, corr, d_ = arg
            # the noise samples set ref_level; then one preamble sample moves correlation `corr` onto ref_level (or one below)
            w = mag[pa: pa + 20].astype(np.int64)
            c = correlations(w)[corr]
            noise = int(w[5] + w[8] + w[16] + w[17])
            v = max(0, min(65535, ((c * 32) // thr) - noise - 40))
            mag[pa + 18] = v
            w = mag[pa: pa + 20].astype(np.int64)
            ref = ((noise + v) * thr) >> 5
            # sample that enters this correlation with +1: pa[11] for corr 0, pa[10] for corr 1 and 2
            s = 11 if corr == 0 else 10
            need = ref + d_ - correlations(w)[corr]
            mag[pa + s] = int(np.clip(int(w[s]) + need, 0, 65535))
            w = mag[pa: pa + 20].astype(np.int64)
            info.update(thr=thr, corr=corr, delta=int(correlations(w)[corr] - (((w[5] + w[8] + w[16] + w[17] + w[18]) * thr) >> 5)))
        elif kind == "zero":
            (k,) = arg
            # the cell's samples in the proportions that zero its slicer: 18-15-3, 14-5-9, 16*5+5*4-20*5, 7+11-18, 4+15-20+1
            (s, f), = bit_cells(pa, phase, k)
            c = max(int(mag[s]) // 5, 1)
            for q, vq in enumerate((5, 4, 5) if f == 2 else (5,) * (4 if f == 4 else 3)):
                mag[s + q] = c * vq
            info.update(bit=k)
        elif kind == "strong":
            cls = "accepted[0]"
        T.frames.append((5 * pa + phase, msg, amp))
        T.add(name, "D", cls or "any", buf, [msg], info)
    return T, mag


def correlations(p) -> tuple:
    """The three preamble correlations of demod_2400.c:344-376 at the window p = pa[0..19]."""
    d23, s14, d1011 = p[2] - p[3], p[1] + p[4], p[10] - p[11]
    common = s14 - d23 + p[9] + p[12]
    return int(common - d1011), int(common + d1011), int(s14 + 2 * d23 + d1011 + p[12])


SLICE = {0: ([(0, 0), (2, 2), (4, 4), (7, 1), (9, 3), (12, 0), (14, 2), (16, 4)], 19),
         1: ([(0, 1), (2, 3), (5, 0), (7, 2), (9, 4), (12, 1), (14, 3), (17, 0)], 19),
         2: ([(0, 2), (2, 4), (5, 1), (7, 3), (10, 0), (12, 2), (14, 4), (17, 1)], 19),
         3: ([(0, 3), (3, 0), (5, 2), (7, 4), (10, 1), (12, 3), (15, 0), (17, 2)], 19),
         4: ([(0, 4), (3, 1), (5, 3), (8, 0), (10, 2), (12, 4), (15, 1), (17, 3)], 20)}


def bit_cells(pa: int, try_phase: int, k: int):
    """The sample where slice_byte (demod_2400.c:133-213) reads message bit k of try_phase at pa, and its slicer (0..4)."""
    p, ph = pa + 19 + try_phase // 5, try_phase % 5
    for _ in range(k // 8):
        p += SLICE[ph][1]
        ph = (ph + 1) % 5
    off, f = SLICE[ph][0][k % 8]
    return [(p + off, f)]


def slice_frame(mag: np.ndarray, pa: int, try_phase: int, nbits: int) -> bytes:
    """slice_byte in numpy: the bits the reference would read (encoder self-check)."""
    fns = {0: (18, -15, -3, 0), 1: (14, -5, -9, 0), 2: (16, 5, -20, 0), 3: (7, 11, -18, 0), 4: (4, 15, -20, 1)}
    out = bytearray(nbits // 8)
    for k in range(nbits):
        (s, f), = bit_cells(pa, try_phase, k)
        v = sum(c * int(mag[s + q]) for q, c in enumerate(fns[f]))
        if v > 0:
            out[k >> 3] |= 1 << (7 - (k & 7))
    return bytes(out)


# ---- capture b: filter generations ----------------------------------------------------------------------------------------
def capture_b(rng):
    """30 ms filter TTL: the decode loop's flip (readsb.c:1227-1231) after buffer 0 and then about every 35 buffers.  X is taught
    between flips 1 and 2, then seen (DF11 with a bit error: only the filter vouches for it) after flip 2 (older generation: known)
    and after flip 3 (gone).  Y is taught between flips 1 and 2; after flip 2, 85 new addresses keep it, the 86th resizes the active
    generation and forgets the older one (icao_filter.c:112-130)."""
    T = Table("b", LA)
    X, Y = 0x3C6589, 0xA0B1C2
    plan = {1: [("teach_x", df17(X, rng))], 2: [("teach_y", df17(Y, rng))], 5: [("x_one_flip_before", flip(df11(X), 20))]}
    flips = flip_buffers(60)
    after2, after3 = flips[1] + 1, flips[2] + 1
    plan[after2] = [("x_older_generation", flip(df11(X), 20))]
    plan[after2 + 1] = [("y_older_generation", flip(df11(Y), 30))]
    b = after2 + 2
    newa = iter(range(0x200001, 0x2FFFFF, 0x101))
    for i in range(85):
        plan.setdefault(b + i // 3, []).append((f"new{i + 1}", df17(next(newa), rng)))
    b += 29
    plan[b] = [("y_after_85_new", flip(df11(Y), 31))]
    plan[b + 1] = [("new86", df17(next(newa), rng))]
    plan[b + 2] = [("y_after_86_new", flip(df11(Y), 33))]
    plan[b + 3] = [("x_still_older_generation", flip(df11(X), 40))]
    plan[after3 + 1] = [("x_two_flips_later", flip(df11(X), 21))]
    nbuf = after3 + 3
    expected = {"teach_x": "accepted[0]", "teach_y": "accepted[0]", "x_one_flip_before": "accepted[1]", "x_older_generation": "accepted[1]",
                "y_older_generation": "accepted[1]", "y_after_85_new": "accepted[1]", "new86": "accepted[0]", "y_after_86_new": "rejected_unknown",
                "x_still_older_generation": "rejected_unknown", "x_two_flips_later": "rejected_unknown"}
    for buf in range(nbuf):
        for i, (name, msg) in enumerate(plan.get(buf, [])):
            pa = buf * LA + 30 + 300 * i
            phase = 4 + (buf + i) % 5
            T.frames.append((5 * pa + phase, msg, AMP))
            T.add(name, "B", expected.get(name, "accepted[0]"), buf, [msg], dict(pa=pa, phase=phase, index=i))
    assert (max(len(v) for v in plan.values()) - 1) * 300 + 30 + 300 < LA and b + 3 < flips[2]
    return T, render(nbuf * LA, T.frames), flips


def flip_buffers(n: int) -> list:
    """Buffers after which the reference's filter flips with capture b's TTL (sysTimestamp = sample clock / 12000 + epoch; the first
    flip follows buffer 0).  Only the buffer clock moves synthetic_now in these buffers' positions (frames lie early in them)."""
    out, nxt = [], 0
    for b in range(n * 40):
        now = (b * LA * 5) // 12000
        if now >= nxt:
            out.append(b)
            nxt = now + TTL["b"]
        if len(out) == 4:
            break
    return out


# ---- capture c: placement -------------------------------------------------------------------------------------------------
def capture_c(rng):
    """65536-sample buffers.  Frames at the kernels' boundaries in data positions j of a buffer (the 326 halo positions first):
    scan chunks of 512, tiles of 2048, 8-tile runs of 16384, stage B sub-ranges and quads of 8192, each at -3..+2; frames whose skip
    reaches across an 8192 boundary; each buffer's first positions (which read the halo) and last positions; and pairs whose second
    frame lies skip - 1, skip or skip + 1 positions after an accepted long / short frame or after a rejected one."""
    T = Table("c", LC)
    nbuf = 6
    placed = []                                                   # (global position, name, message, amplitude, class)

    def g_of(b, j):
        return b * LC - HALO + j

    # pairs: 18 reserved regions, three per buffer, halfway between sub-range boundaries
    regions = [(b, j) for b in range(nbuf) for j in (3500, 19884, 36268)]
    r = iter(regions)
    for first in ("long", "short", "rejected"):
        for d in (-1, 0, 1):
            for second in ("long", "short"):
                b, j = next(r)
                if first == "rejected":                          # score 700, decodeModesMessage -1 (AA repaired to an unknown address)
                    m1, skip = flip(df17(0x5D0000 + len(placed), rng), 12), 225
                else:
                    m1 = df17(KNOWN, rng) if first == "long" else df11(KNOWN)
                    skip = len(m1) * 8 * 8 // 4 + 1               # demod_2400.c:468 plus the loop's pa++
                m2 = df17(KNOWN, rng) if second == "long" else df11(KNOWN)
                tag = f"{first}_{d:+d}_{second}"
                placed.append((g_of(b, j), f"pair_first_{tag}", m1, 4 * AMP, "rejected_unknown" if first == "rejected" else "any"))
                placed.append((g_of(b, j) + skip + d, f"pair_second_{tag}", m2, AMP // 2, "any"))
    # buffer edges: odd buffers get frames at their first positions (drawn in the previous buffer's last 326 samples) and their
    # last ones; buffer 3 of the magnitude capture starts with a zero halo (a receiver that dropped samples)
    for b, k in ((1, 0), (3, 1), (5, 2)):
        placed.append((g_of(b, k), f"edge_first_j{k}_buf{b}", df17(KNOWN, rng), AMP, "any"))
        placed.append((g_of(b, LC - 1 - k), f"edge_last_j{LC - 1 - k}_buf{b}", df11(KNOWN), AMP, "accepted[0]"))
    # kernel boundaries, away from the pairs and the edges
    busy = [p[0] for p in placed]
    k, per_kind = 0, {}
    slots = [(b, X) for b in range(nbuf) for X in range(2048, LC - 1024, 2048)]           # tiles, quads and runs first,
    slots += [(b, X) for b in range(nbuf) for X in range(1536, LC - 1024, 1024)]         # then the chunks between them
    for b, X in slots:
        if X % 8192 == 0 and (b + X // 8192) % 3 == 0:
            j = X - 100                                       # accepted just before the boundary: its skip reaches across
            name = f"skip_across_{X}_buf{b}"
        else:
            kind = "run16384" if X % 16384 == 0 else "quad8192" if X % 8192 == 0 else "tile2048" if X % 2048 == 0 else "chunk512"
            off = per_kind.get(kind, 0) % 6 - 3                # each kind of boundary cycles through -3..+2 on its own
            j = X + off
            name = f"{kind}_{X}{off:+d}_buf{b}"
        g = g_of(b, j)
        if g < 0 or any(abs(g - q) < 700 for q in busy):
            continue
        if not name.startswith("skip"):
            per_kind[kind] = per_kind.get(kind, 0) + 1
        placed.append((g, name, df17(KNOWN, rng) if k % 3 else df11(KNOWN), AMP, "accepted[0]"))
        busy.append(g)
        k += 1
    for g, name, msg, amp, cls in sorted(placed, key=lambda p: p[0]):
        phase = 4 + (g % 5)
        T.frames.append((5 * g + phase, msg, amp))
        b = (g + HALO) // LC
        T.add(name, "C", cls, b, [msg], dict(pa=g, phase=phase, j=g - b * LC + HALO))
    T.restart = [3]
    return T, render(nbuf * LC, T.frames)


# ---- uc8 twin of a magnitude capture ------------------------------------------------------------------------------------------
def to_uc8(mag: np.ndarray, lut: np.ndarray) -> np.ndarray:
    """The I/Q pair whose table magnitude (convert.c's uc8 table) is nearest to each magnitude."""
    order = np.argsort(lut, kind="stable")
    vals = lut[order]
    i = np.clip(np.searchsorted(vals, mag), 1, len(vals) - 1)
    pick = np.where(np.abs(vals[i - 1].astype(np.int64) - mag) <= np.abs(vals[i].astype(np.int64) - mag), i - 1, i)
    idx = order[pick]
    iq = np.empty(2 * mag.size, np.uint8)
    iq[0::2], iq[1::2] = idx >> 8, idx & 0xFF
    return iq


# ---- the reference's verdicts -------------------------------------------------------------------------------------------------
def feed_mag(ref, mag: np.ndarray, L: int, restart=(), cases=None, score_out=None):
    """demodulate2400 buffer by buffer with the halo carried (a zero halo for buffer 0 and the `restart` buffers); optionally the
    reference's scoreModesMessage of each case's message, taken with the filter as it stands before that case's buffer."""
    frames, levels, bufres = [], [], []
    by_buf = {}
    for i, c in enumerate(cases or []):
        by_buf.setdefault(c["buffer"], []).append(i)
    for b in range(mag.size // L):
        halo = mag[b * L - HALO: b * L] if b > 0 and b not in restart else np.zeros(HALO, np.uint16)
        data = np.ascontiguousarray(np.concatenate([halo, mag[b * L: (b + 1) * L]]))
        for i in by_buf.get(b, []):
            msg = bytes.fromhex(cases[i]["msg"])
            score_out[i] = ref.score(msg, 112 if (LONG_OK >> (msg[0] >> 3)) & 1 else 56)
        f, lv, r = ref.demodulate(data, L, b * L * 5)
        frames.append(f); levels.append(lv)
        bufres.append(np.frombuffer(bytearray(r), dtype=BUFRES_DTYPE).copy())
    return np.concatenate(frames), np.concatenate(levels), np.concatenate(bufres)


def generate() -> dict:
    """Everything the fixture holds, made in memory (deterministic for a given reference build)."""
    from oraclelib import Reference
    rng = np.random.default_rng(2026)
    lut = Reference().lut()
    ta, mag_a = capture_a(rng)
    tb, mag_b, _ = capture_b(rng)
    tc, mag_c = capture_c(rng)
    out = {"mag_a": mag_a, "mag_b": mag_b, "mag_c": mag_c}
    meta = {"buf": {"a": LA, "b": LA, "c": LC}, "ttl": TTL, "options": OPTIONS, "restart": {"c": tc.restart},
            "cases": {t.capture: t.cases for t in (ta, tb, tc)}, "stats": {}}
    for t, mag in ((ta, mag_a), (tb, mag_b), (tc, mag_c)):
        cap = t.capture
        out[f"uc8_{cap}"] = to_uc8(mag, lut)
        for o, (thr, nfix, fixdf) in enumerate(OPTIONS):
            kw = dict(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=TTL[cap])
            ref = Reference(**kw)
            score = np.zeros(len(t.cases), np.int32)
            f, lv, br = feed_mag(ref, mag, t.L, t.restart, t.cases, score)
            out[f"frames_{cap}_mag_{o}"], out[f"levels_{cap}_mag_{o}"], out[f"bufres_{cap}_mag_{o}"] = f, lv, br
            out[f"score_{cap}_{o}"] = score
            meta["stats"][f"{cap}_mag_{o}"] = stats_of(ref)
            ref = Reference(**kw)
            f, lv, br, _, _ = ref.run_stream(out[f"uc8_{cap}"], t.L, cap=8192)
            out[f"frames_{cap}_uc8_{o}"], out[f"levels_{cap}_uc8_{o}"], out[f"bufres_{cap}_uc8_{o}"] = f, lv, br
            meta["stats"][f"{cap}_uc8_{o}"] = stats_of(ref)
    out["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    return out


def stats_of(ref) -> dict:
    s, d = ref.stats()
    s.pop("sum_signal_power"); s.pop("reserved_", None)
    s["peak_signal_power"] = d["peak_signal_power"]
    return s


def main():
    out = generate()
    OUT.parent.mkdir(exist_ok=True)
    np.savez_compressed(OUT, **out)
    meta = json.loads(bytes(out["meta"]).decode())
    print(OUT.name, OUT.stat().st_size, "bytes;", {k: len(v) for k, v in meta["cases"].items()}, "cases;",
          {k: len(v) for k, v in out.items() if k.startswith("frames_") and k.endswith("_0")}, "frames under the defaults")


if __name__ == "__main__":
    main()
