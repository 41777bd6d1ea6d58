"""-m "not gpu": the crafted verdict captures of tests/golden/verdicts/verdicts.npz (tests/golden/make_verdicts.py), one decision of
demodulate2400() per case, against what the reference itself returned for them.

- The oracle reproduces the fixture: frames, signal levels, per-buffer counters and receiver statistics, for every capture, input
  kind (magnitudes / uc8 I/Q) and option set.
- Where the reference can be built, the fixture made again in memory equals the committed one.
- The fixture reaches what it is for: every case meets its expected outcome class in the reference's counters, and across the cases
  every score of scoreModesMessage, every repairable bit position, every DF, the -3 dBFS counter, and the exact ties the kernels'
  comparisons turn on all occur.  Regenerating it with fewer or neutralised cases fails here.

The GPU side (tests/test_gpu_verdicts.py) compares the CUDA library with the same fixture."""
import importlib.util
import json
from collections import defaultdict
from pathlib import Path

import numpy as np
import pytest

from oraclelib import Oracle, have_ref
from paritylib import STATS_INT_FIELDS, diff_bufres, diff_frames, diff_stats
from readsb_b200.abi import BUFRES_DTYPE

FIXTURE = Path(__file__).resolve().parent / "golden" / "verdicts" / "verdicts.npz"
HALO = 326
# what the reference harness reports: the frame fields it defines (signal power as a level) and the counters of one call
FRAME_FIELDS = ("timestamp", "j", "crc", "addr", "score", "buffer_seq", "signal_len", "phase", "msgtype", "msgbits", "correctedbits",
                "fix_bit", "msg")
BUFRES_FIELDS = ("sample_timestamp", "length", "n_frames", "buffer_seq", "icao_flipped", "demod_preambles", "demod_rejected_bad",
                 "demod_rejected_unknown_icao", "demod_accepted", "demod_preamblePhase", "demod_bestPhase")
STATS_FIELDS = tuple(f for f in STATS_INT_FIELDS if f != "sum_signal_power")      # the reference keeps that one as fp64 only
CAPTURES = ("a", "b", "c")
KINDS = ("mag", "uc8")


class Fixture:
    def __init__(self):
        self.z = np.load(FIXTURE)
        self.meta = json.loads(bytes(self.z["meta"]).decode())
        self.options = [tuple(o) for o in self.meta["options"]]

    def buf(self, cap):
        return self.meta["buf"][cap]

    def capture(self, cap, kind):
        return np.ascontiguousarray(self.z[f"{kind}_{cap}"])

    def restart(self, cap, kind):
        """Buffers of the magnitude capture that start with a zero halo (the uc8 capture's halo always continues)."""
        return set(self.meta["restart"].get(cap, [])) if kind == "mag" else set()

    def want(self, cap, kind, o):
        z = self.z
        return z[f"frames_{cap}_{kind}_{o}"], z[f"levels_{cap}_{kind}_{o}"], z[f"bufres_{cap}_{kind}_{o}"], self.meta["stats"][f"{cap}_{kind}_{o}"]

    def kwargs(self, cap, o):
        thr, nfix, fixdf = self.options[o]
        return dict(preamble_threshold=thr, nfix_crc=nfix, fix_df=fixdf, icao_ttl_ms=self.meta["ttl"][cap])

    def cases(self, cap):
        return self.meta["cases"][cap]


_FIX = []


def fixture() -> Fixture:
    if not _FIX:
        _FIX.append(Fixture())
    return _FIX[0]


def mag_buffers(mag: np.ndarray, L: int, restart=()):
    """(data with its halo, length, sample timestamp, exact magnitude sums) per buffer, as a frontend hands them over."""
    for b in range(mag.size // L):
        halo = mag[b * L - HALO: b * L] if b > 0 and b not in restart else np.zeros(HALO, np.uint16)
        new = mag[b * L: (b + 1) * L]
        yield np.ascontiguousarray(np.concatenate([halo, new])), L, b * L * 5, int(new.astype(np.uint64).sum()), int((new.astype(np.uint64) ** 2).sum())


def compare(frames, bufres, stats, want) -> list:
    """Differences between a result (frames with sigpow_sum, buffer results, receiver statistics) and the reference's."""
    wf, wl, wb, ws = want
    problems = diff_frames(frames, wf, fields=FRAME_FIELDS)
    if not problems and not np.array_equal(frames["sigpow_sum"] / 65535.0 / 65535.0 / frames["signal_len"], wl):
        problems.append("signal levels differ")       # demod_2400.c:447-448 in fp64
    problems += diff_bufres(bufres, wb, fields=BUFRES_FIELDS)
    if stats is not None:
        problems += diff_stats(stats, ws, fields=STATS_FIELDS)
    return problems


def oracle_run(cap, kind, o):
    F = fixture()
    orc = Oracle(**F.kwargs(cap, o))
    L = F.buf(cap)
    if kind == "uc8":
        f, b = orc.run_stream(F.capture(cap, kind), L, cap=8192)
    else:
        fs, bs = [], []
        for data, n, ts, sl, sp in mag_buffers(F.capture(cap, kind), L, F.restart(cap, kind)):
            f, r = orc.demodulate(data, n, ts, sl, sp)
            fs.append(f); bs.append(np.frombuffer(bytearray(r), dtype=BUFRES_DTYPE).copy())
        f, b = np.concatenate(fs), np.concatenate(bs)
    return f, b, orc.stats()


@pytest.mark.parametrize("o", range(7))
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cap", CAPTURES)
def test_oracle_equals_the_reference_verdicts(cap, kind, o):
    f, b, st = oracle_run(cap, kind, o)
    problems = compare(f, b, st, fixture().want(cap, kind, o))
    assert not problems, "\n".join(problems)


needs_ref = pytest.mark.skipif(not have_ref(), reason="reference tree not available to build oracle/_ref")


def _generator():
    path = FIXTURE.parent.parent / "make_verdicts.py"
    spec = importlib.util.spec_from_file_location("make_verdicts", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@needs_ref
def test_committed_fixture_is_what_the_generator_makes():
    made = _generator().generate()
    z = fixture().z
    assert sorted(made) == sorted(z.files)
    for k in z.files:
        assert made[k].dtype == z[k].dtype and np.array_equal(made[k], z[k]), k


# ---- what the fixture reaches ------------------------------------------------------------------------------------------------
def agrees(cls: str, r, n: int = 1) -> bool:
    """Does one buffer's counters show `n` frames of outcome class `cls`?  Rejections allow other rejected candidates in the same
    buffer (a frame rejected at one phase or position is often looked at again one position later)."""
    if cls.startswith("accepted["):
        return r["n_frames"] == n and r["demod_accepted"][int(cls[9])] == n and r["demod_accepted"].sum() == n
    if cls == "rejected_unknown":
        return r["n_frames"] == 0 and r["demod_rejected_unknown_icao"] > 0
    if cls == "rejected_bad":
        return r["n_frames"] == 0 and r["demod_rejected_bad"] > 0
    if cls == "not_detected":
        return r["demod_preambles"] == 0
    assert cls == "any", cls
    return True


@pytest.mark.parametrize("cap", ["a", "b"])
def test_every_case_meets_its_expected_class(cap):
    """Families A and B, defaults: each buffer's counters are its cases' verdict (accepted with 0 / 1 corrected bits, rejected as
    unknown, rejected as bad)."""
    F = fixture()
    br = F.want(cap, "mag", 0)[2]
    by_buf = defaultdict(list)
    for c in F.cases(cap):
        by_buf[c["buffer"]].append(c)
    checked = 0
    for b, cs in by_buf.items():
        (cls,) = {c["expect"] for c in cs}
        assert agrees(cls, br[b], len(cs)), (b, [c["name"] for c in cs], cls, br[b])
        checked += cls != "any"
    assert checked >= (700 if cap == "a" else 35)


def test_family_b_reaches_the_filter_generations():
    F = fixture()
    cases = {c["name"]: c for c in F.cases("b")}
    br = F.want("b", "mag", 0)[2]
    flips = np.nonzero(br["icao_flipped"])[0]
    b = lambda n: cases[n]["buffer"]                                              # noqa: E731
    # taught between the first two flips, seen after the second (older generation) and after the third (gone)
    assert flips[0] < b("teach_x") < flips[1] < b("x_older_generation") < b("y_after_86_new") < flips[2] < b("x_two_flips_later")
    assert [c for c in F.cases("b") if c["name"].startswith("new")][-1]["name"] == "new86"
    assert b("new85") < b("y_after_85_new") < b("new86") < b("y_after_86_new")
    assert cases["y_after_85_new"]["expect"] == "accepted[1]" and cases["y_after_86_new"]["expect"] == "rejected_unknown"


def test_scores_repairs_and_types_are_all_reached():
    F = fixture()
    scores = set()
    for cap in ("a", "b"):
        scores |= set(F.z[f"score_{cap}_0"].tolist())
    assert {1800, 1400, 900, 700, 1600, 1000, 800, 750, -1, -2} <= scores, sorted(scores)
    fr = F.want("a", "mag", 0)[0]
    long_fix = set(fr["fix_bit"][fr["msgbits"] == 112].tolist())
    short_fix = set(fr["fix_bit"][fr["msgbits"] == 56].tolist())
    assert set(range(5, 112)) <= long_fix
    # DF11 bits 49..55: their single-bit syndromes are below 0x80, so scoreModesMessage takes them for an IID (mode_s.c:365) and
    # never repairs them; 5..48 is every short position the reference can repair
    assert set(range(5, 49)) <= short_fix and not short_fix & set(range(49, 56))
    dfs = {bytes.fromhex(c["msg"])[0] >> 3 for c in F.cases("a")}
    assert dfs == set(range(32))
    assert {c["msg"][:2] for c in F.cases("a") if c["name"].startswith("df17_")} >= {f"{(17 << 3) | ca:02x}" for ca in range(8)}


def test_signal_levels_reach_both_sides_of_minus_3_dbfs():
    F = fixture()
    for kind in KINDS:
        st = F.want("a", kind, 0)[3]
        assert 0 < st["strong_signal_count"] < sum(st["demod_accepted"])
    levels = F.want("a", "mag", 0)[1]
    assert (levels > 0.50119).any() and ((levels > 0.45) & (levels <= 0.50119)).any()


def _window(mag, c):
    return mag[c["pa"]: c["pa"] + 20].astype(np.int64)


def test_exact_ties_are_in_the_magnitude_capture():
    """The comparisons a kernel can get wrong by one: the pre-check's strict `>`, the correlators' `>= ref_level` for every
    threshold of the option sets, the slicers' `> 0` and magnitudes 0 / 65535."""
    F = fixture()
    mag = F.capture("a", "mag")
    cases = [c for c in F.cases("a") if c["family"] == "D"]
    pre = [(c, _window(mag, c)) for c in cases if c["name"].startswith("precheck")]
    for i, j in ((1, 7), (12, 14), (12, 15)):
        assert any(w[i] == w[j] for c, w in pre if f"pa{i}_pa{j}_equal" in c["name"])
        assert any(w[i] == w[j] + 1 for c, w in pre if f"pa{i}_pa{j}_plus1" in c["name"])
    seen = set()
    for c in cases:
        if "thr" in c:
            w = _window(mag, c)
            d23, s14, d1011 = w[2] - w[3], w[1] + w[4], w[10] - w[11]
            corr = [s14 - d23 + w[9] + w[12] - d1011, s14 - d23 + w[9] + w[12] + d1011, s14 + 2 * d23 + d1011 + w[12]][c["corr"]]
            ref_level = ((w[5] + w[8] + w[16] + w[17] + w[18]) * c["thr"]) >> 5
            seen.add((c["thr"], c["corr"], int(corr - ref_level)))
    assert seen >= {(o[0], k, d) for o in F.options for k in range(3) for d in (0, -1)}
    coef = {0: (18, -15, -3, 0), 1: (14, -5, -9, 0), 2: (16, 5, -20, 0), 3: (7, 11, -18, 0), 4: (4, 15, -20, 1)}
    gen = _generator()
    zero = 0
    for c in cases:
        if "bit" in c:
            (s, f), = gen.bit_cells(c["pa"], c["phase"], c["bit"])
            zero += sum(k * int(mag[s + q]) for q, k in enumerate(coef[f])) == 0
    assert zero >= 10
    assert any(mag[c["pa"]: c["pa"] + 300].min() == 0 and mag[c["pa"]: c["pa"] + 300].max() == 65535 for c in cases)


def test_placement_reaches_the_boundaries():
    """Family C: frames at -3..+2 of every kind of kernel boundary, at the first and last positions of buffers, across a sub-range
    boundary with their skip, and pairs at skip - 1 / skip / skip + 1 whose first frame the reference accepted (or rejected)."""
    F = fixture()
    cases = F.cases("c")
    L = F.buf("c")
    names = " ".join(c["name"] for c in cases)
    for kind, P in (("chunk512", 512), ("tile2048", 2048), ("quad8192", 8192), ("run16384", 16384)):
        offs = {c["j"] % P for c in cases if c["name"].startswith(kind)}
        assert {0, 1, 2, P - 3, P - 2, P - 1} <= offs, (kind, sorted(offs))
    assert {c["j"] for c in cases if c["name"].startswith("edge_first")} == {0, 1, 2}
    assert {c["j"] for c in cases if c["name"].startswith("edge_last")} == {L - 1, L - 2, L - 3}
    assert "skip_across" in names
    fr = F.want("c", "mag", 0)[0]
    ts = fr["timestamp"].astype(np.int64)
    accepted_first = 0
    for c in cases:
        if c["name"].startswith("pair_first"):
            # the buffer clock counts from its halo; a strong frame may win at a neighbouring phase
            hit = bool((np.abs(ts - (5 * (c["pa"] + HALO) + c["phase"] + 768)) <= 5).any())
            assert hit == (not c["name"].startswith("pair_first_rejected")), c["name"]
            accepted_first += hit
    assert accepted_first == 12
