"""-m "not gpu": the crafted Mode A/C captures of tests/golden/verdicts/modeac_verdicts.npz (tests/golden/make_modeac_verdicts.py)
against what the reference's demodulate2400AC returned for them.

- The oracle reproduces the fixture: replies (timestamp, f1_sample, code, buffer), per-buffer reply counts and the Mode S frames
  of the same buffers, for every capture and input kind (magnitudes with given levels or with their own sums, uc8, sc16, sc16q11).
- Where the reference can be built, the fixture made again in memory equals the committed one.
- The fixture reaches what it is for: every case meets its class, every reject reason is reached by a case that fails it alone,
  the exact ties hold in the magnitudes, all 26 clock phase offsets and every code bit occur, the noise floors wrap and vanish
  where they should, and the placement captures reach the buffer, skip and scan-tile edges they are named for.

The GPU side (tests/test_gpu_modeac_verdicts.py) compares the CUDA library with the same fixture."""
import importlib.util
import json
import re
from pathlib import Path

import numpy as np
import pytest

from oraclelib import Oracle, have_ref
from paritylib import diff_frames
from test_verdicts import FRAME_FIELDS

ROOT = Path(__file__).resolve().parent.parent
FIXTURE = ROOT / "tests" / "golden" / "verdicts" / "modeac_verdicts.npz"
AC_SRC = ROOT / "readsb_b200" / "csrc" / "modeac_kernel.cu"
HALO = 326
AC_FIELDS = ("timestamp", "f1_sample", "modeac", "buffer_idx")


def generator():
    spec = importlib.util.spec_from_file_location("make_modeac_verdicts", ROOT / "tests" / "golden" / "make_modeac_verdicts.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = generator()


class Fixture:
    def __init__(self):
        self.z = np.load(FIXTURE)
        self.meta = json.loads(bytes(self.z["meta"]).decode())

    def buf(self, cap):
        return self.meta["buf"][cap]

    def restart(self, cap):
        return set(self.meta["restart"].get(cap, []))

    def cases(self, cap):
        return self.meta["cases"][cap]

    def capture(self, cap, kind):
        src = {"given": "mag", "mag": "mag"}.get(kind, kind)
        return np.ascontiguousarray(self.z[f"{src}_{cap}"])

    def levels(self, cap):
        return self.z[f"lv_{cap}"]

    def want(self, cap, kind):
        """(Mode S frames, their signal levels, replies, per-buffer reply counts) the reference returned."""
        z = self.z
        return z[f"frames_{cap}_{kind}"], z[f"flevels_{cap}_{kind}"], z[f"ac_{cap}_{kind}"], z[f"acn_{cap}_{kind}"]

    def runs(self):
        return [(cap, kind) for cap, kinds in sorted(self.meta["kinds"].items()) for kind in kinds]


_FIX = []


def fixture() -> Fixture:
    if not _FIX:
        _FIX.append(Fixture())
    return _FIX[0]


def mag_buffers(cap, kind):
    """(data with its halo, length, sample timestamp, mean_level, mean_power) per buffer as the capture's frontend hands them
    over: magnitudes with the given levels or their own sums, or uc8 / sc16 / sc16q11 through the converter."""
    F = fixture()
    L = F.buf(cap)
    x = F.capture(cap, kind)
    restart = F.restart(cap) if kind in ("mag", "uc8") else set()
    if kind in ("given", "mag"):
        for b, data in G.buffers(x, L, restart):
            ml, mp = (float(F.levels(cap)[b, 0]), float(F.levels(cap)[b, 1])) if kind == "given" else G.sums_levels(data[HALO:])
            yield data, L, b * L * 5, ml, mp
        return
    halo = np.zeros(HALO, np.uint16)
    for b in range(x.size // 2 // L):
        if kind == "uc8":
            mag, sl, sp = Oracle.convert(x[2 * b * L: 2 * (b + 1) * L])
            ml, mp = float(np.float64(sl) / 65536.0 / L), float(np.float64(sp) / 65535.0 / 65535.0 / L)
        else:
            mag, sl, sp = Oracle.convert_sc16(x[2 * b * L: 2 * (b + 1) * L], kind == "sc16q11")
            ml, mp = float(sl / np.float32(L)), float(sp / np.float32(L))      # `sum_level / nsamples` in float (convert.c:243-249)
        if b in restart:
            halo = np.zeros(HALO, np.uint16)
        data = np.ascontiguousarray(np.concatenate([halo, mag]))
        yield data, L, b * L * 5, ml, mp
        halo = data[L: L + HALO].copy() if L >= HALO else np.zeros(HALO, np.uint16)


def diff_replies(got: np.ndarray, want: np.ndarray) -> list:
    if len(got) != len(want):
        return [f"{len(got)} replies, the reference has {len(want)}"]
    return [f"replies differ in {f} at {int(np.argmax(got[f] != want[f]))}" for f in AC_FIELDS if not np.array_equal(got[f], want[f])]


@pytest.mark.parametrize("cap_kind", [f"{c}-{k}" for c, k in Fixture().runs()])
def test_oracle_equals_the_reference_verdicts(cap_kind):
    cap, kind = cap_kind.split("-")
    orc, dem = Oracle(), Oracle()
    acs, counts, frames = [], [], []
    for b, (data, L, ts, ml, mp) in enumerate(mag_buffers(cap, kind)):
        a = orc.demodulate_ac_levels(data, L, ts, ml, mp)
        a["buffer_idx"] = b
        acs.append(a); counts.append(len(a))
        f, _ = dem.demodulate(data, L, ts)
        frames.append(f)
    wf, _, wa, wn = fixture().want(cap, kind)
    problems = diff_replies(np.concatenate(acs), wa) + diff_frames(np.concatenate(frames), wf, fields=FRAME_FIELDS)
    assert np.array_equal(np.array(counts, np.uint32), wn), "per-buffer reply counts differ"
    assert orc.stats()["demod_modeac"] == len(wa)
    assert not problems, "\n".join(problems)


needs_ref = pytest.mark.skipif(not have_ref(), reason="reference tree not available to build oracle/_ref")


@needs_ref
def test_committed_fixture_is_what_the_generator_makes():
    made = G.generate()
    z = fixture().z
    assert sorted(made) == sorted(z.files)
    for k in z.files:
        assert made[k].dtype == z[k].dtype and np.array_equal(made[k], z[k], equal_nan=made[k].dtype.kind == "f"), k


# ---- what the fixture reaches ------------------------------------------------------------------------------------------------
def _data(cap, b):
    F = fixture()
    return dict(G.buffers(F.capture(cap, "mag"), F.buf(cap), F.restart(cap)))[b].astype(np.int64)


def _verdicts(cap):
    """Per case of capture a / b (given levels): the model's conditions at its position, and the reference's replies in its buffer."""
    F = fixture()
    ac = F.want(cap, "given")[2]
    out = []
    for c in F.cases(cap):
        r = G.decide(_data(cap, c["buffer"]), c["j"], c["noise"])
        out.append((c, r, ac[ac["buffer_idx"] == c["buffer"]]))
    return out


@pytest.mark.parametrize("cap", ["a", "b"])
def test_every_case_meets_its_class(cap):
    checked = 0
    for c, r, got in _verdicts(cap):
        cls = c["expect"]
        if cls.startswith("accepted"):
            assert len(got) == 1 and got["f1_sample"][0] == c["j"] and got["modeac"][0] == int(cls[9:], 16), (c, got)
            assert r["ok"] and r["code"] == int(cls[9:], 16)
        elif cls.startswith("rejected"):
            assert len(got) == 0 and not r["ok"] and not r["cond"][cls[9:]], (c, got)
        checked += cls != "any"
        # the model and the reference agree on every case, classed or not
        assert (c["j"] in got["f1_sample"]) == r["ok"], c
    assert checked >= (80 if cap == "a" else 12)


def test_every_reject_reason_is_reached_alone():
    alone = {}
    for cap in ("a", "b"):
        for c, r, got in _verdicts(cap):
            failing = [k for k in G.CONDITIONS if not r["cond"][k]]
            if len(failing) == 1:
                assert len(got) == 0
                alone.setdefault(failing[0], []).append(c["name"])
    assert set(alone) == set(G.CONDITIONS), sorted(set(G.CONDITIONS) - set(alone))


def test_exact_ties_hold_in_the_magnitudes():
    """The comparisons a kernel can get wrong by one, each on both sides of its tie: (what, value - threshold) per case."""
    seen = set()
    for cap in ("a", "b"):
        for c, r, got in _verdicts(cap):
            m, j, n, name = _data(cap, c["buffer"]), c["j"], c["noise"], c["name"]
            f2 = (r["clock"] + 87 * 14) // 25
            cs = [j + s for s in G.cells(j, r["clock"])]
            w = name.split("_")
            ties = {"edge1": lambda: m[j - 1] - m[j], "edge2": lambda: m[f2 - 1] - m[f2],
                    "quiet1": lambda: m[j + 2] - min(m[j], m[j + 1]), "quiet2": lambda: m[f2 + 2] - min(m[f2], m[f2 + 1]),
                    "level1": lambda: 2 * n - (m[j] + m[j + 1]) // 2, "level2": lambda: 2 * n - (m[f2] + m[f2 + 1]) // 2,
                    "bit": lambda: m[cs[2] + int(w[1][1])] - r["sig"], "half": lambda: 2 * n - r["f1f2"],
                    "quiet_sample": lambda: m[cs[int(w[2])] + 2] - r["sig"],
                    "uncertain": lambda: min(m[cs[int(w[1])]], m[cs[int(w[1])] + 1]) - r["noi"]}
            key = "quiet_sample" if name.startswith("quiet_sample") else w[0]
            if key in ties and (key != "uncertain" or w[1].isdigit()):
                seen.add((key, int(ties[key]())))
            if name.startswith("phase_half_tie"):
                x = G.clock_x(j, m[j], m[j + 1])
                assert x - np.floor(x) == np.float32(0.5) and r["ok"]
                seen.add(("phase_half", int(r["clock"] - 25 * j)))
    for key, sides in (("edge1", (0, -1)), ("edge2", (0, -1)), ("quiet1", (0, 1)), ("quiet2", (0, 1)), ("level1", (0, 1)),
                       ("level2", (0, 1)), ("bit", (0, -1)), ("quiet_sample", (0, -1)), ("uncertain", (0, 1)), ("half", (0, 2))):
        assert {(key, v) for v in sides} <= seen, key
    assert len({v for k, v in seen if k == "phase_half"}) >= 2


def test_every_phase_offset_and_code_bit_is_reached():
    F = fixture()
    phases, codes = set(), set()
    for cap in ("a", "c65536", "cbig"):
        kind = "given" if cap == "a" else "mag"
        ac = F.want(cap, kind)[2]
        mags = dict(G.buffers(F.capture(cap, "mag"), F.buf(cap), F.restart(cap)))
        for a in ac:
            m, j = mags[int(a["buffer_idx"])], int(a["f1_sample"])
            clock = G.f1_clock(j, int(m[j]), int(m[j + 1]))
            assert int(a["timestamp"]) == int(a["buffer_idx"]) * F.buf(cap) * 5 + (clock + 87 * 14) // 5
            phases.add((cap, clock - 25 * j))
            codes.add(int(a["modeac"]))
    assert {p for c, p in phases if c == "a"} == set(range(26))
    assert {p for c, p in phases if c == "c65536"} >= {0, 6, 7, 25} and len({p for c, p in phases if c == "cbig"}) >= 10
    for cb in G.CODE_MAP.values():
        assert cb in codes, hex(cb)
    assert sum(G.CODE_MAP.values()) in codes and 0 in codes


def test_noise_floors_wrap_and_vanish_like_the_reference():
    """x86-64 converts the floor through 64 bits: it wraps past 2^32 and is 0 for NaN, inf and 2^63 on."""
    F = fixture()
    cases = {c["name"]: c for c in F.cases("b")}
    lv = F.levels("b")
    ac = F.want("b", "given")[2]
    acc = lambda n: bool((ac["buffer_idx"] == cases[n]["buffer"]).any())                # noqa: E731
    raw = lambda n: (lv[cases[n]["buffer"], 1] + np.sqrt(lv[cases[n]["buffer"], 1] - lv[cases[n]["buffer"], 0] ** 2)) * 65535 + 0.5   # noqa: E731
    with np.errstate(invalid="ignore"):
        assert 2 ** 31 <= raw("wrap2_even") < 2 ** 32 and acc("wrap2_even") and not acc("wrap2_even_high")
        assert 2 ** 32 <= raw("beyond_2_32") < 2 ** 33 and cases["beyond_2_32"]["noise"] == 1000 and acc("beyond_2_32")
        assert raw("far_beyond") > 2 ** 40 and acc("far_beyond") and raw("huge") >= 2.0 ** 63 and not acc("huge")
        for n in ("nan", "neg_var_tiny"):
            assert np.isnan(raw(n)) and cases[n]["noise"] == 0 and not acc(n)
        assert np.isinf(raw("inf")) and cases["inf"]["noise"] == 0 and not acc("inf")
    assert acc("half_level") and not acc("half_level_plus1")
    # the same replies with the buffers' own sums are all accepted; the sc16 captures end with a negative float variance
    assert len(F.want("b", "mag")[2]) == len(cases)
    for kind in ("sc16", "sc16q11"):
        x = F.capture("b", kind)
        _, sl, sp = Oracle.convert_sc16(x[-2 * F.buf("b"):], kind == "sc16q11")
        ml, mp = np.float64(sl / np.float32(F.buf("b"))), np.float64(sp / np.float32(F.buf("b")))
        assert mp - ml * ml < 0
        assert F.want("b", kind)[3][-1] == 0 and len(F.want("b", kind)[2]) > 0


def test_placement_reaches_the_edges():
    F = fixture()
    L = F.buf("c65536")
    ac = F.want("c65536", "mag")[2]
    got = set(zip(ac["buffer_idx"].tolist(), ac["f1_sample"].tolist()))
    hit = {c["name"]: (c["buffer"], c["j"]) in got for c in F.cases("c65536")}
    assert hit["f1_sample_1_buf2"] and hit["f1_sample_2_buf5"] and hit["last_65535_buf5"] and hit["last_65466_buf2"]
    # position 0 of a buffer is its predecessor's position `len`: neither reports it
    g0 = [c["g"] for c in F.cases("c65536") if c["name"] == "f1_sample_0_buf4"][0]
    assert not any(int(a["buffer_idx"]) * L - HALO + int(a["f1_sample"]) == g0 for a in ac)
    assert [hit[f"skip_second_{d}"] for d in (69, 70, 71)] == [False, True, True] and all(hit[f"skip_first_{d}"] for d in (69, 70, 71))
    assert hit["skip_into_next_first"] and hit["skip_into_next_second_69"]       # the skip does not carry into the next buffer
    assert not hit["in_zero_halo"] and hit["after_zero_halo"] and F.restart("c65536") == {3}
    dense = [c for c in F.cases("c65536") if c["name"] == "dense"]
    n_dense = int(F.want("c65536", "mag")[3][dense[0]["buffer"]])
    assert all(hit["dense"] for _ in [0]) and n_dense == len(dense) == (L - 2) // 70 + 1 and L // 70 < n_dense <= L // 70 + 2
    # replies whose F1 lies 49 .. 0 positions before a scan tile's end (F2 and the bit cells in the next tile and the look-ahead),
    # with F2 48 and 49 samples on
    mags = dict(G.buffers(F.capture("c65536", "mag"), L, F.restart("c65536")))
    edges = set()
    for c in F.cases("c65536"):
        if c["name"].startswith("tile_") and hit[c["name"]]:
            m, j = mags[c["buffer"]], c["j"]
            x = c["buffer"] * L + j                  # tile coordinate in a run that starts at buffer 0 (lead 0)
            f2 = (G.f1_clock(j, int(m[j]), int(m[j + 1])) + 87 * 14) // 25 - j
            edges.add((x % 2048 - 2048 if x % 2048 > 1024 else x % 2048, f2))
    assert {(dx, f2) for dx in (-49, -48, -2, -1) for f2 in (48, 49)} <= edges and {(0, 48), (0, 49)} <= edges
    # more than 32 front-test survivors in one 512-position chunk
    c = [c for c in F.cases("c65536") if c["name"] == "after_survivor_train"][0]
    m = mags[c["buffer"]]
    js = np.arange(1, L - 100)
    edge = (m[js - 1] < m[js]) & (m[js + 2] <= m[js]) & (m[js + 2] <= m[js + 1])
    front = [j for j in js[edge] if G.decide(m, int(j), G.noise_floor(*G.sums_levels(m[HALO:])))["cond"]["level2"]
             and G.decide(m, int(j), 0)["cond"]["edge2"]]
    per_chunk = np.bincount((c["buffer"] * L + np.array(front)) // 512)
    assert per_chunk.max() > 32 and hit["after_survivor_train"]
    # Mode S frames beside the replies
    assert len(F.want("c65536", "mag")[0]) >= 4
    # buffers that start inside a 32-position word of the reply map (8191 samples), with replies at their first positions
    ac8 = F.want("c8191", "mag")[2]
    firsts = {(int(a["buffer_idx"]), int(a["f1_sample"])) for a in ac8 if a["f1_sample"] < 8}
    assert {(b, (1, 2, 3, 4, 5, 1, 2, 3, 4, 5)[b]) for b in range(5, 10)} <= firsts
    # 1000-sample buffers: a 2048-position tile spans three of them, loud and quiet ones with floors far apart
    # (every reply accepted in a quiet buffer would fail its level test under a loud buffer's floor)
    mags = dict(G.buffers(F.capture("c1000", "mag"), 1000))
    loud = min(G.noise_floor(*G.sums_levels(mags[b][HALO:])) for b in range(1, len(mags), 3))
    ac = F.want("c1000", "mag")[2]
    quiet = [a for a in ac if a["buffer_idx"] % 3 != 1]
    levels = [(int(mags[int(a["buffer_idx"])][a["f1_sample"]]) + int(mags[int(a["buffer_idx"])][a["f1_sample"] + 1])) // 2 for a in quiet]
    assert len(quiet) > 60 and max(levels) < 2 * loud
    # 400-sample buffers in runs of eight: a tile's first buffers are bt and bt + 1 (loud); replies in bt + 2 .. are measured against
    # their own floor, which a loud one's would reject
    mags = dict(G.buffers(F.capture("c400", "mag"), 400))
    floor = {b: G.noise_floor(*G.sums_levels(d[HALO:])) for b, d in mags.items()}
    far = 0
    for a in F.want("c400", "uc8")[2]:
        b, j = int(a["buffer_idx"]), int(a["f1_sample"])
        b0 = b - b % 8
        bt = (((b - b0) * 400 + j) // SCAN_TILE * SCAN_TILE) // 400
        level = (int(mags[b][j]) + int(mags[b][j + 1])) // 2
        far += b - b0 - bt >= 2 and (b0 + bt + 1) % 3 == 1 and level < 2 * floor[b0 + bt + 1]
    assert far >= 3
    # buffers shorter than the halo: the next one starts with a zero halo (sdr_ifile.c:207-212), and nothing is found
    assert all(len(F.want(cap, k)[2]) == 0 for cap in ("c100", "c300") for k in ("mag", "uc8"))
    # f1_sample past 2^17 and 2^20
    big = F.want("cbig", "mag")[2]["f1_sample"]
    assert (big > 1 << 17).sum() >= 4 and (big > 1 << 20).sum() >= 3


# ---- the scan tile's magnitude sources -----------------------------------------------------------------------------------------
SCAN_TILE, B200_TRAIL, AC2_BEHIND, AC2_AHEAD = 2048, 326, 8, 104


def tile_sources(lead: int, npos: int, halo_zero: bool, is_mag: bool) -> list:
    """Where modeac_scan_kernel takes each tile's magnitudes from: the Mode S scan's copy ("mag_copy"), the samples converted in
    place ("convert"), a magnitude hand-off copied as it is ("copy"), or piece by piece with bounds tests ("bounds")."""
    n_tiles = (lead + npos + SCAN_TILE - 1) // SCAN_TILE
    x_data_end, x_zero_end = lead + npos + B200_TRAIL, lead + B200_TRAIL if halo_zero else lead
    out = []
    for t in range(n_tiles):
        x0 = t * SCAN_TILE
        if x0 >= x_zero_end + AC2_BEHIND and x0 + SCAN_TILE + AC2_AHEAD <= x_data_end:
            out.append("copy" if is_mag else "mag_copy" if x0 + SCAN_TILE + AC2_AHEAD <= n_tiles * SCAN_TILE else "convert")
        else:
            out.append("bounds")
    return out


def test_tile_source_rule_is_the_kernels():
    src = AC_SRC.read_text()
    assert "#define AC2_BEHIND 8\n" in src and "#define AC2_AHEAD 104\n" in src
    assert "const uint32_t x_data_end = seg.lead + seg.npos + B200_TRAIL;" in src
    assert "const uint32_t x_zero_end = (seg.flags & SEG_HALO_ZERO) ? seg.lead + B200_TRAIL : seg.lead;" in src
    assert "if (x0 >= x_zero_end + AC2_BEHIND && x0 + SCAN_TILE + AC2_AHEAD <= x_data_end) {" in src
    assert "if (convert && P.mag_copy && x0 + SCAN_TILE + AC2_AHEAD <= seg.n_tiles * SCAN_TILE) {" in src
    common = (AC_SRC.parent / "common.h").read_text()
    assert re.search(r"#define SCAN_TILE\s+2048\b", common) and re.search(r"#define B200_TRAIL\s+326\b", common)
    assert "g.n_tiles = npos ? (g.lead + npos + SCAN_TILE - 1) / SCAN_TILE : 0;" in (AC_SRC.parent / "demod_api.cu").read_text()


def test_every_tile_source_holds_replies():
    """submit_iq + run with eight buffers per run (one segment per run, lead 0, the arena's first bytes): the 65536- and
    8191-sample captures put accepted replies in tiles of every kind, the restarted buffer's first tile included."""
    F = fixture()
    seen = set()
    for cap in ("c65536", "c8191"):
        L = F.buf(cap)
        ac = F.want(cap, "uc8")[2]
        nb = F.capture(cap, "uc8").size // 2 // L
        restart = F.restart(cap)
        b0 = 0
        while b0 < nb:                               # the runs the GPU test makes: eight buffers, or up to a restart
            b1 = min(b0 + 8, nb)
            b1 = min([r for r in restart if b0 < r < b1] + [b1])
            src = tile_sources(0, (b1 - b0) * L, b0 == 0 or b0 in restart, False)
            for a in ac[(ac["buffer_idx"] >= b0) & (ac["buffer_idx"] < b1)]:
                x = (int(a["buffer_idx"]) - b0) * L + int(a["f1_sample"])
                seen.add((src[x // SCAN_TILE], b0 in restart and x < SCAN_TILE))
            b0 = b1
    assert {("mag_copy", False), ("convert", False), ("bounds", False), ("bounds", True)} <= seen, seen
    assert tile_sources(0, 65536, True, True)[1] == "copy"
