"""Generates tests/golden/*.npz by running the REFERENCE ITSELF (oracle/_ref/libreadsb_ref.so, built from
/root/reference by oracle/Makefile) on small seeded synthetic captures.  Only runs where /root/reference exists;
the fixtures it writes are committed so the pin holds on boxes without the reference tree.

    python tests/golden/make_golden.py
"""
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from oraclelib import Reference  # noqa: E402
from readsb_b200 import synth  # noqa: E402

CASES = {
    # name: (generator kwargs, nsamples, buf_samples, demod options)
    "df17_sparse": (dict(seed=41, frames_per_sec=1500.0, df_mask=synth.DF17, n_icao=8), 70000, 32768, dict()),
    "dense_df11_df17": (dict(seed=42, frames_per_sec=10000.0, df_mask=synth.DF17 | synth.DF11, n_icao=16), 70000, 32768, dict()),
    "mixed_biterrors": (dict(seed=43, frames_per_sec=6000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP | synth.DF18 | synth.DF11_IID,
                             n_icao=6, p_bit_error=0.4, p_two_bit_error=0.1), 70000, 32768, dict()),
    "modeac_mix": (dict(seed=46, frames_per_sec=3000.0, df_mask=synth.MODEAC | synth.DF17, n_icao=8, amp=(0.4, 0.9)),
                   120000, 32768, dict()),
    "mixed_nofix": (dict(seed=44, frames_per_sec=6000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP, n_icao=6, p_bit_error=0.4),
                    50000, 65536, dict(nfix_crc=0)),
    "mixed_thr40_nofixdf": (dict(seed=45, frames_per_sec=6000.0, df_mask=synth.DF17 | synth.DF11 | synth.AP, n_icao=6, p_bit_error=0.4),
                            50000, 65536, dict(preamble_threshold=40, fix_df=0)),
}


def main():
    for name, (gen_kw, ns, buf, opts) in CASES.items():
        iq = synth.generate(ns, **gen_kw)
        ref = Reference(**opts)
        frames, levels, bufres, ml, mp = ref.run_stream(iq, buf)
        stats, dstats = ref.stats()
        modeac = Reference(**opts).run_stream_ac(iq, buf)      # demodulate2400AC of the same reference build, same buffers
        np.savez_compressed(HERE / f"{name}.npz", iq=iq, modeac=modeac, frames=frames, signal_level=levels, bufres=bufres, mean_level=ml,
                            mean_power=mp, meta=np.frombuffer(json.dumps(dict(buf_samples=buf, options=opts, stats=stats, dstats=dstats,
                                                                             generator=gen_kw)).encode(), dtype=np.uint8))
        print(name, len(frames), "frames", stats["demod_preambles"], "preambles")


def sc16_vectors():
    """The reference's float-path converters (convert.c:212-250, 329-367) on a small random block, both formats."""
    out = {}
    for q11 in (0, 1):
        rng = np.random.default_rng(90 + q11)
        lim = 2048 if q11 else 32768
        iq = rng.integers(-lim, lim, size=2 * 6001, dtype=np.int32)
        iq[:32] = [-lim, lim - 1] * 16
        iq[2000:6000] = rng.integers(-lim // 40, lim // 40, size=4000)
        iq = iq.astype(np.int16)
        mag, ml, mp = Reference().convert_sc16(iq, bool(q11))
        out[f"iq{q11}"] = iq; out[f"mag{q11}"] = mag; out[f"means{q11}"] = np.array([ml, mp], np.float64)
    np.savez_compressed(HERE / "sc16_converters.npz", **out)
    print("sc16_converters", {k: v.shape for k, v in out.items()})


CONFIG1_CAPTURE = dict(seed=2024, frames_per_sec=180.0, df_mask=synth.DF17 | synth.DF11 | synth.AP, n_icao=64, p_bit_error=0.1)


def config1_frames():
    """The reference's frames for tests/test_gpu_fullsize.py::test_config1_ten_second_replay (its 10 s capture is regenerated
    from the seed there, so only the frames are stored)."""
    iq = synth.generate(24_000_000, **CONFIG1_CAPTURE)
    frames = Reference().run_stream(iq, 131072, cap=8192)[0]
    (HERE / "replay").mkdir(exist_ok=True)
    np.savez_compressed(HERE / "replay" / "config1_10s.npz", frames=frames)
    print("config1_10s", len(frames), "frames")


if __name__ == "__main__":
    main()
    sc16_vectors()
    config1_frames()
