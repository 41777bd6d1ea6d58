"""Instruction model of scan_kernel: dynamic trip counts (from the kernels' source run under the SIMT emulator with
-DB200_SCAN_COUNTERS, tests/emu/) x static SASS instruction counts per section (nvdisasm of the sm_90a cubin, inline chains
resolved; numbers below were read off HEAD's cubin — re-derive them with `nvdisasm --print-line-info-inline` after changing
the kernel).  TEST / ANALYSIS TOOLING; says where the warp instructions go, not how long they take.

    python tools/scan_model.py [cfg2|cfg5]
"""
from __future__ import annotations

import ctypes
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "tests" / "emu"))

# static warp instructions per trip (fast paths; out-of-line divergence handlers of the collectives not counted)
STATIC = {
    "window_pass (pre-check 16 positions + 80 ticks per lane)": ("window_chunks", 429),
    "convert_chunk_fast (8 sample pairs through the table, sums, REDUX)": ("fast_converts", 191),
    "q1 compaction: prefix scan": ("window_chunks", 50),
    "q1 compaction: one pass of the set-bit loop": ("q1_loop_trips", 17),
    "chunk loop control, staging, classification (fast chunk)": ("loop_iters", 60),
    "threshold batch (32 pre-check passers)": ("thr_batches", 66),
    "batch with threshold passers: PosEntry writes": ("pass_batches", 28),
    "DF-gate trip (32 (position, phase) slots)": ("gate_trips", 90),
    "slice round: per message byte": ("slice_bytes", 30),
    "slice round: classification + emission": ("slice_rounds", 170),
    "run set-up and end of run": ("runs", 420),
}
NAMES = ["runs", "loop_iters", "window_chunks", "fast_converts", "edge_converts", "q1_entries", "q1_loop_trips", "thr_batches",
         "pass_batches", "passers", "gate_trips", "survivors", "slice_rounds", "slice_bytes"]


def main():
    wl = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
    os.environ["B200_EMU"] = "1"
    os.environ.setdefault("B200_EMU_SMS", "8")
    import build_emu
    lib = build_emu.build(defines=("B200_SCAN_COUNTERS",), sanitize=os.environ.get("SCAN_MODEL_SANITIZE"))
    os.environ["B200_DEMOD_LIB"] = str(lib)
    import numpy as np
    import devbuf
    from readsb_b200 import synth
    from readsb_b200.demod import Demodulator
    S, B, BUF = 64, 8, 65536                      # a quarter of the bench step (256 receivers): same per-chunk statistics
    gen = synth.config5_stream if wl == "cfg5" else synth.config2_stream
    base = [gen(900 + i, 2 * B * BUF) for i in range(8)]
    host = np.stack([np.roll(base[s % 8], 2 * 1013 * (s // 8)) for s in range(S)])
    pad = 4096
    dev = devbuf.zeros(pad + host.size + 256); dev[pad:pad + host.size] = host.reshape(-1)
    d = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B)
    cnt = (ctypes.c_ulonglong * 16).in_dll(ctypes.CDLL(str(lib)), "b200_scan_counters")
    for k in range(2):                              # second step: receivers' filters warm, halo continues
        for i in range(16):
            cnt[i] = 0
        d.run_device(dev.data_ptr() + pad + k * B * BUF * 2, host.shape[1], B, BUF, continues=k > 0, first_sample_timestamp=k * B * BUF * 5)
    c = dict(zip(NAMES, list(cnt)))
    samples = S * B * BUF
    print(f"workload {wl}: {samples} samples, {c['window_chunks']} chunks of 512 (look-ahead chunks included: x{c['window_chunks'] * 512 / samples:.3f})")
    print(f"per chunk: {c['q1_entries'] / c['window_chunks']:.1f} pre-check passers, {c['passers'] / c['window_chunks']:.2f} threshold passers, "
          f"{c['survivors'] / c['window_chunks']:.2f} DF-gate survivors; edge converts {c['edge_converts']}")
    rows, total = [], 0.0
    for name, (key, static) in STATIC.items():
        n = c[key] * static
        rows.append((name, c[key] / c['window_chunks'], static, n)); total += n
    for name, trips, static, n in rows:
        print(f"  {name:<68} {trips:7.3f} trips/chunk x {static:4d} = {n / samples:6.3f} instr/sample  {100 * n / total:5.1f} %")
    print(f"  {'model total':<68} {'':>28} {total / samples:6.3f} warp instructions per sample")


if __name__ == "__main__":
    main()
