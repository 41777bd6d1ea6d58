"""Steps of independent receivers at the bench shape: 256 receivers x up to 8 buffers x 65536 samples, pipelined with three steps in
flight, each receiver's count drawn from {7, 8} per step and 5 % of the receivers absent (b200_demod_run_device_rx_async /
run_host_rx_async), timed alternately with the uniform step of the same size (run_device_*_async / run_host_*_async, 8 buffers each),
for uc8 and sc16, device-resident and from pinned host memory.  Rates count the samples the step delivered.  Also reports the card.

    python tools/gpu_rx_timing.py [--out DIR]      (needs an H100; prints one JSON line, and with --out also writes DIR/rx_timing.json)
"""
import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import numpy as np
import torch

from gpu_sc16_timing import Card, to16
from readsb_b200 import synth
from readsb_b200.abi import FORMAT_SC16, FORMAT_UC8, RX_CONTINUES, RX_STEP_DTYPE
from readsb_b200.demod import Demodulator, PinnedBuffer

S, B, BUF, R = 256, 8, 65536, 2          # R distinct steps of input per receiver, replayed
FMTS = {"uc8": (FORMAT_UC8, 2), "sc16": (FORMAT_SC16, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory for rx_timing.json (default: print only)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    out = Path(args.out) if args.out else None
    if out:
        out.mkdir(parents=True, exist_ok=True)
    card = Card()
    res = {"card": card.info(), "shape": {"receivers": S, "buffers": B, "buf_samples": BUF, "depth": 3, "counts": "{7, 8}, 5 % absent"}}

    base = [synth.config2_stream(900 + i, R * B * BUF) for i in range(16)]
    host = {"uc8": np.stack([np.roll(base[s % 16], 2 * 1013 * (s // 16)) for s in range(S)])}
    rows16 = [to16(base[i], False, i) for i in range(16)]
    host["sc16"] = np.stack([np.roll(rows16[s % 16], 2 * 1013 * (s // 16)) for s in range(S)])
    pad = 4096
    dev, pin = {}, {}
    for f in FMTS:
        h = host[f].view(np.uint8).reshape(S, -1)
        dev[f] = torch.zeros(pad + h.size + 256, dtype=torch.uint8, device="cuda")
        dev[f][pad:pad + h.size] = torch.from_numpy(h.reshape(-1)).cuda()
        pin[f] = PinnedBuffer(h.size)
        pin[f].array[:] = h.reshape(-1)
    torch.cuda.synchronize()

    # descriptor arrays drawn once per step index of the ring: counts 7 / 8, 5 % absent; a receiver continues unless it was absent
    rng = np.random.default_rng(1)
    n_desc = 64
    counts = rng.choice([7, 8], size=(n_desc, S))
    counts[rng.random((n_desc, S)) < 0.05] = 0

    def launch(d, f, k, hm, rx_mode):
        fmt, bps = FMTS[f]
        row = R * B * BUF * bps
        ptr = (pin[f].ptr if hm else dev[f].data_ptr() + pad) + (k % R) * B * BUF * bps
        if not rx_mode:
            if f == "uc8":
                (d.run_host_async if hm else d.run_device_async)(ptr, row, B, BUF, k > 0, k * B * BUF * 5)
            else:
                (d.run_host_sc16_async if hm else d.run_device_sc16_async)(ptr, row, B, BUF, k > 0, k * B * BUF * 5)
            return S * B * BUF
        rx = np.zeros(S, RX_STEP_DTYPE)
        c = counts[k % n_desc]
        prev = counts[(k - 1) % n_desc]
        # continuing needs the previous step's samples in front on the device path: only within the ring and after a present step
        cont = (prev > 0) & (k > 0) & ((k % R) > 0 if not hm else True)
        rx["first_sample_timestamp"] = k * B * BUF * 5
        rx["n_buffers"] = c
        rx["flags"] = np.where(cont, RX_CONTINUES, 0)
        (d.run_host_rx_async if hm else d.run_device_rx_async)(fmt, ptr, row, BUF, rx)
        return int(c.sum()) * BUF

    ctx = {(f, hm, rxm): Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B) for f in FMTS for hm in (False, True) for rxm in (False, True)}
    kstep = {key: 0 for key in ctx}

    def window(key, seconds):
        d, (f, hm, rxm) = ctx[key], key
        k = kstep[key]
        torch.cuda.synchronize()
        card.samples.clear(); card.on = True
        t0 = time.perf_counter()
        flying, samples = [], 0
        while True:
            flying.append(launch(d, f, k, hm, rxm)); k += 1
            if len(flying) == 3:
                d.wait(); samples += flying.pop(0)
                if time.perf_counter() - t0 >= seconds:
                    break
        while flying:
            d.wait(); samples += flying.pop(0)
        el = time.perf_counter() - t0
        card.on = False
        kstep[key] = k
        return samples / el / 1e6, float(np.median(card.samples)) if card.samples else None

    for key in ctx:
        window(key, 0.3)                                # warm-up
    thr = {f"{f}_{'host' if hm else 'device'}_{'rx' if rxm else 'uniform'}": [] for f, hm, rxm in ctx}
    clocks = []
    for _ in range(args.rounds):
        for key in ctx:
            v, mhz = window(key, 1.0)
            thr[f"{key[0]}_{'host' if key[1] else 'device'}_{'rx' if key[2] else 'uniform'}"].append(v); clocks.append(mhz)
    res["msamples_per_s"] = {k: {"median": float(np.median(v)), "all": v} for k, v in thr.items()}
    res["sm_mhz_median"] = float(np.median([c for c in clocks if c]))
    for d in ctx.values():
        d.close()
    card.stop = True
    if out:
        (out / "rx_timing.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
