"""sc16 / sc16q11 steps at the bench shape (256 receivers x 8 buffers x 65536 samples, pipelined, three steps in flight):
throughput device-resident and from pinned host memory with uc8 timed alternately beside them, the converter kernel's own time
against its 6 bytes of traffic per sample, the per-buffer time of the submit_iq_sc16 path, and the card it all ran on.  Before
the timed windows, the first pipelined sc16 step of each format is checked against the same step through the blocking call.

    python tools/gpu_sc16_timing.py [--out DIR]      (needs an H100; prints one JSON line, and with --out also writes DIR/sc16_timing.json)

--submit-only times only the submit path (copied into another checkout, it gives the per-buffer figure of that build)."""
import argparse
import json
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch

from readsb_b200 import synth
from readsb_b200.demod import Demodulator, PinnedBuffer

S, B, BUF, R = 256, 8, 65536, 2          # R distinct steps of input per receiver, replayed (continues within the ring)
STEP = S * B * BUF
FMTS = ("uc8", "sc16", "sc16q11")


def to16(iq8: np.ndarray, q11: bool, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    scale = 16 if q11 else 256
    v = (iq8.astype(np.int32) - 128) * scale + rng.integers(0, scale, size=iq8.size)
    return np.clip(v, -2048 if q11 else -32768, 2047 if q11 else 32767).astype(np.int16)


class Card:
    """Name, power limit and the SM clock sampled every millisecond while a window runs (NVML queries only)."""

    def __init__(self):
        import pynvml as nv
        nv.nvmlInit()
        self.nv, self.h = nv, nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        self.samples, self.on, self.stop = [], False, False
        threading.Thread(target=self._loop, daemon=True).start()

    def info(self):
        nv, h = self.nv, self.h
        name = nv.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                "sm_max_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)}

    def _loop(self):
        while not self.stop:
            if self.on:
                self.samples.append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
            time.sleep(0.001)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory for sc16_timing.json (default: print only)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--submit-only", action="store_true")
    args = ap.parse_args()
    out = Path(args.out) if args.out else None
    if out:
        out.mkdir(parents=True, exist_ok=True)
    card = Card()
    res = {"card": card.info(), "shape": {"receivers": S, "buffers": B, "buf_samples": BUF, "depth": 3}}

    # per-buffer time of submit_iq_sc16 + run, 4 receivers x 8 buffers
    base = [synth.config2_stream(900 + i, R * B * BUF) for i in range(16)]
    small = [to16(base[s], False, s) for s in range(4)]
    d = Demodulator(n_streams=4, buf_samples=BUF, max_buffers_per_run=B)
    ts = []
    for rep in range(6):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for k in range(B):
            for s in range(4):
                d.submit_iq_sc16(s, small[s][2 * k * BUF: 2 * (k + 1) * BUF], (rep * B + k) * BUF * 5)
        d.run()
        ts.append((time.perf_counter() - t0) / (4 * B) * 1e6)
    d.close()
    res["submit_path_us_per_buffer"] = {"median": float(np.median(ts[1:])), "all": ts}
    if args.submit_only:
        print(json.dumps(res))
        if out:
            (out / "sc16_timing_submit.json").write_text(json.dumps(res, indent=1))
        return

    # inputs: receiver s replays capture s % 16, shifted; R steps per receiver row
    n = R * B * BUF
    host = {"uc8": np.stack([np.roll(base[s % 16], 2 * 1013 * (s // 16)) for s in range(S)])}
    for f, q11 in (("sc16", False), ("sc16q11", True)):
        rows = [to16(base[i], q11, i) for i in range(16)]
        host[f] = np.stack([np.roll(rows[s % 16], 2 * 1013 * (s // 16)) for s in range(S)])
    pad = 4096
    dev, pin = {}, {}
    for f in FMTS:
        h = host[f].view(np.uint8).reshape(S, -1)
        dev[f] = torch.zeros(pad + h.size + 256, dtype=torch.uint8, device="cuda")
        dev[f][pad:pad + h.size] = torch.from_numpy(h.reshape(-1)).cuda()
        pin[f] = PinnedBuffer(h.size)
        pin[f].array[:] = h.reshape(-1)
    torch.cuda.synchronize()
    bps = {"uc8": 2, "sc16": 4, "sc16q11": 4}

    def step_args(f, k, host_mem):
        row = n * bps[f]
        ptr = (pin[f].ptr if host_mem else dev[f].data_ptr() + pad) + (k % R) * B * BUF * bps[f]
        return (ptr, row, B, BUF, (k % R) > 0, k * B * BUF * 5)

    def launch(d, f, k, host_mem):
        a = step_args(f, k, host_mem)
        if f == "uc8":
            (d.run_host_async if host_mem else d.run_device_async)(*a)
        else:
            (d.run_host_sc16_async if host_mem else d.run_device_sc16_async)(*a, f == "sc16q11")

    def results(d):
        return [(d.frames(s).tobytes(), d.buffer_results(s).tobytes()) for s in range(S)]

    # the first timed step of a pipelined session equals the blocking call on the same steps
    checks = {}
    for f in ("sc16", "sc16q11"):
        p = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B)
        q = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B)
        warm = 5
        for k in range(warm + 1):
            launch(p, f, k, False)
            if k >= 2:
                p.wait()
        for k in range(warm + 1):
            q.run_device_sc16(*step_args(f, k, False), f == "sc16q11")
        p.wait(); p.wait()          # steps warm-1 and warm (the first timed one)
        checks[f] = results(p) == results(q)
        p.close(); q.close()
    res["first_timed_step_equals_blocking"] = checks

    # throughput: each window about a second of pipelined steps, formats and memory kinds alternating
    ctx = {(f, hm): Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B) for f in FMTS for hm in (False, True)}
    kstep = {key: 0 for key in ctx}

    def window(key, seconds):
        d, (f, hm) = ctx[key], key
        k0 = kstep[key]
        torch.cuda.synchronize()
        card.samples.clear(); card.on = True
        t0 = time.perf_counter()
        for k in range(k0, k0 + 2):
            launch(d, f, k, hm)
        k = k0 + 2; done = 0
        while True:
            launch(d, f, k, hm); k += 1
            d.wait(); done += 1
            if time.perf_counter() - t0 >= seconds:
                break
        d.wait(); d.wait(); done += 2
        el = time.perf_counter() - t0
        card.on = False
        kstep[key] = k + 1
        kstep[key] += (R - kstep[key] % R) % R          # next window starts a ring cycle (continues from a step in the ring)
        return done * STEP / el / 1e6, float(np.median(card.samples)) if card.samples else None

    for key in ctx:
        window(key, 0.3)                                # warm-up
    thr = {f"{f}_{'host' if hm else 'device'}": [] for f, hm in ctx}
    clocks = []
    for _ in range(args.rounds):
        for key in ctx:
            v, mhz = window(key, 1.0)
            thr[f"{key[0]}_{'host' if key[1] else 'device'}"].append(v); clocks.append(mhz)
    res["msamples_per_s"] = {k: {"median": float(np.median(v)), "all": v} for k, v in thr.items()}
    res["sm_mhz_median"] = float(np.median([c for c in clocks if c]))
    for d in ctx.values():
        d.close()

    # the converter kernel's own time (CUPTI via torch.profiler, in a run of its own)
    from torch.profiler import ProfilerActivity, profile
    d = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B)
    for k in range(4):
        launch(d, "sc16", k, False)
        if k >= 2:
            d.wait()
    d.wait(); d.wait()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(4, 16):
            launch(d, "sc16", k, False)
            if k >= 6:
                d.wait()
        d.wait(); d.wait()
        torch.cuda.synchronize()
    d.close()
    ev = [e for e in prof.key_averages() if "sc16_convert_kernel" in e.key]
    us = float(getattr(ev[0], "device_time", 0) or getattr(ev[0], "cuda_time", 0))         # mean over the launches
    nbytes = STEP * 6          # 4 bytes in, 2 bytes out per sample (+ 326 halo samples per receiver on continued steps)
    res["converter_kernel"] = {"launches": ev[0].count, "us_mean": us, "bytes_per_step": nbytes,
                               "gb_per_s": nbytes / (us * 1e-6) / 1e9, "share_of_3_35_tb_s": nbytes / (us * 1e-6) / 3.35e12}
    card.stop = True
    if out:
        (out / "sc16_timing.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
