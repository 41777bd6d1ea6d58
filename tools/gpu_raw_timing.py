"""Times b200_demod_fetch_raw against b200_demod_fetch_beast on a bench-shaped device step (256 receivers x 8 x 65536 samples,
Mode A/C on).  The first fetch of a run in a format encodes every receiver (one kernel launch), copies the packed records to
the host and returns receiver 0's; a call for another format or other flags encodes again.  Each figure is the host wall time
of such a first call (the call synchronises with its own stream), median of the repeats; the card and its power limit are
printed beside them."""
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from readsb_b200 import synth  # noqa: E402
from readsb_b200.demod import Demodulator  # noqa: E402

S, B, BUF, REPEATS = 256, 8, 65536, 20


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    print("device:", torch.cuda.get_device_name(0), "| nvidia-smi name, power limit:", q.stdout.strip() or q.stderr.strip())
    base = [synth.modeac_stream(900 + i, B * BUF) for i in range(16)]
    host = np.stack([np.roll(base[s % 16], 2 * 1013 * (s // 16)) for s in range(S)])
    pad = 4096
    dev = torch.zeros(pad + host.size + 4096, dtype=torch.uint8, device="cuda")
    dev[pad:pad + host.size] = torch.from_numpy(host.reshape(-1)).cuda()
    d = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B, mode_ac=True)
    d.run_device(dev.data_ptr() + pad, host.shape[1], B, BUF, continues=False, first_sample_timestamp=0)
    n_ac = sum(len(d.modeac(s)) for s in range(S))
    print(f"one step: {d.total_frames()} frames, {n_ac} Mode A/C replies, run_ms {d.timing()['run_ms']:.3f}")
    calls = {"beast": lambda: d.beast(0), "beast verbatim": lambda: d.beast(0, verbatim=True),
             "raw": lambda: d.raw(0), "raw mlat": lambda: d.raw(0, mlat=True), "raw mlat stdout": lambda: d.raw(0, mlat=True, stdout=True)}
    times = {k: [] for k in calls}
    sizes = {}
    for _ in range(REPEATS + 2):
        for k, f in calls.items():                       # each call changes format or flags: it encodes the whole run again
            t0 = time.perf_counter()
            out = f()
            times[k].append(time.perf_counter() - t0)
            sizes[k] = len(out)
    for k in calls:
        t = np.array(times[k][2:]) * 1e3
        print(f"{k:16s} first call of a run: median {np.median(t):.3f} ms, min {t.min():.3f} ms; receiver 0: {sizes[k]} bytes")
    d.close()


if __name__ == "__main__":
    main()
