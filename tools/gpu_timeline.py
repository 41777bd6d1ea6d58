"""Kernel timeline of the pipelined device-resident path at the bench shape, from torch.profiler (CUDA activities).

    python tools/gpu_timeline.py --out DIR [--launches 12] [--warmup 160] [--depth 3] [--workload config3_256streams]

Runs bench.py's `value` loop (256 receivers x 8 buffers x 65536 samples per launch, inputs resident in HBM, `--depth` steps in
flight) long enough for the session to settle its SM partition (demod_api.cu tune_partition), then traces `--launches` more.
Writes DIR/timeline.json (chrome trace) and prints, per kernel in GPU start order: start, duration, stream, the idle time of
the whole GPU before it, and which step it belongs to; then the mean step period and, per step, how long after its scan ended
its stage B started and its results were complete.  Profile in a run of its own: tracing slows the host.
"""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--launches", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=160)
    ap.add_argument("--depth", type=int, default=3)
    ap.add_argument("--streams", type=int, default=256)
    ap.add_argument("--buffers", type=int, default=8)
    ap.add_argument("--workload", choices=["config3_256streams", "config5_dense"], default="config3_256streams")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from readsb_b200.demod import Demodulator

    S, B, R, BUF = args.streams, args.buffers, 4, bench.BUF
    per_stream = R * B * BUF
    host = np.empty((S, 2 * per_stream), dtype=np.uint8)
    bench.generate_streams(S, per_stream, 1, args.workload, host)
    pad = 4096
    dev = torch.zeros(pad + host.size + 256, dtype=torch.uint8, device="cuda")
    dev[pad:pad + host.size] = torch.from_numpy(host.reshape(-1)).cuda()
    torch.cuda.synchronize()
    d = Demodulator(n_streams=S, buf_samples=BUF, max_buffers_per_run=B)
    d.set_stream(torch.cuda.current_stream().cuda_stream)

    def step(k):
        d.run_device_async(dev.data_ptr() + pad + (k % R) * B * BUF * 2, 2 * per_stream, B, BUF, continues=(k % R) > 0,
                           first_sample_timestamp=k * B * BUF * 5)

    def loop(k0, n):
        flying = 0
        for k in range(k0, k0 + n):
            step(k); flying += 1
            if flying == args.depth:
                d.wait(); flying -= 1
        while flying:
            d.wait(); flying -= 1
        torch.cuda.synchronize()

    loop(0, args.warmup)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loop(args.warmup, args.launches)
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    prof.export_chrome_trace(str(out / "timeline.json"))
    d.close()

    ev = json.loads((out / "timeline.json").read_text())["traceEvents"]
    ks = sorted([e for e in ev if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "dur" in e], key=lambda e: e["ts"])
    t0 = ks[0]["ts"]
    rows, busy_until, scan_i = [], t0, -1
    for e in ks:
        name = e["name"].split("(")[0].split("<")[0].replace("void ", "")
        if e["cat"] != "kernel":
            name = e["cat"].replace("gpu_", "") + " " + e["name"][:20]
        if name == "scan_kernel":
            scan_i += 1
        rows.append({"name": name, "ts": e["ts"] - t0, "dur": e["dur"], "stream": e.get("args", {}).get("stream"),
                     "idle_before": max(0.0, e["ts"] - busy_until), "scan_idx": scan_i})
        busy_until = max(busy_until, e["ts"] + e["dur"])
    print("%-26s %10s %9s %7s %10s  %s" % ("kernel", "start_us", "dur_us", "stream", "gpu_idle", "scan running / last started"))
    for r in rows:
        print("%-26s %10.1f %9.1f %7s %10.1f  %d" % (r["name"][:26], r["ts"], r["dur"], r["stream"], r["idle_before"], r["scan_idx"]))
    scans = [r for r in rows if r["name"] == "scan_kernel"]
    if len(scans) > 2:
        per = np.diff([r["ts"] for r in scans])
        print("scan kernels: %d, mean %.1f us each; scan start to next scan start: mean %.1f us, median %.1f us"
              % (len(scans), np.mean([r["dur"] for r in scans]), per.mean(), np.median(per)))
        gaps = [scans[i + 1]["ts"] - (scans[i]["ts"] + scans[i]["dur"]) for i in range(len(scans) - 1)]
        print("between one scan's end and the next scan's start: mean %.1f us, median %.1f us" % (np.mean(gaps), np.median(gaps)))
    names = sorted({r["name"] for r in rows})
    summary = {n: {"count": sum(1 for r in rows if r["name"] == n), "mean_us": float(np.mean([r["dur"] for r in rows if r["name"] == n]))} for n in names}
    print(json.dumps(summary))
    (out / "timeline_rows.json").write_text(json.dumps(rows))


if __name__ == "__main__":
    main()
