"""BASELINE configs[1] alone: per-call latency of the drop-in's call shape (bench.py's latency leg), with the device timeline."""
import json, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench
print(json.dumps(bench.latency_leg(0, 3350.0, None), indent=1))

import ctypes as C, os
from readsb_b200.demod import lib
L = lib()
if hasattr(L, "b200_demod_debug_ctl"):       # analysis build (-DB200_SOLO_CLOCKS): the one-receiver stage B kernel's own timeline
    import numpy as np
    from readsb_b200 import synth
    from readsb_b200.demod import Demodulator
    d = Demodulator(n_streams=1, buf_samples=65536, max_buffers_per_run=1)
    iq = synth.config2_stream(7, 32 * 65536)
    rows = []
    for k in range(6 * 32):               # the bench leg's pattern: 32 buffers, over and over (every aircraft known after the first pass)
        b = k % 32
        d.submit_iq(0, iq[2 * b * 65536: 2 * (b + 1) * 65536], k * 65536 * 5); d.run()
        out = (C.c_uint32 * 8)(); L.b200_demod_debug_ctl(d.h, out)
        rows.append([out[1], out[6], out[7], out[5], out[0]])
    rows = rows[4 * 32:]
    r = np.median(np.array(rows), axis=0)
    print("solo kernel ns: check+tables %d, speculation %d, commit %d, write-back+prefix %d, finalize %d" % tuple(r))
