"""-m gpu: bench.py --dump-outputs writes what the timed path returned, the same for the same arguments."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.gpu


def test_bench_dump_outputs_are_reproducible(cuda, tmp_path):
    args = [sys.executable, str(ROOT / "bench.py"), "--steps", "2", "--warmup", "1", "--launches-per-step", "2", "--streams", "8",
            "--buffers", "2", "--ring", "2", "--no-extra", "--no-e2e", "--no-cpu"]
    dumps = []
    for run in ("a", "b"):
        out = subprocess.run(args + ["--dump-outputs", str(tmp_path / run)], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        line = json.loads(out.stdout.strip().splitlines()[-1])
        assert line["steps"] == 2 and line["gpu_launches"] > 0 and line["dumped_outputs"]["bytes"] <= 64 << 20
        dumps.append({p.stem: np.load(p) for p in (tmp_path / run).glob("*.npy")})
    a, b = dumps
    assert a.keys() == b.keys() and len(a["frames_timestamp"]) > 0 and len(a["buffers_length"]) == 8 * 2
    for name in a:
        assert a[name].dtype == np.float64 and np.array_equal(a[name], b[name]), name
