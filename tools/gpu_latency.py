"""BASELINE configs[1] alone: per-call latency of the drop-in's call shape (bench.py's latency leg), with the device timeline."""
import json, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench
print(json.dumps(bench.latency_leg(0, 3350.0, None), indent=1))
