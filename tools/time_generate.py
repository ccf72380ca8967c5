"""BASELINE configs[4]: 10 s three-stage generation on the KV-cache decode path (bench.measure_generation)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import bench
r = bench.measure_generation()
print(json.dumps({k: r[k] for k in ("tokens_in_output", "ms_device", "ms_wall", "tokens_per_s", "audio_seconds_per_second")}), flush=True)
