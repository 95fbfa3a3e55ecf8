"""CPU: the reference arm of bench.py (`--impl reference`: the oracle port timed on host cores) prints one JSON line with
the keys its consumers read.  (The GPU arm needs a GPU.)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--arch", "vit_small", "--steps", "1",
                        "--warmup", "0", "--cpu-sample-batch", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines                      # exactly one line on stdout; progress goes to stderr
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "global_crops_per_sec" and d["unit"] == "global-crops/s"
    for k in ("value", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
              "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["value"] > 0 and d["higher_is_better"] is True and d["cpu_baseline"]["kind"] == "port"
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert "workload" in d["config"] and "model" not in d["config"]
