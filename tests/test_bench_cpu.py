"""bench.py's CPU-only arm (`--impl reference`): the driver launches it on the GPU box next to the GPU arm and parses ONE JSON
line with the contract's keys.  It times the oracle port of the reference path -- the one place outside tests/ where oracle/
may run (as the thing the GPU arm is compared with, never as the product)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_contract_line():
    t0 = time.time()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "tiny3", "--steps", "2", "--warmup", "1",
                        "--ref-procs", "1"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.strip().splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "config",
              "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["steps"] == 2 and d["warmup"] == 1 and d["higher_is_better"] is True
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"]
    split = d["latency_mode"]["time_split"]
    assert set(split) == {"cdf", "net", "pop", "push", "tables"} and abs(sum(split.values()) - 1.0) < 1e-6
    print(f"reference arm (tiny3, 1 worker): {d['value']:.5f} Mpixel/s, {time.time() - t0:.1f} s wall")

