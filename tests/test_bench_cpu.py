"""bench.py's CPU arm (`--impl reference`) prints ONE JSON line with the contract's keys; the GPU arm refuses to run without a
device instead of falling back."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    j = json.loads(lines[0])
    assert j["impl"] == "reference" and j["metric"] == "ar_frames_per_sec" and j["unit"] == "frames/s" and j["higher_is_better"] is True
    assert j["value"] > 0 and j["steps"] == 1 and j["config"]["workload"].startswith("batch=64/GPU")
    assert j["e2e"] == {"value": j["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = j["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == j["value"]
    if cb["kind"] == "reference":  # the unmodified reference is installed under baseline/_ref: CLI timing points + TTFA
        st = cb["stages"]
        assert st["frames"] == 401 and st["rtf"] > 0 and st["ttfa_ms_p50"] > 0


def test_b200_arm_has_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "0"], capture_output=True, text=True,
                       timeout=300, cwd=ROOT)
    assert r.returncode != 0 and "no CUDA device" in (r.stderr + r.stdout)
