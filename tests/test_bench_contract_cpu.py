"""The driver-facing contract of bench.py that can be checked without a GPU: the reference arm prints ONE JSON line with the
agreed keys (and does nothing on ranks != 0), and the GPU arm fails loudly — no silent CPU fallback — when no GPU exists."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None, timeout=600):
    e = dict(os.environ); e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, timeout=timeout, env=e, cwd=ROOT)


def test_reference_arm_json_line():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "0"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["metric"] == "features+matches/sec" and d["higher_is_better"] is True and d["value"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["config"]["workload"] == "batch640"


def test_reference_arm_is_silent_on_other_ranks():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "0", "--gpus", "2"], env={"RANK": "1", "WORLD_SIZE": "2"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_b200_arm_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    r = _run(["--steps", "1", "--warmup", "3", "--no-cpu-baseline"], timeout=300)
    assert r.returncode != 0 and not any(l.startswith("{") for l in r.stdout.splitlines())
