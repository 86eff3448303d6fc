"""CPU: the reference arm of bench.py (the oracle port on the host cores) prints ONE JSON line with the
contract's keys; the GPU arm refuses to run without a CUDA device instead of falling back to the CPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*flags):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *flags], capture_output=True, text=True,
                          cwd=ROOT, timeout=600)


def test_reference_arm_prints_the_contract_line():
    r = _run("--impl", "reference", "--gaussians", "50000", "--steps", "1", "--warmup", "1")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "gaussians_rasterized_per_sec_fwd_bwd"
    assert d["unit"] == "Gaussians/s" and d["higher_is_better"] is True and d["n_gpus"] == 1
    assert d["steps"] == 1 and d["warmup"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["gpu_launches"] == 0 and d["vs_baseline"] is None and "workload" in d["config"]


def test_b200_arm_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a CUDA device is present")
    r = _run("--steps", "1", "--warmup", "1")
    assert r.returncode != 0
    assert "no CPU fallback" in r.stderr
