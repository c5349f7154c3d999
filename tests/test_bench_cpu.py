"""CPU-only: the bench.py contract the driver depends on, exercised through the reference arm (the only arm that runs
without a GPU) on a tiny configuration, plus the loud failure of the product arm when there is no GPU."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def run_bench(*args, env=None, timeout=600):
    proc = subprocess.run([sys.executable, str(ROOT / "bench.py"), *args], capture_output=True, text=True, timeout=timeout,
                          cwd=str(ROOT), env=env)
    return proc


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    proc = run_bench("--impl", "reference", "--model", "tiny", "--batch", "4", "--seq", "32", "--new", "8", "--steps", "2",
                     "--warmup", "1", "--cpu-sample", "4")
    assert proc.returncode == 0, proc.stderr[-2000:]
    lines = [ln for ln in proc.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    for k in ("metric", "value", "unit", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config"):
        assert k in d, k
    assert d["unit"] == "tokens/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["value"] > 0 and d["ms_per_step"] > 0 and "workload" in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_product_arm_fails_loudly_without_a_gpu():
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    proc = run_bench("--model", "tiny", "--batch", "4", "--seq", "32", "--new", "8", "--steps", "1", "--warmup", "3",
                     "--no-cpu-baseline")
    assert proc.returncode != 0
    assert "no CPU fallback" in (proc.stderr + proc.stdout) or "CUDA" in (proc.stderr + proc.stdout)
    assert not any(ln.lstrip().startswith("{") for ln in proc.stdout.splitlines())  # no number is reported
