"""CPU: the parts of bench.py that are plain host logic and that a silent regression would turn into missing JSON keys — the
peak lookup, the workload table the flags select from, and the reference arm's JSON contract on a bounded step (the arm itself
is CPU code)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_peaks_and_workload_table():
    import bench
    p = bench.peaks()
    assert p["bf16_tflops"] > 500 and p["hbm_gbs"] > 3000 and p["src"]
    src = open(os.path.join(ROOT, "bench.py")).read()
    for name in ("gpt2-110m", "ziya-llama-13b", "megatronbert-1.3b", "bert-base", "randeng-t5-784m"):
        assert name in src
    assert bench.HEADLINE[8][0] == "ziya-llama-13b" and bench.HEADLINE[4][0] == "megatronbert-1.3b"


@pytest.mark.timeout(600)
def test_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (what the driver runs first at round end): one JSON line with the keys of the contract."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "1",
                          "--warmup", "0", "--workload", "bert-base"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "tokens_per_sec" and d["unit"] == "tokens/s" and d["value"] > 0
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"]
