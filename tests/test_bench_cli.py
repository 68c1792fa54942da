"""bench.py's reference arm runs anywhere (it times the CPU port in oracle/): one JSON line on stdout with the
contract's keys, the same metric / unit / workload naming as the GPU arm, and nothing else on stdout.  Ranks
other than 0 exit without work (the driver launches the arm under torchrun at N > 1)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(env_extra, *args):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                       env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def test_reference_arm_prints_one_contract_line():
    out = run({}, "--impl", "reference", "--steps", "1", "--warmup", "0")
    lines = [l for l in out.splitlines() if l.strip()]
    assert len(lines) == 1, out
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "blocks/s" and d["higher_is_better"] is True
    assert d["metric"].startswith("RDO candidate blocks/s") and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["config"]["workload"] == "1080p-8bit-speed6-me16x16"
    c = d["cpu_baseline"]
    assert c["kind"] == "port" and c["cores"] >= 1 and c["value"] == d["value"] > 0 and c["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "blocks/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_reference_arm_other_ranks_do_no_work():
    out = run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}, "--impl", "reference", "--gpus", "2", "--steps", "1",
              "--warmup", "0")
    assert out.strip() == ""
