"""The bench line's contract (driver-facing): the committed measurement of this tree (profiles/bench_h100.json,
written by `python bench.py --gpus 1` on an H100) carries every key the contract names, with sane types and
internally consistent numbers.  Guards the output format against accidental edits to bench.py."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(name):
    with open(os.path.join(ROOT, "profiles", name)) as f:
        lines = [l for l in f.read().splitlines() if l.startswith("{")]
    assert len(lines) == 1, "exactly ONE JSON line"
    return json.loads(lines[0])


@pytest.mark.parametrize("name,n", [("bench_h100.json", 1)])
def test_contract_keys(name, n):
    d = load(name)
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "clocks", "gpu_launches"):
        assert k in d, k
    assert d["n_gpus"] == n and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert d["vs_baseline"] is None                      # BASELINE.md publishes no number for this metric
    assert d["dtype"] == "u8" and d["data"] == "synthetic" and d["warmup"] >= 3
    assert "workload" in d["config"] and "model" not in d["config"]
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and r["unit"] == "GB/s"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(r["achieved"] - r["algorithmic_bytes_per_launch"] / (r["launch_ms"] * 1e-3) / 1e9) < 1e-6 * r["achieved"]
    c = d["cpu_baseline"]
    assert c["kind"] in ("reference", "port") and c["cores"] >= 1 and c["value"] > 0 and c["sample"]
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
    assert e["value"] < d["value"]                       # PCIe inside the timed region cannot beat resident inputs
    assert d["gpu_launches"] > 0
    cl = d["clocks"]
    assert not set(cl["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    # value = units of all ranks / max-over-ranks time
    cfg = d["config"]
    units = n * cfg["frames_per_gpu"] * cfg["blocks_per_frame"] * (
        cfg["legs"]["sad_candidates_per_block"] + cfg["legs"]["satd_candidates_per_block"] + 1)
    assert abs(d["value"] - units / (d["ms_per_step"] * 1e-3)) < 1e-6 * d["value"]


@pytest.mark.parametrize("name,n", [("bench_h100.json", 1)])
def test_strong_scaling_object(name, n):
    """auto mode carries the 4K tile workload (BASELINE configs[4]) beside the headline: whole-job units over
    the max-over-ranks step time, total work independent of N"""
    t = load(name)["strong_scaling_4k_tiles"]
    assert t["scaling"] == "strong" and t["n_gpus"] == n and t["tiles"] == 8
    units = t["frame_pairs"] * t["blocks_per_frame"] * (64 + 8 + 1)
    assert abs(t["value"] - units / (t["ms_per_step"] * 1e-3)) < 1e-6 * t["value"]
    assert set(t["per_rank_leg_ms"]) == {"sad_cand", "satd_cand", "residual+fwd_txfm", "cdef_find_dir", "cdef_filter"}

