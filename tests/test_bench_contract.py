"""bench.py's contract, checked without a GPU: the committed bench lines (profiles/, measured on an H100) carry every key
a reader of the line relies on, and say what they were measured on."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_committed_bench_lines_follow_the_contract():
    ours = json.load(open(os.path.join(ROOT, "profiles", "bench_n1.json")))
    ref = json.load(open(os.path.join(ROOT, "profiles", "bench_reference_n1.json")))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert k in ours, k
    assert ours["config"] == ref["config"] and ref["impl"] == "reference" and ours["metric"] == ref["metric"]
    assert "H100" in ours["clocks"]["gpu"] and ours["clocks"]["power_limit_w"] > 0
    r = ours["roofline"]
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert ours["e2e"]["h2d_bytes_per_step"] > 0 and ours["e2e"]["d2h_bytes_per_step"] > 0 and ours["gpu_launches"] > 0
    assert ours["e2e"]["matches_device_resident_flags"] is True
    assert {"config4_windows", "config5_varlen", "config3_nng_pipeline"} <= set(ours["extra"]["configs"])
    assert ours["cpu_baseline"]["kind"] == "port" and "reference_engine" in ours["cpu_baseline"]
