"""The one-line JSON contract of bench.py, checked on lines recorded with this build (tests/golden/bench_*.json: the GPU arm on an H100, the CPU reference arm on 8 host cores): every key a reader of
the line needs is present with the right type, for both arms.  (bench.py itself needs the GPU; this guards the schema on CPU.)"""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(name):
    return json.load(open(os.path.join(ROOT, "tests", "golden", name)))


BASE_KEYS = {"metric": str, "value": (int, float), "unit": str, "n_gpus": int, "steps": int, "warmup": int, "ms_per_step": (int, float),
             "higher_is_better": bool, "scaling": str, "dtype": str, "data": str, "config": dict, "e2e": dict, "gpu_launches": int,
             "cpu_baseline": dict}


def check_base(line):
    for k, t in BASE_KEYS.items():
        assert k in line, k
        assert isinstance(line[k], t), (k, type(line[k]))
    assert "vs_baseline" in line and line["vs_baseline"] is None          # BASELINE.md publishes no number for this metric
    assert "workload" in line["config"] and "model" not in line["config"]
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in line["e2e"], k
    for k in ("value", "unit", "cores", "kind", "sample"):
        assert k in line["cpu_baseline"], k
    assert line["cpu_baseline"]["kind"] in ("port", "reference")


@pytest.mark.parametrize("name", ["bench_h100.json"])
def test_our_arm_line(name):
    line = load(name)
    assert "H100" in line["device"]
    if "react" in line:
        # the reference's own request shapes, the multi-step loop and (N >= 2) the served mix + tensor parallelism are inside the contract
        assert "verbatim" in line["e2e"]["prompts"] and set(line["e2e"]["prompt_tokens_by_kind"]) <= {"analyze", "diagnose", "execute"}
        r = line["react"]
        assert r["conversations_with_final_answer"] == r["conversations"] and 0 < r["prefix_hit_rate"] < 1 and r["react_steps_per_sec"] > 0
        if line["n_gpus"] >= 2:
            assert "configs[2]" in line["config"]["workload"] and set(line["e2e"]["prompt_tokens_by_kind"]) == {"analyze", "diagnose", "execute"}
            assert line["router"]["completed"] == line["router"]["requests"] == line["n_gpus"] * 128
            if "front" in line["router"]:          # the serving block goes through the native front
                assert line["router"]["front"] == "native" and line["router"]["errors"] == [] and line["router"]["rejected_429"] == 0
            tp = line["tp"]
            assert tp["parity"]["ok"] is True and tp["parity"]["t"] == line["n_gpus"] and tp["parity"]["max_dlogit"] < 2.5e-2
            assert tp["t"] == line["n_gpus"] and 0 < tp["roofline_frac_per_gpu"] < 1
    check_base(line)
    assert line["metric"] == "decode_tokens_per_sec" and line["unit"] == "tokens/s" and line["higher_is_better"] is True
    assert line["scaling"] == "weak" and line["dtype"] == "bf16" and line["warmup"] >= 3
    assert line["gpu_launches"] > 0
    assert abs(line["value"] - line["n_gpus"] * line["config"]["batch_per_gpu"] / (line["ms_per_step"] / 1e3)) / line["value"] < 1e-3
    # inputs larger than L2 between timed iterations, stated in config
    assert "l2" in line["config"]
    clk = line["clocks"]
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(clk) and not ({"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(clk["reasons"]))
    e2e = line["e2e"]
    assert e2e["h2d_bytes_per_step"] > 0 and e2e["d2h_bytes_per_step"] > 0 and e2e["value"] < line["value"]     # host copies inside, prefill included
    r = line["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3 and 0 < r["frac"] <= 1.0
    assert r["traffic"] is None or r["traffic"] >= 0.9 * r["algorithmic_bytes_per_launch"]


@pytest.mark.parametrize("ref,ours_name", [("bench_reference_arm.json", "bench_h100.json")])
def test_reference_arm_line(ref, ours_name):
    line = load(ref)
    check_base(line)
    ours = load(ours_name)
    assert line["impl"] == "reference" and line["gpu_launches"] == 0
    for k in ("metric", "unit", "higher_is_better"):
        assert line[k] == ours[k]
    assert line["e2e"] == {"value": line["value"], "unit": line["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["cpu_baseline"]["value"] == line["value"]
