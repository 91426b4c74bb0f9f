"""bench.py's JSON contract, checked on CPU against the lines recorded on an H100 (profiles/*_h100.json) and on the helper logic."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (file under profiles/, number of GPUs): the bench lines kept as records; every one of them must carry the contract
RECORDED = [("bench_n1_h100.json", 1)]
REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "clocks"]


def test_recorded_bench_lines_carry_the_contract():
    for name, n in RECORDED:
        d = json.load(open(os.path.join(ROOT, "profiles", name)))
        assert all(k in d for k in REQUIRED), (name, [k for k in REQUIRED if k not in d])
        assert d["metric"] == "wake_h2d_gbs" and d["unit"] == "GB/s" and d["higher_is_better"] is True
        assert d["n_gpus"] == n and d["scaling"] == "weak" and d["vs_baseline"] is None and d["dtype"] == "u8"
        assert "workload" in d["config"] and "model" not in d["config"]
        assert d["warmup"] >= 3 and d["gpu_launches"] > 0 and d["bit_exact"] is True
        e = d["e2e"]
        assert e["unit"] == "GB/s" and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and 0 < e["value"] <= d["value"] * 1.001
        r = d["roofline"]
        assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3 and r["launches"] > 0
        assert d["clocks"]["sm_max_mhz"] and not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


def test_recorded_reference_line():
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_ref_n1_h100.json")))
    assert d["impl"] == "reference" and d["metric"] == "wake_h2d_gbs" and d["n_gpus"] == 1
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_helpers_and_cli_defaults():
    import bench

    assert bench.workload_for(1, None) == "llama-3-8b" and bench.workload_for(8, None) == "llama-3-70b-tp8"
    assert bench.workload_for(4, "mistral-7b") == "mistral-7b"
    peak, src = bench.hbm_peak()
    assert peak > 1000 and ("measured" in src or "fallback" in src)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"], capture_output=True, text=True)
    assert out.returncode == 0 and "--impl" in out.stdout and "--gpus" in out.stdout


def test_recorded_lines_carry_the_contract_and_the_extras():
    """The recorded lines (executor-style phases, median-based value / e2e with the mean beside them, the extras of their N, and the
    card they were measured on)."""
    for name, n in RECORDED:
        d = json.loads(open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()[-1])
        assert all(k in d for k in REQUIRED), (name, [k for k in REQUIRED if k not in d])
        assert d["metric"] == "wake_h2d_gbs" and d["n_gpus"] == n and d["scaling"] == "weak" and d["dtype"] == "u8" and d["bit_exact"] is True
        assert "phases" in d["config"] and "segments_per_rank" in d["config"] and "weights_gib_per_rank" in d["config"]
        assert "median" in d["aggregation"].lower() and d["value_mean"] > 0 and d["e2e"]["mean_gbs"] > 0
        lo, hi = d["wake_latency_s_min_max"]
        assert lo <= d["wake_latency_s"] <= hi and len(d["wake_latency_s_steps"]) == d["steps"]
        assert 0 < d["e2e"]["value"] <= d["value"] * 1.001 and d["e2e"]["h2d_bytes_per_step"] > 0
        assert d["roofline"]["traffic_source"] and abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-3
        assert d["gpu"]["name"] and d["gpu"]["power_limit_w"] > 0
        if n == 1:
            assert d["swap_config4"]["bit_exact"] is True and d["swap_config4"]["cycles"] == 20 and d["swap_config4"]["swap_s_median"] < d["swap_config4"]["serial_sleep_then_wake_s_median"]
            assert d["cpu_baseline"]["kind"] == "reference" and len(d["cpu_baseline"]["value_min_max"]) == 2
            assert d["packed_image"]["bit_exact"] is True and d["packed_image"]["stored_frac"] < 0.76
        else:
            assert d["peer_tier"]["bit_exact"] is True and d["peer_tier"]["wake_latency_s"] < 1.0          # north_star: <= 1.0 s via the peer tier
        if n == 8:
            assert d["e2e"]["value"] >= 410.0 and d["wake_latency_s"] <= 3.0                                 # north_star: >= 80 % of 8 x 64 GB/s, <= 3.0 s
            rr = d["roundrobin_config5"]
            assert rr["bit_exact"] is True and rr["models"] == 4 and rr["frac_of_nvlink"] > 0.7
