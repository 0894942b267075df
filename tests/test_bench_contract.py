"""The measurement contract of bench.py, checked without a GPU: the committed bench lines under profiles/ (H100 output of the
current bench.py) carry every key a reader of the line relies on, and the reference arm runs here on the CPU and prints its line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _line(name):
    return json.loads(open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()[-1])


def test_committed_bench_line_has_the_contract_keys():
    d = _line("h100_bench.json")
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
              "config", "gpu", "clocks", "gpu_launches", "e2e", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["unit"] == "pairs/s" and d["n_gpus"] == 1 and d["warmup"] >= 3 and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert d["vs_baseline"] is None and d["data"] == "synthetic" and "workload" in d["config"] and "8192" in d["config"]["workload"]
    assert d["gpu_launches"] > 0 and d["config"]["exactness_errors"] == 0 and "pinned host memory" in d["config"]["value_timing"]
    assert "H100" in d["gpu"]["name"] and d["gpu"]["power_limit_w"] > 0          # the card and its power limit belong to the number
    e = d["e2e"]
    assert e["unit"] == "pairs/s" and 0 < e["value"] < d["value"] and e["h2d_bytes_per_step"] == 100 * 8192 * (128 + 8) and e["d2h_bytes_per_step"] > 0   # uchar staging + positions
    r = d["roofline"]
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and "data sheet" in r["peak_source"]
    flop = d["value"] * r["flop_per_pair"] / 1e12
    assert 0.9 * r["achieved"] < flop <= r["achieved"] * 1.001          # kernel time <= step time
    c = d["cpu_baseline"]
    assert c["kind"] in ("reference", "port") and c["cores"] >= 1 and c["unit"] == "pairs/s" and c["value"] > 0 and c["sample"]
    assert c["cores"] == c["host"]["threads_used"] <= c["host"]["affinity_cpus"]
    assert d["clocks"]["sm_mhz"] and not {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(d["clocks"]["reasons"])
    assert d["cpu_baseline_cascade_hashing"]["value"] > c["value"]
    h = _line("h100_bench_hamming_40img.json")
    assert h["roofline"]["bound"] == "hbm" and h["roofline"]["unit"] == "GB/s" and h["dtype"] == "u32-popcount" and "H100" in h["gpu"]["name"]


def test_real_valued_and_reference_arm_lines():
    """The real-valued line (tensor-core filter + exact re-scoring) and the CPU reference arm on the same host."""
    d = _line("h100_bench.json")
    real = _line("h100_bench_real.json")
    assert real["config"]["real_valued_tensor_core_pairs"] == 4950 and real["config"]["tensor_core_pairs"] == 0 and real["config"]["exactness_errors"] == 0
    assert 0 < real["config"]["fallback_rows_fraction_of_queries"] < 0.01 and real["value"] > 0.5 * d["value"]
    assert real["gpu"] == d["gpu"]
    ref = _line("h100_bench_reference_arm.json")
    assert ref["impl"] == "reference" and "100 synthetic images" in ref["config"]["workload"] and ref["cpu_baseline_cascade_hashing"]["value"] > ref["value"]


def test_reference_arm_runs_on_the_cpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1", "--images", "4",
                        "--features", "256", "--cpu-seconds", "2"], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    assert d["impl"] == "reference" and d["unit"] == "pairs/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"] == {"value": d["value"], "unit": "pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # under torchrun only rank 0 works: the others exit 0 without output
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip() == ""
