"""The bench.py JSON contract, checked on the committed record of an H100 run (profiles/h100_bench_1gpu.json) and on
the argument parser.  (The bench itself needs a GPU; the CPU reference
arm is exercised by the driver.)"""
import json
import subprocess
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]


def _record():
    name = "h100_bench_1gpu.json"
    return json.loads((REPO / "profiles" / name).read_text()), name


def test_recorded_line_has_every_contract_key():
    d, name = _record()
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "cpu_baseline", "clocks"):
        assert k in d, k
    base = json.loads((REPO / "BASELINE.json").read_text())
    assert "samples/sec" in base["metric"] and d["metric"] == "audio_samples_per_sec" and d["unit"] == "samples/s"
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert d["vs_baseline"] is None and d["data"] == "synthetic" and "workload" in d["config"] and "model" not in d["config"]
    assert abs(d["value"] - 32 * 312 * 256 / (d["ms_per_step"] / 1e3)) / d["value"] < 1e-6
    e = d["e2e"]
    assert e["unit"] == d["unit"] and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] == 32 * 312 * 256 * 4
    assert e["value"] != d["value"]                     # measured separately, through host buffers
    r = d["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert r["traffic"] is None or r["traffic"] > 0
    c = d["cpu_baseline"]
    assert c["kind"] in ("port", "reference") and c["cores"] >= 1 and c["value"] > 0 and c["sample"]
    assert d["gpu_launches"] > 0 and d["gpu_launches"] % d["steps"] == 0     # every step launches the same kernels, all ours
    # the other BASELINE configs and the per-stage rooflines travel in the same line
    assert set(d["sweep"]) >= {"1", "8", "32", "128"} and d["strict_fp32"]["value"] > 0
    assert set(d["configs"]) >= {"c4", "c5"} and d["configs"]["c5"]["padding_frac"] <= 0.08
    assert {"nat_decoder_scan", "hifigan_stage0", "hifigan_stage3", "hifigan_conv_post", "melspec"} <= set(d["roofline_stages"])
    assert d["e2e"]["pageable_result"]["value"] > 0
    assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


def test_bench_cli_flags():
    out = subprocess.run([sys.executable, str(REPO / "bench.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0
    for flag in ("--gpus", "--steps", "--warmup", "--impl"):
        assert flag in out.stdout
