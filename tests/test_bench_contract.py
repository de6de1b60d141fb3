"""bench.py's output contract: the committed line (profiles/bench_h100_bf16.json, produced on an H100 by the default
`python bench.py`) and the live `--impl reference` line carry every key a consumer of the line reads, with consistent values."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config"]


def _check_common(line):
    for k in BASE_KEYS:
        assert k in line, k
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert "reasoning" in line["metric"] and "reasoning steps/sec" in base["metric"]
    assert line["higher_is_better"] is True and line["scaling"] == "weak" and line["data"] == "synthetic"
    assert line["vs_baseline"] is None                       # BASELINE.json publishes no number for this metric
    assert "workload" in line["config"] and "model" not in line["config"]
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in line["e2e"], k
    for k in ("value", "unit", "cores", "kind", "sample"):
        assert k in line["cpu_baseline"], k
    assert line["cpu_baseline"]["kind"] in ("reference", "port")


def test_committed_gpu_line_has_the_full_contract():
    line = json.load(open(os.path.join(ROOT, "profiles", "bench_h100_bf16.json")))
    _check_common(line)
    assert line["n_gpus"] == 1 and line["dtype"] == "bf16" and line["warmup"] >= 3
    L = 12
    assert abs(line["value"] - line["steps"] * L / (line["ms_per_step"] * 1e-3 * line["steps"])) < 1e-6 * line["value"]
    assert line["gpu_launches"] > 0
    assert line["e2e"]["h2d_bytes_per_step"] > 0 and line["e2e"]["d2h_bytes_per_step"] > 0
    assert line["e2e"]["value"] < line["value"]              # the copies are inside the timed region
    for k in ("sm_mhz", "sm_max_mhz", "reasons"):
        assert k in line["clocks"], k
    assert not set(line["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    for roof in (line["roofline"], line["roofline_kb_attend"]):
        for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
            assert k in roof, k
        assert roof["bound"] in ("hbm", "tensor") and abs(roof["frac"] - roof["achieved"] / roof["peak"]) < 1e-9
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else None
    if peaks:
        assert line["roofline_kb_attend"]["peak"] == peaks["hbm_gbs"]


def test_reference_arm_line_live():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-500:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    _check_common(line)
    assert line["impl"] == "reference" and line["dtype"] == "f32"
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    assert line["e2e"]["value"] == line["value"] == line["cpu_baseline"]["value"]
    assert line["cpu_baseline"]["cores"] >= 1
