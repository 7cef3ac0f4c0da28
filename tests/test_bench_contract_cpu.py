"""CPU: the committed bench lines (profiles/h100_bench_*.json, produced by `python bench.py --workload W` on an H100) carry every key
of the bench contract, with consistent values - a schema guard for bench.py's output, not a measurement."""
import json
from pathlib import Path

import pytest

PROFILES = Path(__file__).resolve().parent.parent / "profiles"
WORKLOADS = ["vga_lightglue", "mp1_lightglue", "seq_superglue", "superpoint_only", "small_stop"]


@pytest.mark.parametrize("w", WORKLOADS)
def test_line_has_the_contract_keys(w):
    d = json.loads((PROFILES / f"h100_bench_{w}.json").read_text())
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None and d["warmup"] >= 3
    assert d["value"] > 0 and d["gpu_launches"] > 0 and d["data"] == "synthetic" and "workload" in d["config"]
    e = d["e2e"]
    assert e["value"] > 0 and e["unit"] == d["unit"] and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
    assert e["value"] <= d["value"] * 1.02  # host buffers and copies cannot beat the device-resident path
    r = d["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert 0 < r["frac"] < 0.4 and "traffic" in r
    c = d["cpu_baseline"]
    assert c["kind"] in ("reference", "port") and c["value"] > 0 and c["cores"] >= 1 and c["unit"] == d["unit"] and c["sample"]
    assert d["value"] / c["value"] > 50  # north_star: >= 50x the reference's CPU path on one GPU
    k = d["clocks"]
    assert not {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(k["reasons"])


def test_default_line_is_the_dominant_kernel_story():
    d = json.loads((PROFILES / "h100_bench_vga_lightglue.json").read_text())
    r = d["roofline"]
    assert r["kernel"].startswith("k_flash") and "traffic" in r and 0.5 < r["kernel_share_of_step"] < 0.65
    fam = d["extra"]["kernel_family_ms_per_step"]
    assert fam["k_gemm_ws"]["ms_per_step"] < r["kernel_ms_per_step"]  # attention, not the linears, dominates the step
    assert d["e2e"]["host_threads"] >= 1 and d["e2e"]["single_thread"] <= d["e2e"]["value"] * 1.05
