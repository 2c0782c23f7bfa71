"""CPU: the bench.py output contract, checked on a committed result line (tests/golden/bench_line_h100_b1.json, produced by
`python bench.py --gpus 1 --steps 2 --warmup 1` on one H100 SXM at a 700 W power limit; the line records warmup 3,
the bench's minimum): every key a consumer of the line
reads is present and typed, the roofline / cpu_baseline / e2e objects are complete, and the derived numbers are
self-consistent."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,n", [("bench_line_h100_b1.json", 1)])
def test_bench_line_contract(name, n):
    d = json.load(open(os.path.join(ROOT, "tests", "golden", name)))
    for k, typ in (("metric", str), ("value", float), ("unit", str), ("n_gpus", int), ("steps", int), ("warmup", int),
                   ("ms_per_step", float), ("higher_is_better", bool), ("scaling", str), ("dtype", str), ("data", str),
                   ("config", dict), ("e2e", dict), ("gpu_launches", int), ("clocks", dict), ("roofline", dict)):
        assert isinstance(d[k], typ), k
    assert d["n_gpus"] == n and d["warmup"] >= 3 and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert d["vs_baseline"] is None  # BASELINE.md holds no published number for this metric
    assert d["dtype"] == "bf16" and d["data"] == "synthetic" and "workload" in d["config"]
    # value = whole-job images / max-over-ranks time
    imgs = d["config"]["global_batch"] * d["steps"]
    assert abs(d["value"] - imgs / (d["ms_per_step"] * d["steps"] * 1e-3)) < 1e-2 * d["value"]
    e = d["e2e"]
    assert set(e) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and e["h2d_bytes_per_step"] > 0
    assert 0 < e["value"] <= d["value"] * 1.02  # end to end includes the copies: not faster than the device-resident number
    assert d["gpu_launches"] > 10000  # 50 steps x ~308 kernels + garment pass, per timed step
    c = d["clocks"]
    assert c["sm_mhz"] and not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    r = d["roofline"]
    assert set(r) >= {"bound", "achieved", "peak", "unit", "frac", "traffic"} and r["bound"] in ("hbm", "tensor")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3
    assert [b["batch_per_gpu"] for b in d["batches"]] == [8, 16, 32]
    kinds = [o["workload"] for o in d["other_configs"]]
    assert kinds == ["ipa_controlnet", "inpaint", "train"] and "error" not in d["other_configs"][2]
    assert d["other_configs"][2]["step_mode"] == "cuda-graph"
    if n == 1:
        cb = d["cpu_baseline"]
        assert set(cb) >= {"value", "unit", "cores", "kind", "sample"} and cb["kind"] in ("port", "reference") and cb["cores"] >= 1
