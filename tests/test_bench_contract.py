"""The committed bench line (profiles/) keeps bench.py's JSON contract: a change to bench.py that drops a key shows here
without a GPU."""
import glob
import json
import os

import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
LINES = sorted(glob.glob(os.path.join(ROOT, "profiles", "r*_bench_n*_*_*.json")))


@pytest.mark.parametrize("path", LINES, ids=[os.path.basename(p) for p in LINES])
def test_bench_line_contract(path):
    d = json.loads(open(path).read().strip().splitlines()[-1])
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    # BASELINE.json: "voxels/s full-texture voxel-based on 256^3 @1/2/4/8 H100; %HBM roofline" -- the line carries the
    # quantity, the "@N H100" part is n_gpus and the roofline part is the `roofline` object
    assert base["metric"].startswith(d["metric"])
    assert d["unit"] == "voxels/s" and d["higher_is_better"] is True and d["data"] == "synthetic"
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["steps"] >= 1 and d["warmup"] >= 3
    assert d["scaling"] in ("weak", "strong") and d["dtype"] == "f64" and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    assert d["gpu_launches"] > 0
    c = d["clocks"]
    assert c["sm_mhz"] and c["sm_max_mhz"] and not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] != d["value"]
    r = d["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s")
    assert r["frac"] == pytest.approx(r["achieved"] / r["peak"])
    if d["n_gpus"] == 1 and d.get("cpu_baseline"):
        b = d["cpu_baseline"]
        assert b["kind"] in ("reference", "port") and b["cores"] >= 1 and b["value"] > 0 and b["sample"]


def test_at_least_one_line_is_committed():
    assert LINES
