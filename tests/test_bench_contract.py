"""The bench.py JSON contract, checked on the committed lines of the last GPU runs (profiles/r2_bench_*.json): the keys
a reader of the line relies on must be there, with consistent values.  (bench.py itself needs a GPU; this keeps edits
of the emitting code honest on machines without one.)"""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(name):
    path = os.path.join(ROOT, "profiles", name)
    if not os.path.exists(path):
        pytest.skip(f"{name} not committed")
    return json.loads(open(path).read().strip().splitlines()[-1])


@pytest.mark.parametrize("name,n", [("r2_bench_n1.json", 1)])
def test_our_arm_line(name, n):
    d = _line(name)
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "roofline", "gpu_launches", "clocks"):
        assert k in d, k
    assert d["metric"] == "agg_input_rows_per_s" and d["unit"] == "rows/s" and d["n_gpus"] == n
    assert d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["warmup"] >= 3 and d["gpu_launches"] > 0 and "workload" in d["config"] and "model" not in d["config"]
    assert "H100" in d["gpu"]["name"] and d["gpu"]["power_limit_w"] > 0   # what the numbers were measured on
    assert len(d["ms_steps"]) == d["steps"]
    # value = whole-job rows / time of the K-step region
    rows = d["config"]["rows_per_gpu"] * n
    assert abs(d["value"] - rows / (d["ms_per_step"] / 1e3)) / d["value"] < 1e-6
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert 0.0 < r["frac"] < 1.0
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    if "e2e" in d:
        e = d["e2e"]
        assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] < d["value"]
    if n == 1:
        c = d["cpu_baseline"]
        for k in ("value", "unit", "cores", "kind", "sample", "parity"):
            assert k in c, k
        assert c["kind"] == "reference" and c["cores"] >= 1
        assert all(v.startswith("bit-exact") for v in c["parity"].values()), c["parity"]
        assert d["e2e_duckdb"]["q1"]["same_result"] and d["e2e_duckdb"]["q14"]["same_result"]
    else:
        # both shuffle plans and the broadcast plan are reported at every N > 1
        for k in ("join_probe", "join_probe_shuffle", "join_probe_shuffle_pipelined"):
            assert d[k]["n_gpus"] == n and d[k]["value"] > 0
        assert d["join_probe_shuffle"]["nvlink_bytes_per_step_per_gpu"] > 0


def test_reference_arm_line():
    d = _line("r2_bench_reference_n1.json")
    assert d["impl"] == "reference" and d["metric"] == "agg_input_rows_per_s" and d["unit"] == "rows/s"
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] >= 1
    assert d["cpu_baseline"]["value"] == d["value"] == d["e2e"]["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["steps"] >= 1 and d["config"]["rows"] > 0
