"""The numbers DESIGN.md quotes are the ones in the committed evidence file (profiles/h100_bench_n1.json), which records the
GPU they were measured on and carries every key the benchmark line names.  No GPU: this only reads JSON that a GPU run left
behind."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = lambda *a: os.path.join(ROOT, "profiles", *a)


def _fmt(n: float) -> str:
    s = f"{round(n):,}"
    return s.replace(",", " ")


def test_headline_bench_line_is_complete_and_consistent():
    rec = json.load(open(P("h100_bench_n1.json")))
    gpu = rec["gpu"]
    assert "H100" in gpu["name"] and float(gpu["power_limit_w"]) > 0
    d = rec["bench"]
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline", "parity"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["higher_is_better"] is True and "workload" in d["config"]
    r = d["roofline"]
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] < d["value"]
    assert d["gpu_launches"] > 0 and d["parity"]["ok"] is True
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    assert _fmt(d["value"]) in design and _fmt(d["e2e"]["value"]) in design, "DESIGN.md section 6 quotes another run"
    assert f"{r['frac']:.3f}" in design
    assert gpu["name"] in design and f"{float(gpu['power_limit_w']):.0f} W" in design, "DESIGN.md names another GPU"
