"""The JSON line bench.py prints checked on the committed lines: keys, types and the internal arithmetic (value <->
ms_per_step, roofline.frac = achieved / peak, e2e declares its copies).  CPU only: the lines were produced on an H100 by
the commands profiles/README.md lists and live under profiles/."""
import json
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT  # noqa: E402

LINES = ["r02_bench_llama3-8b-fp8_final.jsonl", "r02_bench_mistral-7b-gf4.jsonl", "r02_bench_mixtral-8x7b-fp8.jsonl"]


def _line(name):
    for l in open(os.path.join(ROOT, "profiles", name)):
        if l.startswith("{"):
            return json.loads(l)
    raise AssertionError(name)


@pytest.mark.parametrize("name", LINES)
def test_bench_line_contract(name):
    d = _line(name)
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config",
              "e2e", "gpu_launches", "clocks", "roofline"):
        assert k in d, k
    assert d["unit"] == "tok/s" and d["higher_is_better"] is True and d["data"] == "synthetic" and d["vs_baseline"] is None
    assert d["warmup"] >= 3 and d["gpu_launches"] > d["steps"] * 100
    assert "workload" in d["config"] and "model" not in d["config"]
    tp = d["n_gpus"] > 1 and d["config"]["parallelism"].startswith("tp")
    assert d["scaling"] == ("strong" if tp else "weak")
    n_streams = 1 if (tp or d["n_gpus"] == 1) else d["n_gpus"]
    assert abs(d["value"] - n_streams * 1e3 / d["ms_per_step"]) < 1e-6 * d["value"]
    e = d["e2e"]
    assert e["unit"] == "tok/s" and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 1000 and 0.5 * d["value"] < e["value"] <= 1.02 * d["value"]
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and 0 < r["frac"] < 1.1
    assert "hw_slowdown" not in d["clocks"]["reasons"] and "hw_thermal_slowdown" not in d["clocks"]["reasons"]
    if d["n_gpus"] == 1 and "cpu_baseline" in d:
        c = d["cpu_baseline"]
        assert c["kind"] in ("reference", "port") and c["cores"] >= 1 and c["unit"] == "tok/s"
