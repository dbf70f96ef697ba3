"""The JSON lines bench.py printed on the H100 (committed under profiles/) carry every key the measurement contract
names, with consistent values — a schema regression in bench.py shows up here before a GPU visit is spent on it."""
import glob
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(name):
    return json.loads(open(os.path.join(ROOT, "profiles", name)).read().strip().splitlines()[-1])


@pytest.mark.parametrize("name", ["h100_bench.json", "h100_bench_sdxl.json"])
def test_gpu_arm_line(name):
    d = _line(name)
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "clocks", "gpu_launches", "roofline"):
        assert k in d, (name, k)
    assert d["unit"] == "images/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["warmup"] >= 3 and d["steps"] >= 1 and d["gpu_launches"] > 0 and "synthetic" in d["data"]
    assert "workload" in d["config"] and "model" not in d["config"]
    # value = images of the whole job / device time of the timed region
    images = d["config"]["global_batch"] * d["steps"]
    assert abs(d["value"] - images / (d["ms_per_step"] * d["steps"] / 1e3)) <= 1e-6 * d["value"]
    r = d["roofline"]
    assert r["bound"] in ("tensor", "hbm") and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and 0 < r["frac"] < 1
    assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    if d.get("e2e"):     # None in the --no-e2e experiment lines
        e = d["e2e"]
        assert e["unit"] == d["unit"] and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
        assert 0.5 * d["value"] < e["value"] <= 1.02 * d["value"]
    if d.get("cpu_baseline"):
        c = d["cpu_baseline"]
        assert c["kind"] in ("port", "reference") and c["cores"] >= 1 and c["unit"] == d["unit"] and c["sample"]


def test_bench_defaults_and_flags():
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    src = open(spec.origin).read()
    for flag in ("--gpus", "--steps", "--warmup", "--impl"):
        assert f'"{flag}"' in src
    assert 'ap.add_argument("--gpus", type=int, default=1)' in src and 'ap.add_argument("--warmup", type=int, default=3)' in src
    # the product arm must not reach into oracle/ outside the declared legs
    import re
    uses = [m.start() for m in re.finditer(r"from oracle|import oracle|sd_oracle", src)]
    assert uses, "bench.py's cpu_baseline / reference / stock legs use the oracle"


def test_every_profile_json_parses():
    for f in glob.glob(os.path.join(ROOT, "profiles", "*.json")):
        txt = open(f).read().strip()
        try:
            json.loads(txt)
        except json.JSONDecodeError:
            for line in txt.splitlines():
                if line.strip().startswith("{"):
                    json.loads(line)
