"""The committed evidence under profiles/ belongs to the committed sources, and the bench line keeps its contract
(no GPU needed: these read files only)."""
import json
import os
import re

import pytest

from beast_mcmc_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = os.path.join(ROOT, "profiles")


def _line(name):
    path = os.path.join(P, name)
    if not os.path.exists(path):
        pytest.skip(f"{name} not collected yet")
    return json.loads(open(path).read().strip().splitlines()[-1])


def test_sass_excerpts_belong_to_this_tree():
    path = os.path.join(P, "h100_sass_excerpts.txt")
    if not os.path.exists(path):
        pytest.skip("no SASS excerpts collected yet")
    m = re.search(r"library source hash (\w+)", open(path).read())
    assert m, "the excerpt file records the source hash of the library it was taken from"
    assert m.group(1) == build.source_hash()[:len(m.group(1))], "engine sources changed after the evidence was collected: re-run " \
                                                                  "tools/collect_round_evidence.sh + tools/summarise_round_evidence.py"
    text = open(path).read()
    for kernel, mnemonic in (("k_walk4p<4, 4>", "LDGSTS"), ("k_walk_mma<8, 4, false, false, 2>", "DMMA"),
                             ("k_walk_mma<8, 4, false, false, 2>", "UBLKCP")):
        rows = [l for l in text.splitlines() if l.startswith(kernel)]
        assert rows and mnemonic in rows[0], (kernel, mnemonic)


@pytest.mark.parametrize("name", ["h100_bench_cfg2.json", "h100_bench_codon.json", "h100_bench_cfg2_steps20.json"])
def test_bench_line_contract(name):
    d = _line(name)
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "roofline", "e2e", "gpu_launches", "clocks", "repeats", "block_ms_p10", "block_ms_p50",
                "block_ms_p90"):
        assert key in d, key
    assert d["dtype"] == "f64" and d["data"] == "synthetic" and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]
    r = d["roofline"]
    assert r["bound"] == ("fp64" if d["config"]["states"] > 20 else "hbm")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) <= 1e-9 * max(1.0, r["frac"])
    assert d["warmup"] >= 3 and d["repeats"] == d["steps"] >= 20 and d["gpu_launches"] > 0
    assert d["clocks"]["gpu"] and "H100" in d["clocks"]["gpu"] and d["clocks"]["power_limit_w"] > 0
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] == 8 and e["value"] != d["value"]
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    # value = 1 / (median step) up to the max-over-ranks bookkeeping
    assert abs(d["value"] - d["n_gpus"] * 1e3 / d["ms_per_step"]) <= 1e-6 * d["value"]


def test_reference_arm_line_contract():
    d = _line("h100_bench_cfg2_reference.json")
    assert d["impl"] == "reference" and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    g = _line("h100_bench_cfg2.json")
    assert d["metric"] == g["metric"] and d["unit"] == g["unit"] and d["config"]["workload"] == g["config"]["workload"]
