#!/usr/bin/env python3
"""Mode B (SURVEY.md 8e): ONE BEAGLE instance whose patterns the engine shards over g GPUs of this process (csrc/multi.cu)
-- what an unmodified BEAST run sees when it names the "GPU x N (pattern-sharded)" resource.  Times full evaluations
through the synchronous reference-facing calls (host buffers in, joint log-likelihood out) for g = 1, 2, 4, 8 (as many as
the box has) on one alignment, and checks the value against the single-GPU instance.  Prints one JSON line."""
import ctypes as C
import json, os, statistics, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402

WORKLOAD = os.environ.get("WORKLOAD", "makona_like_1610x6k")
STEPS = int(os.environ.get("STEPS", 300))
import torch
ngpu = torch.cuda.device_count()
lib = beagle.load_library()
res = [r.number for r in beagle.BeagleFactory.getResourceDetails() if "pattern-sharded" in r.name][0]
w, tree, pats, model, site = bench.build_workload(WORKLOAD, 0, {})
scaling = WORKLOAD.startswith("makona")
S, Cc, P = w["states"], site.getCategoryCount(), pats.patternCount
ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=scaling)
out = np.zeros(1)
rows = {}
base = None
for g in (1, 2, 4, 8):
    if g > ngpu:
        break
    devs = (C.c_int * g)(*range(g))
    assert lib.b200SetShardDevices(devs, g) == 0
    inst = bench.create_instance(beagle.BeagleFactory.loadBeagleInstance, ev, S, Cc, P, [res, 0])
    for k in range(10):
        val = bench.issue_sync(inst, ev, k & 1, out)
    per = []
    for k in range(STEPS):
        t0 = time.perf_counter()
        val = bench.issue_sync(inst, ev, k & 1, out)
        per.append(time.perf_counter() - t0)
    inst.finalize()
    if base is None:
        base = val
    rows[str(g)] = {"joint_evals_per_s": 1.0 / statistics.median(per), "ms_per_eval": 1e3 * statistics.median(per),
                    "p10_ms": 1e3 * sorted(per)[len(per) // 10], "p90_ms": 1e3 * sorted(per)[(9 * len(per)) // 10],
                    "logL": float(val), "rel_diff_vs_1gpu": abs(val - base) / abs(base)}
one = rows["1"]["joint_evals_per_s"]
for g, r in rows.items():
    r["speedup_vs_1gpu"] = r["joint_evals_per_s"] / one
    r["efficiency"] = r["speedup_vs_1gpu"] / int(g)
print(json.dumps({"what": "one sharded instance (mode B) over g GPUs of one process, synchronous calls with host buffers; "
                          "median of %d full evaluations" % STEPS, "workload": WORKLOAD, "patterns": P, "taxa": tree.tipCount,
                  "rescaled": scaling, "gpus": rows}))
