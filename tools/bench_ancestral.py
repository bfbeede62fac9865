"""One joint ancestral-state sample per pattern: the device route (b200SampleAncestralStates) against the host route that
AncestralStateBeagleTreeLikelihood takes (getPartials on every internal node, getTransitionMatrix on every branch, then the
per-row draws on the host -- here vectorised numpy, which is faster than the Java loop it stands for).

Per workload: the instance is evaluated once as bench.py does (rescaled if the unscaled evaluation underflows); then
--reps device samples and --host-reps host samples are timed with a host clock around calls that end in a device
synchronise (the device call returns after its outputs have landed in host memory).  Also the bytes each route moves over
the bus.  Prints ONE JSON line with the card's name and power limit.

    python tools/bench_ancestral.py --reps 20 --host-reps 2
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402

WORKLOADS = ("gtr_g4_1000x10k", "makona_like_1610x6k")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return name, limit


def preorder_rows(tree):
    """(node buffer, parent row, matrix buffer) in pre-order at buffer parity 0 (buffer = matrix = node index)"""
    rows, stack = [], [(tree.root, -1)]
    while stack:
        node, parent = stack.pop()
        rows.append((node, parent, node))
        for k in tree.child[node]:
            if k >= 0:
                stack.append((int(k), len(rows) - 1))
    return [np.array([r[k] for r in rows], dtype=np.int32) for k in range(3)]


def host_route(inst, ev, rows, S, C, P, rng):
    """getPartials / getTransitionMatrix for everything, then one inverse-CDF draw per (row, pattern) in numpy"""
    nb, pr, mi = rows
    N = ev.N
    part = np.zeros(C * P * S)
    partials = {}
    for b in nb:
        if b >= N:
            inst.getPartials(int(b), -1, part)
            partials[int(b)] = part.reshape(C, P, S).copy()
    mats, m = {}, np.zeros(C * S * S)
    for r in range(1, len(nb)):
        inst.getTransitionMatrix(int(mi[r]), m)
        mats[int(mi[r])] = m.reshape(C, S, S).copy()
    w = ev.site.getCategoryProportions()[:, None, None] * ev.model.getFrequencies()[None, None, :]
    joint = (w * partials[int(nb[0])]).transpose(1, 0, 2).reshape(P, C * S)
    cum = np.cumsum(joint, axis=1)
    q = (cum < rng.random(P)[:, None] * cum[:, -1:]).sum(axis=1)
    cats, states = q // S, np.zeros((len(nb), P), dtype=np.int64)
    states[0] = q % S
    cols = np.arange(P)
    for r in range(1, len(nb)):
        b = int(nb[r])
        wts = mats[int(mi[r])][cats, states[pr[r]], :]                         # [P][S]: P_c[i][.]
        if b >= N:
            wts = wts * partials[b][cats, cols, :]
        else:
            obs = ev.pats.states[b]
            wts = np.where((obs[:, None] >= S) | (obs[:, None] == np.arange(S)[None, :]), wts, 0.0)
        cum = np.cumsum(wts, axis=1)
        states[r] = np.minimum((cum < rng.random(P)[:, None] * cum[:, -1:]).sum(axis=1), S - 1)
    return states, cats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ancestral: no CUDA device")
    name, limit = card()
    out = []
    for wname in args.workloads.split(","):
        w, tree, pats, model, site = bench.build_workload(wname, 0, {})
        S, C, P = w["states"], site.getCategoryCount(), pats.patternCount
        ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=bool(w.get("scaling")))
        inst = bench.create_instance(beagle.BeagleFactory.loadBeagleInstance, ev, S, C, P, [1, 0])
        logL = float(bench.issue_sync(inst, ev, 0, np.zeros(1)))
        if not np.isfinite(logL):                      # as BEAST after its first underflow: evaluate rescaled
            inst.finalize()
            ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=True)
            inst = bench.create_instance(beagle.BeagleFactory.loadBeagleInstance, ev, S, C, P, [1, 0])
            logL = float(bench.issue_sync(inst, ev, 0, np.zeros(1)))
        rows = preorder_rows(tree)
        sample = lambda k: inst.sampleAncestralStates(*rows, ev.rootIdx[0], 0, 0, 2024, k)
        for k in range(3):                             # warm-up: module load, scratch allocation
            sample(k)
        dev = []
        for k in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sample(100 + k)
            dev.append(1e3 * (time.perf_counter() - t0))
        host_route(inst, ev, rows, S, C, P, np.random.default_rng(0))          # warm-up
        host = []
        for k in range(args.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            host_route(inst, ev, rows, S, C, P, np.random.default_rng(k))
            host.append(1e3 * (time.perf_counter() - t0))
        R, internal = len(rows[0]), tree.nodeCount - tree.tipCount
        out.append({"workload": wname, "taxa": tree.tipCount, "patterns": P, "categories": C, "rows": R,
                    "rescaled": bool(ev.scaling), "logL": logL,
                    "device_ms_p50": float(np.median(dev)), "device_ms_min": float(np.min(dev)),
                    "host_route_ms_p50": float(np.median(host)),
                    "host_over_device": float(np.median(host) / np.median(dev)),
                    "device_bus_bytes": int(16 * R + 4 * (R + 1) * P),
                    "host_route_bus_bytes": int(internal * C * P * S * 8 + (R - 1) * C * S * S * 8)})
        inst.finalize()
    print(json.dumps({"tool": "bench_ancestral", "card": name, "power_limit": limit, "reps": args.reps,
                      "host_reps": args.host_reps, "workloads": out}))


if __name__ == "__main__":
    main()
