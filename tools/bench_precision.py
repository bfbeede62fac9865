"""Double against single (PRECISION_SINGLE: fp32 partials storage, fp64 arithmetic) on one GPU, same process, alternating.

For every workload: a double and a single instance of the same evaluation, timed in blocks of --steps steps with bench.py's
pattern (resident eigen system, buffers flipping like BEAST's, a CUDA event between consecutive steps).  The blocks run in
ABBA order (double, single, single, double, ...), so drift over the run falls on both arms alike.  Per arm: the p10 / p50 /
p90 step of every block and, as the arm's figures, the median over its blocks of each of the three; the partials-kernel time
per step (b200SetKernelTiming, the mean of two runs per arm, also ABBA); the algorithmic bytes per step at that element size.  Each arm first evaluates the
workload as bench.py does (unscaled unless the workload is a rescaled one); an arm that underflows there (-inf or NaN) runs
rescaled, as BEAST does after its first underflow, and the line says which arm did.  The other arm keeps its own scaling:
a double run that does not underflow is timed unscaled, as a -beagle_double user runs it.  Also the largest per-site
difference between the two arms next to the bound 1.001 n u + 1e-9 (n = internal nodes, u = 2^-24).  Prints ONE JSON line.

    python tools/bench_precision.py --steps 200 --warmup 20 --blocks 4
"""
import argparse
import ctypes as Cc
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402

WORKLOADS = ("gtr_g4_1000x10k", "gtr_g4_1000x10k_rescaled", "makona_like_1610x6k", "hky_1441x593", "benchmark2_xml")
U = 2.0 ** -24


class _Local:
    """the single-process subset of bench.Dist that bench.timed_blocks uses"""

    def __init__(self, torch):
        self.torch, self.device = torch, torch.device("cuda:0")

    def bracket(self):
        self.torch.cuda.synchronize()

    def max_over_ranks(self, values):
        return list(values)


def algorithmic_bytes(ev, S, C, P, elem):
    """bench.Evaluation.algorithmic with the partials at `elem` bytes per value (matrices stay fp64)"""
    pp, sp, ss = ev.mix["pp"], ev.mix["sp"], ev.mix["ss"]
    mats = 2 * C * S * S * 8
    return pp * (3 * C * P * S * elem + mats) + sp * (2 * C * P * S * elem + 4 * P + mats) + ss * (C * P * S * elem + 8 * P + mats)


def create(ev, S, C, P, pref):
    N, n = ev.N, ev.n
    inst = beagle.BeagleJNIImpl(N, 2 * (n - N) + N, N, S, P, 2, 2 * n, C, 2 * (n - N + 1), [1, 0], pref, 0)
    for t in range(N):
        inst.setTipStates(t, np.ascontiguousarray(ev.pats.states[t], dtype=np.int32))
    inst.setPatternWeights(np.ascontiguousarray(ev.pats.weights))
    return inst


class Arm:
    def __init__(self, D, lib, ev, S, C, P, pref):
        self.D, self.lib, self.ev, self.S, self.C, self.P = D, lib, ev, S, C, P
        self.inst = create(ev, S, C, P, pref)
        self.out = np.zeros(1)
        self.first = float(bench.issue_sync(self.inst, ev, 0, self.out))
        devp, strm = Cc.c_void_p(), Cc.c_void_p()
        rc = lib.b200RootLogLikelihoodDevice(self.inst.instance, ev.rootIdx[0], 0, 0, ev.cumIdx[0] if ev.scaling else -1,
                                             Cc.byref(devp), Cc.byref(strm))
        assert rc == 0
        self.stream = bench.external_stream(D, strm)
        self.p50, self.p10, self.p90 = [], [], []

    def step(self, k):
        ev, inst, p = self.ev, self.inst, k & 1
        inst.updateTransitionMatrices(0, ev.probIdx[p], None, None, ev.lengths, len(ev.lengths))
        inst.updatePartials(ev.ops[p], len(ev.nodeOps), -1)
        cum = -1
        if ev.scaling:
            inst.resetScaleFactors(ev.cumIdx[p])
            inst.accumulateScaleFactors(ev.scaleIdx[p], len(ev.nodeOps), ev.cumIdx[p])
            cum = ev.cumIdx[p]
        self.lib.b200RootLogLikelihoodDevice(inst.instance, ev.rootIdx[p], 0, 0, cum, None, None)

    def block(self, steps, warmup):
        r = bench.timed_blocks(self.D, self.stream, self.step, steps, warmup)
        self.p10.append(r["block_ms_p10"]); self.p50.append(r["block_ms_p50"]); self.p90.append(r["block_ms_p90"])

    def partials_ms(self, steps):
        self.D.bracket()
        self.inst.setKernelTiming(True)
        for k in range(steps):
            self.step(k)
        self.D.bracket()
        ms, launches = self.inst.getKernelTiming(0)
        self.inst.setKernelTiming(False)
        return ms / steps, launches / steps

    def sites(self):
        bench.issue_sync(self.inst, self.ev, 0, self.out)
        s = np.zeros(self.P)
        self.inst.getSiteLogLikelihoods(s)
        return s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = [x.strip() for x in q.split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=4, help="timed blocks per arm, in ABBA order")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision: no CUDA device")
    D = _Local(torch)
    lib = beagle.load_library()
    name, limit = card()
    rows = []
    for wname in args.workloads.split(","):
        w, tree, pats, model, site = bench.build_workload(wname, 0, {})
        S, C, P = w["states"], site.getCategoryCount(), pats.patternCount
        scaled = bool(w.get("scaling"))
        ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=scaled)
        arms, underflowed = {}, {}
        for a, pref in (("double", 0), ("single", beagle.BeagleFlag.PRECISION_SINGLE)):
            arm = Arm(D, lib, ev, S, C, P, pref)
            assert bool(arm.inst.getDetails().flags & beagle.BeagleFlag.PRECISION_SINGLE) == (a == "single")
            underflowed[a] = not np.isfinite(arm.first)
            if underflowed[a] and not scaled:          # what BEAST does after the first underflow: evaluate rescaled
                arm.inst.finalize()
                arm = Arm(D, lib, bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=True),
                          S, C, P, pref)
            arms[a] = arm
        double, single = arms["double"], arms["single"]
        for b in range(args.blocks):                   # ABBA
            for arm in ((double, single) if b % 2 == 0 else (single, double)):
                arm.block(args.steps, args.warmup)
        ks = {"double": [], "single": []}
        for a, arm in (("double", double), ("single", single), ("single", single), ("double", double)):     # ABBA
            ks[a].append(arm.partials_ms(args.steps))
        ks = {a: tuple(float(np.mean(v)) for v in zip(*m)) for a, m in ks.items()}
        sd, ss = double.sites(), single.sites()
        n = tree.nodeCount - tree.tipCount
        row = {"workload": wname, "taxa": tree.tipCount, "patterns": P, "categories": C, "workload_rescaled": scaled,
               "max_site_diff": float(np.max(np.abs(ss - sd))), "site_bound": 1.001 * n * U + 1e-9,
               "joint_double": float(np.sum(pats.weights * sd)), "joint_single": float(np.sum(pats.weights * ss))}
        for a, arm, elem in (("double", double, 8), ("single", single, 4)):
            row[a] = {"unscaled_underflowed": bool(underflowed[a] and not scaled), "rescaled": bool(arm.ev.scaling),
                      "step_ms_p50": float(np.median(arm.p50)), "step_ms_p10": float(np.median(arm.p10)),
                      "step_ms_p90": float(np.median(arm.p90)), "block_p50s": [float(x) for x in arm.p50],
                      "partials_kernel_ms_per_step": ks[a][0], "partials_launches_per_step": ks[a][1],
                      "algorithmic_bytes_per_step": algorithmic_bytes(arm.ev, S, C, P, elem)}
        row["single_over_double_step"] = row["single"]["step_ms_p50"] / row["double"]["step_ms_p50"]
        rows.append(row)
        double.inst.finalize()
        single.inst.finalize()
    print(json.dumps({"tool": "bench_precision", "card": name, "power_limit": limit, "steps": args.steps,
                      "warmup": args.warmup, "blocks_per_arm": args.blocks, "workloads": rows}))


if __name__ == "__main__":
    main()
