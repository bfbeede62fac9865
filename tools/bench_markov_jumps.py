"""Markov-jump counts conditioned on one joint ancestral sample: the device route (b200SampleMarkovJumps) against the sampler
alone (b200SampleAncestralStates) and against the host route MarkovJumpsBeagleTreeLikelihood takes (getPartials on every
internal node, getTransitionMatrix on every branch, the draws on the host, then the conditional matrices and one lookup per
(branch, pattern) -- here vectorised numpy, faster than the Java loop it stands for).

Workloads: gtr_g4_1000x10k with the all-changes register (and a reward register as the second), codon_mg94_500x5k with the
synonymous and non-synonymous registers, and a discrete-trait shape (12 states, one category, one pattern, 200 tips) built
from a seed here.  Every call is timed with a host clock around calls that end in a device synchronise (a device call
returns after its outputs have landed in host memory): the sampler alone, the jumps call with 1 and 2 registers, with and
without the states copied back.  --profile instead runs a few jumps calls under torch.profiler and reports the device time
of each kernel, which splits the conditional-matrix kernel from the sampling walk.  Prints ONE JSON line with the card's
name and power limit.

    python tools/bench_markov_jumps.py --reps 20 --host-reps 2
    python tools/bench_markov_jumps.py --profile
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_ancestral import card, host_route, preorder_rows  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402
from harness import evomodel as em  # noqa: E402
from oracle import markov_jumps as mj  # noqa: E402

WORKLOADS = ("gtr_g4_1000x10k", "codon_mg94_500x5k", "discrete_trait_200x1")


def build(name):
    if name == "discrete_trait_200x1":
        rng = np.random.default_rng(12)
        tree = em.Tree.coalescent(200, 0.5, 12)
        model = em.SubstitutionModel(rng.uniform(0.2, 3.0, 66), rng.dirichlet(np.full(12, 5.0)))
        site = em.GammaSiteRateModel()
        return 12, tree, em.synthetic_patterns(tree, model, site, 1, seed=12), model, site, False
    w, tree, pats, model, site = bench.build_workload(name, 0, {})
    return w["states"], tree, pats, model, site, bool(w.get("scaling"))


def registers(name, model):
    Q = model.infinitesimalMatrix()
    changes = Q - np.diag(np.diag(Q))
    if name.startswith("codon"):
        aa = [em._AA[c] for c in em.SENSE_CODONS]
        syn = np.array([[a == b for b in aa] for a in aa])
        return np.stack([np.where(syn, changes, 0.0), np.where(~syn, changes, 0.0)])
    return np.stack([changes, np.diag((np.arange(Q.shape[0]) == 0).astype(np.float64))])


def host_jumps(inst, ev, rows, lengths, regs, S, C, P, rng):
    """the host route: the draws (bench_ancestral.host_route), then N per (branch, category, register) and the lookups"""
    states, cats = host_route(inst, ev, rows, S, C, P, rng)
    nb, pr, _ = rows
    eig, rates = ev.eig, ev.site.getCategoryRates()
    branch, pattern = np.zeros((len(regs), len(nb))), np.zeros((len(regs), P))
    for r in range(1, len(nb)):
        for c in range(C):
            sel = cats == c
            for g, M in enumerate(regs):
                N = mj.conditional(eig.Evec, eig.Ievc, eig.Eval, M, rates[c] * lengths[r])[0]
                v = N[states[pr[r], sel], states[r, sel]]
                pattern[g, sel] += v
                branch[g, r] += v @ ev.pats.weights[sel]
    return branch, pattern


def timed(fn, reps, torch):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        out.append(1e3 * (time.perf_counter() - t0))
    return {"p50": float(np.median(out)), "min": float(np.min(out))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_markov_jumps: no CUDA device")
    name, limit = card()
    out = []
    for wname in args.workloads.split(","):
        S, tree, pats, model, site, scaling = build(wname)
        C, P = site.getCategoryCount(), pats.patternCount
        ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=scaling)
        inst = bench.create_instance(beagle.BeagleFactory.loadBeagleInstance, ev, S, C, P, [1, 0])
        logL = float(bench.issue_sync(inst, ev, 0, np.zeros(1)))
        if not np.isfinite(logL):                      # as BEAST after its first underflow: evaluate rescaled
            inst.finalize()
            ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=True)
            inst = bench.create_instance(beagle.BeagleFactory.loadBeagleInstance, ev, S, C, P, [1, 0])
            logL = float(bench.issue_sync(inst, ev, 0, np.zeros(1)))
        rows = preorder_rows(tree)
        byNode = np.zeros(tree.nodeCount)
        byNode[ev.branchNodes] = ev.lengths
        lengths = byNode[rows[0]]
        regs = registers(wname, model)
        root = ev.rootIdx[0]
        sample = lambda k: inst.sampleAncestralStates(*rows, root, 0, 0, 2024, k)
        jumps = lambda G, withStates, k=0: inst.sampleMarkovJumps(*rows, lengths, root, 0, 0, 0, 0, regs[:G], 2024, k,
                                                                   states=withStates, categories=withStates)
        for k in range(3):                             # warm-up: module load, scratch allocation at its largest
            sample(k)
            jumps(2, True, k)
        # the device route must draw what the sampler draws
        assert np.array_equal(jumps(2, True, 7)[0], sample(7)[0])
        rec = {"workload": wname, "taxa": tree.tipCount, "patterns": P, "states": S, "categories": C, "rows": len(rows[0]),
               "rescaled": bool(ev.scaling), "logL": logL}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                for k in range(5):
                    jumps(2, False, k)
            kern = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.key.startswith(("k_", "void", "b200")):
                    kern[e.key] = {"calls": e.count, "device_ms_total": e.device_time_total / 1e3}
            rec["profile_5_calls_2_registers"] = kern
        else:
            rec["sampler_ms"] = timed(lambda: sample(11), args.reps, torch)
            for G in (1, 2):
                rec[f"jumps_{G}reg_ms"] = timed(lambda: jumps(G, True), args.reps, torch)
                rec[f"jumps_{G}reg_counts_only_ms"] = timed(lambda: jumps(G, False), args.reps, torch)
            host_jumps(inst, ev, rows, lengths, regs, S, C, P, np.random.default_rng(0))        # warm-up
            rec["host_route_2reg_ms"] = timed(lambda: host_jumps(inst, ev, rows, lengths, regs, S, C, P,
                                                                 np.random.default_rng(1)), args.host_reps, torch)
            rec["host_over_device_2reg"] = rec["host_route_2reg_ms"]["p50"] / rec["jumps_2reg_ms"]["p50"]
        out.append(rec)
        inst.finalize()
    print(json.dumps({"tool": "bench_markov_jumps", "card": name, "power_limit": limit, "reps": args.reps,
                      "host_reps": args.host_reps, "profile": args.profile, "workloads": out}))


if __name__ == "__main__":
    main()
