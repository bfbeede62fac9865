"""Complete substitution histories by uniformization conditioned on one joint ancestral sample: the device route
(b200SampleSubstitutionHistories) against the sampler alone (b200SampleAncestralStates) and against the host route
(getPartials on every internal node, getTransitionMatrix on every branch, the draws on the host, then one uniformized
history per (branch, pattern) -- here the numpy restatement oracle/uniformization.py, one Python loop per pair).

Workloads: gtr_g4_1000x10k with the all-changes and a reward register, codon_mg94_500x5k with the synonymous and
non-synonymous registers, and the discrete-trait shape (12 states, one category, one pattern, 200 tips) with a seeded
non-reversible generator (its partials come from a reversible model of the same size: the shape, not the posterior, sets
the cost).  Device calls are timed with a host clock around calls that end in a device synchronise: the sampler alone, the
histories with registers and jump counts only, and with the events too (the sizing call and the full call).  The host route
runs in full on the trait shape; on the large workloads its history draws run on the first --host-pairs (row, pattern)
pairs, and the record gives the measured time of those pairs, the per-pair rate and the full-workload time extrapolated
from that rate (marked as such).  --profile instead runs a few calls under torch.profiler and reports each kernel's device
time.  Prints ONE JSON line with the card's name and power limit.

    python tools/bench_substitution_histories.py --reps 10 --host-reps 1
    python tools/bench_substitution_histories.py --profile
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
from bench_markov_jumps import build, registers  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402
from oracle import uniformization as un  # noqa: E402

WORKLOADS = ("gtr_g4_1000x10k", "codon_mg94_500x5k", "discrete_trait_200x1")


def generator(name, model):
    if name == "discrete_trait_200x1":
        rng = np.random.default_rng(3)
        off = rng.uniform(0.0, 1.0, (12, 12)) * (rng.random((12, 12)) < 0.6)
        np.fill_diagonal(off, 0.0)
        return off - np.diag(off.sum(axis=1))
    return model.infinitesimalMatrix()


def host_histories(inst, ev, rows, lengths, Q, regs, S, C, P, rng, pairs):
    """the host route on the first `pairs` (row >= 1, pattern) pairs: the draws, then one history per pair"""
    states, cats = host_route(inst, ev, rows, S, C, P, rng)
    _, pr, _ = rows
    rates = ev.site.getCategoryRates()
    mu, R = un.uniformized(Q)
    N = un.truncation(mu * max(float(lengths[1:].max()) * float(np.max(rates)), 0.0))
    Rn = un.powers(R, N)
    t0 = time.perf_counter()
    done = 0
    for r in range(1, len(pr)):
        u = un.uniforms(int(rng.integers(1 << 62)), 0, np.arange(P), r, 2 * N)
        for p in range(P):
            if done == pairs:
                return time.perf_counter() - t0, done
            tau = lengths[r] * rates[cats[p]]
            _, U, s, _ = un.history(int(states[pr[r], p]), int(states[r, p]), tau, mu, R, Rn, u[p])
            un.registers_of(U, s, tau, Q, regs)
            un.events_of(U, s, lengths[r])
            done += 1
    return time.perf_counter() - t0, done


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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--host-pairs", type=int, default=20_000)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_substitution_histories: no CUDA device")
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
        Q, regs = generator(wname, model), registers(wname, model)
        root = ev.rootIdx[0]
        sample = lambda k: inst.sampleAncestralStates(*rows, root, 0, 0, 2024, k)
        hist = lambda events, k=0: inst.sampleSubstitutionHistories(*rows, lengths, root, 0, 0, 0, Q, regs, 2024, k,
                                                                     states=False, categories=False, events=events)
        for k in range(3):                             # warm-up: module load, scratch and event arrays at their largest
            sample(k)
            hist(True, k)
        full = inst.sampleSubstitutionHistories(*rows, lengths, root, 0, 0, 0, Q, regs, 2024, 7)
        assert np.array_equal(full[0], sample(7)[0])   # the device route draws what the sampler draws
        rec = {"workload": wname, "taxa": tree.tipCount, "patterns": P, "states": S, "categories": C, "rows": len(rows[0]),
               "rescaled": bool(ev.scaling), "logL": logL, "events": int(len(full[5])),
               "events_per_pair": float(len(full[5])) / ((len(rows[0]) - 1) * P)}
        mu = float(np.max(-np.diag(Q)))
        rec["mu_tau_max"] = mu * float(lengths[1:].max()) * float(np.max(site.getCategoryRates()))
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                for k in range(3):
                    hist(True, k)
            kern = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.key.startswith(("k_", "void", "b200")):
                    kern[e.key] = {"calls": e.count, "device_ms_total": e.device_time_total / 1e3}
            rec["profile_3_calls_with_events"] = kern
        else:
            rec["sampler_ms"] = timed(lambda: sample(11), args.reps, torch)
            rec["histories_no_events_ms"] = timed(lambda: hist(False), args.reps, torch)
            rec["histories_with_events_ms"] = timed(lambda: hist(True), args.reps, torch)
            pairs = (len(rows[0]) - 1) * P
            host = []
            for k in range(args.host_reps):
                t0 = time.perf_counter()
                tHist, done = host_histories(inst, ev, rows, lengths, Q, regs, S, C, P, np.random.default_rng(k),
                                             min(pairs, args.host_pairs))
                host.append((1e3 * (time.perf_counter() - t0), 1e3 * tHist, done))
            total, hist_ms, done = (float(np.median([h[i] for h in host])) for i in range(3))
            rec["host_pairs_drawn"] = int(done)
            rec["host_route_measured_ms"] = total
            rec["host_ms_per_pair"] = hist_ms / done
            if done == pairs:
                rec["host_route_ms"] = total
            else:
                rec["host_route_ms_extrapolated"] = total - hist_ms + rec["host_ms_per_pair"] * pairs
            host_ms = rec.get("host_route_ms", rec.get("host_route_ms_extrapolated"))
            rec["host_over_device_with_events"] = host_ms / rec["histories_with_events_ms"]["p50"]
        out.append(rec)
        inst.finalize()
    print(json.dumps({"tool": "bench_substitution_histories", "card": name, "power_limit": limit, "reps": args.reps,
                      "host_reps": args.host_reps, "profile": args.profile, "workloads": out}))


if __name__ == "__main__":
    main()
