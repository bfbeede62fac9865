"""Sibling stack of the staged eigen walk on and off (B200_WALK_STACK_SLOTS=0) on one GPU, same process, alternating.

For every workload: two instances of the same evaluation, one with the per-warp shared-memory sibling stack and one
without, timed in blocks of --steps steps with bench.py's pattern (tools/bench_precision.py's Arm: resident eigen system,
buffers flipping like BEAST's, a CUDA event between consecutive steps).  The blocks run in ABBA order, so drift over the
run falls on both arms alike.  Per arm: the median over its blocks of the block's p50 step, the partials-kernel time per
step (b200SetKernelTiming, two runs per arm, also ABBA) and the plan counts of the B200_BEAGLE_DEBUG line (children read from
the stack / from memory) and, for every staged-walk launch of the first evaluation, its sibling-stack bytes per block and
its cudaOccupancyMaxActiveBlocksPerMultiprocessor (the same debug output).  Also: the card's fill and copy bandwidth
(tools/write_bw.py's method), the store floor of each workload (the partials its walk stores per step -- one buffer per op
that runs, virtual cherries are not run -- over the measured fill bandwidth), and the card name and power limit.  Both
arms must give the same site log-likelihoods bit for bit.  Prints ONE JSON line.

    python tools/bench_walk_stack.py --steps 200 --warmup 20 --blocks 4
"""
import argparse
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import bench_precision as bp  # noqa: E402
from beast_mcmc_b200 import beagle  # noqa: E402

WORKLOADS = ("gtr_g4_1000x10k", "makona_like_1610x6k", "gtr_g4_1000x10k_rescaled", "hky_1441x593", "benchmark2_xml")


def bandwidth(torch):
    """fill (write) and copy (read + write) GB/s over 1.34 GB, as tools/write_bw.py measures them"""
    x = torch.empty(1280 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    y = torch.empty_like(x)

    def t(fn, n=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n

    nbytes = x.numel() * 8
    fill = nbytes / t(lambda: x.fill_(1.0)) / 1e6
    copy = 2 * nbytes / t(lambda: y.copy_(x)) / 1e6
    del x, y
    torch.cuda.empty_cache()
    return fill, copy


def plan_counts(text):
    """(ops run, forwarded, read from the stack, read from memory) of every plan line; (stack bytes per block, blocks per
    SM) of every staged-walk launch line"""
    plans = re.findall(r"plan: (\d+) ops .*?(\d+) forwarded in registers, (\d+) read from the stack, (\d+) from memory", text)
    launches = re.findall(r"staged walk: (\d+) B sibling stack per block, (\d+) blocks per SM", text)
    return [[int(v) for v in row] for row in plans], sorted({(int(a), int(b)) for a, b in launches})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=4, help="timed blocks per arm, in ABBA order")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_walk_stack: no CUDA device")
    D = bp._Local(torch)
    lib = beagle.load_library()
    name, limit = bp.card()
    fill, copy = bandwidth(torch)
    rows = []
    for wname in args.workloads.split(","):
        w, tree, pats, model, site = bench.build_workload(wname, 0, {})
        S, C, P = w["states"], site.getCategoryCount(), pats.patternCount
        ev = bench.Evaluation(tree, pats, model, site, "REVERSE_LEVEL_ORDER", scaling=bool(w.get("scaling")))
        arms, counts = {}, {}
        for a, slots in (("on", None), ("off", "0")):
            old = os.environ.get("B200_WALK_STACK_SLOTS")
            if slots is not None:
                os.environ["B200_WALK_STACK_SLOTS"] = slots
            os.environ["B200_BEAGLE_DEBUG"] = "1"
            with tempfile.TemporaryFile(mode="w+") as err:      # the plan line goes to the process's stderr
                saved = os.dup(2)
                sys.stderr.flush()
                os.dup2(err.fileno(), 2)
                try:
                    arms[a] = bp.Arm(D, lib, ev, S, C, P, 0)
                    arms[a].step(1)
                    D.bracket()
                finally:
                    os.dup2(saved, 2)
                    os.close(saved)
                    os.environ.pop("B200_BEAGLE_DEBUG", None)
                    if old is None:
                        os.environ.pop("B200_WALK_STACK_SLOTS", None)
                    else:
                        os.environ["B200_WALK_STACK_SLOTS"] = old
                err.seek(0)
                plans, launches = plan_counts(err.read())
                counts[a] = {"plan_ops_forwarded_stack_memory": plans, "stack_bytes_blocks_per_sm": launches}
        on, off = arms["on"], arms["off"]
        for b in range(args.blocks):                   # ABBA
            for arm in ((on, off) if b % 2 == 0 else (off, on)):
                arm.block(args.steps, args.warmup)
        ks = {"on": [], "off": []}
        for a, arm in (("on", on), ("off", off), ("off", off), ("on", on)):     # ABBA
            ks[a].append(arm.partials_ms(args.steps))
        ks = {a: tuple(float(np.mean(v)) for v in zip(*m)) for a, m in ks.items()}
        s_on, s_off = on.sites(), off.sites()
        ops_run = counts["on"]["plan_ops_forwarded_stack_memory"][0][0]
        stored_bytes = ops_run * C * (-(-P // 32) * 32) * 4 * 8         # [C][Ppad][4] fp64 per buffer
        row = {"workload": wname, "taxa": tree.tipCount, "patterns": P, "categories": C,
               "rescaled": bool(ev.scaling), "sites_bit_equal": bool(np.array_equal(s_on, s_off)),
               "stored_GB_per_step": stored_bytes / 1e9, "store_floor_ms": stored_bytes / (fill * 1e9) * 1e3}
        for a, arm in (("on", on), ("off", off)):
            row[a] = {"step_ms_p50": float(np.median(arm.p50)), "block_p50s": [float(x) for x in arm.p50],
                      "partials_kernel_ms_per_step": ks[a][0], "partials_launches_per_step": ks[a][1],
                      **counts[a]}
        row["on_over_off_step"] = row["on"]["step_ms_p50"] / row["off"]["step_ms_p50"]
        rows.append(row)
        on.inst.finalize()
        off.inst.finalize()
    print(json.dumps({"tool": "bench_walk_stack", "card": name, "power_limit": limit, "fill_GBps": fill, "copy_GBps": copy,
                      "steps": args.steps, "warmup": args.warmup, "blocks_per_arm": args.blocks, "workloads": rows}))


if __name__ == "__main__":
    main()
