#!/usr/bin/env python3
"""Turn the raw material a GPU-box pass left in gpurun_out/ (tools/collect_round_evidence.sh) into the committed summaries
under profiles/:  python tools/summarise_round_evidence.py h100

  <R>_traffic.json     DRAM bytes per step of the updatePartials launches, per workload (ncu dram__bytes_{read,write}.sum)
  <R>_ncu_raw.txt      selected metrics of the --set full captures (tools/ncu_summary.py)
  <R>_sass_excerpts.txt  per-kernel counts of the SASS mnemonics that identify the hardware paths in the SHIPPED library
  copies of the bench lines / launch list / test logs
"""
import csv
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = sys.argv[1] if len(sys.argv) > 1 else "h100"
G = os.path.join(ROOT, "gpurun_out")
P = os.path.join(ROOT, "profiles")
os.makedirs(P, exist_ok=True)


def launches(path):
    """[(kernel name, grid, {metric: value})] in launch order from an ncu --csv log."""
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 10]
    hdr = next(r for r in rows if r[0] == "ID")
    col = {h: i for i, h in enumerate(hdr)}
    out, by_id = [], {}
    for r in rows:
        if r[0] == "ID" or not r[0].isdigit():
            continue
        key = r[col["ID"]]
        if key not in by_id:
            by_id[key] = (r[col["Kernel Name"]], r[col["Grid Size"]], {})
            out.append(by_id[key])
        v = r[col["Metric Value"]].replace(",", "")
        unit = r[col["Metric Unit"]].lower()
        scale = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "nsecond": 1e-9, "usecond": 1e-6, "msecond": 1e-3,
                 "second": 1, "ns": 1e-9, "us": 1e-6, "ms": 1e-3}.get(unit, 1)
        try:
            by_id[key][2][r[col["Metric Name"]]] = float(v) * scale
        except ValueError:
            pass
    return out


def traffic():
    table = {}
    for f in sorted(os.listdir(G)):
        m = re.match(rf"{R}_traffic_(.+)\.csv$", f)
        if not m:
            continue
        walk = [l for l in launches(os.path.join(G, f)) if "k_walk" in l[0]]
        grids = [l[1] for l in walk]
        period = None
        for L in range(1, 13):
            if len(grids) >= 3 * L and grids[-L:] == grids[-2 * L:-L] == grids[-3 * L:-2 * L]:
                period = L
                break
        if period is None:
            continue
        step = walk[-period:]
        table[m.group(1)] = {
            "dram_bytes_read_per_step": sum(l[2].get("dram__bytes_read.sum", 0.0) for l in step),
            "dram_bytes_write_per_step": sum(l[2].get("dram__bytes_write.sum", 0.0) for l in step),
            "launches_per_step": period,
            "kernels": sorted({re.sub(r"\(.*", "", l[0]) for l in step}),
            "ncu_time_us_per_step": 1e6 * sum(l[2].get("gpu__time_duration.sum", 0.0) for l in step),
            "source": f"gpurun_out/{f} -> profiles/{R}_traffic.json: dram__bytes_read.sum + dram__bytes_write.sum summed over the "
                      f"{period} k_walk* launches of ONE step (ncu --metrics, --clock-control none)"}
    if table:
        json.dump(table, open(os.path.join(P, f"{R}_traffic.json"), "w"), indent=1)
    return table


def sass_excerpts():
    lib = os.path.join(ROOT, "beast-mcmc_b200", "csrc", "libhmsbeagle.so")
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    pat = re.compile(r"\b(DMMA[.\w]*|DFMA|UBLKCP[.\w]*|SYNCS[.\w]*|LDGSTS[.\w]*|LDG\.E\.ENL2\.256[.\w]*|STG\.E\.ENL2\.256|"
                     r"LDS\.128|UTC\w*MMA|LDTM|UTMALDG|HMMA[.\w]*|CCTL\.E\.PF1|R2UR|LDCU[.\w]*)\b")
    per, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            name = name.replace("(anonymous namespace)::", "")
            name = re.sub(r"\(b200::.*|\((const|double|int|unsigned|long|void).*", "", name)
            name = re.sub(r"^void\s+", "", name).replace("b200::", "")
            name = name.replace("(int)", "").replace("(bool)0", "false").replace("(bool)1", "true")
            per[name] = {}
            continue
        if name:
            for op in pat.findall(line):
                key = re.sub(r"\.(CONSTANT|STRONG|GPU|SYS).*", "", op)
                per[name][key] = per[name].get(key, 0) + 1
    keep = ("k_walk4p<4, 4>", "k_walk4ps<4, 4>", "k_walk4p<4, 1>", "k_walk4pv<4, 4>", "k_walk4pv<4, 1>", "k_walk4e<4, 4, false>", "k_walk4<4, 4, false>", "k_walk_mma<8, 4, false, false, 2>",
            "k_walk_mma<8, 4, false, false, 1>", "k_walk_mma<3, 4, false, true, 2>", "k_transition_mma<8>", "k_incremental<4>", "k_root", "k_exchange_sum", "k_cross_mma<8>",
            "k_edge_derivatives_mma<8>")
    with open(os.path.join(P, f"{R}_sass_excerpts.txt"), "w") as f:
        f.write("# SASS mnemonic counts per kernel of the shipped libhmsbeagle.so (cuobjdump -sass; static instruction counts)\n")
        f.write("# DMMA = mma.sync m8n8k4 f64 (fp64 tensor pipe); UBLKCP/SYNCS = cp.async.bulk + mbarrier (TMA engine);\n")
        f.write("# LDGSTS = cp.async; LDCU/R2UR + DFMA = constant-bank operands through\n")
        f.write("# uniform registers; no HGMMA: wgmma has no fp64 kind\n")
        source_hash = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r); import beast_mcmc_b200; "
                                      "from beast_mcmc_b200 import build; print(build.verify_engine())" % ROOT],
                                     capture_output=True, text=True).stdout.strip()
        f.write(f"# library source hash {source_hash}\n")
        for k in keep:
            if k in per:
                f.write((f"{k}: " + ", ".join(f"{op} {n}" for op, n in sorted(per[k].items()))).rstrip() + "\n")
        total = {}
        for d in per.values():
            for op, n in d.items():
                total[op] = total.get(op, 0) + n
        f.write("ALL KERNELS: " + ", ".join(f"{op} {n}" for op, n in sorted(total.items())) + "\n")
    return per


def ncu_raw():
    out = os.path.join(P, f"{R}_ncu_raw.txt")
    with open(out, "w") as f:
        for rep, title in ((f"{R}_walk4p_full", "k_walk4p launches of one cfg-2 step"),
                           (f"{R}_walk_mma_codon_full", "k_walk_mma phase-1 launch, codon workload"),
                           (f"{R}_incremental_full", "k_incremental (fused incremental evaluation), cfg 2")):
            path = os.path.join(G, rep + ".ncu-rep")
            if not os.path.exists(path):
                continue
            f.write(f"# {title} (ncu --set full, gpurun_out/{rep}.ncu-rep)\n")
            f.write(subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_summary.py"), path],
                                   capture_output=True, text=True).stdout)


def copies():
    for f in sorted(os.listdir(G)):
        if f.startswith(R + "_") and (f.endswith(".json") or f.endswith(".txt") or f == f"{R}_launches.csv"):
            shutil.copy(os.path.join(G, f), os.path.join(P, f))


if __name__ == "__main__":
    t = traffic()
    print("traffic:", {k: (round(v["dram_bytes_read_per_step"] / 1e9, 3), round(v["dram_bytes_write_per_step"] / 1e9, 3)) for k, v in t.items()})
    sass_excerpts()
    ncu_raw()
    copies()
    print("profiles/ updated for", R)
