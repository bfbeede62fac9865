#!/bin/bash
# One GPU-box pass that regenerates the raw material under profiles/ for a round:  bash tools/collect_round_evidence.sh h100
# (everything lands in gpurun_out/; tools/summarise_round_evidence.py turns it into the committed summaries here)
R=${1:-h100}
mkdir -p gpurun_out
./tools/bin/fp64_peaks > gpurun_out/${R}_fp64_peaks.json 2> gpurun_out/${R}_fp64_peaks.err; cat gpurun_out/${R}_fp64_peaks.json
python -m pytest tests -m gpu -q 2>&1 | tail -3 > gpurun_out/${R}_gpu_tests.txt; cat gpurun_out/${R}_gpu_tests.txt
python bench.py --steps 3 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1        # alignment cache
# launch list of the default bench command's main section (serialised, cold: shares, not absolutes)
ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/${R}_launches.csv \
    python bench.py --steps 3 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
# DRAM traffic of every walk launch, per workload (algorithmic bytes vs what reaches HBM)
for w in gtr_g4_1000x10k gtr_g4_1000x10k_rescaled makona_like_1610x6k codon_mg94_500x5k aa20_g4_500x5k; do
  python bench.py --workload $w --steps 2 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
  ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none -k regex:k_walk --csv \
      --log-file gpurun_out/${R}_traffic_$w.csv python bench.py --workload $w --steps 2 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
done
# full captures of the dominant kernels (one step's launches)
ncu --set full --clock-control none --import-source on -k regex:k_walk4p -s 30 -c 3 -o gpurun_out/${R}_walk4p_full \
    python bench.py --steps 3 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
ncu --set full --clock-control none --import-source on -k regex:k_walk_mma -s 8 -c 1 -o gpurun_out/${R}_walk_mma_codon_full \
    python bench.py --workload codon_mg94_500x5k --steps 3 --warmup 3 --no-cpu-baseline --no-extras > /dev/null 2>&1
ncu --set full --clock-control none --import-source on -k regex:k_incremental -s 20 -c 2 -o gpurun_out/${R}_incremental_full \
    python bench.py --steps 3 --warmup 3 --no-cpu-baseline > /dev/null 2>&1
# bench lines
python bench.py 2>&1 | tail -1 > gpurun_out/${R}_bench_cfg2.json
python bench.py --impl reference --steps 30 --warmup 3 2>&1 | tail -1 > gpurun_out/${R}_bench_cfg2_reference.json
python bench.py --steps 20 --warmup 5 --no-cpu-baseline 2>&1 | tail -1 > gpurun_out/${R}_bench_cfg2_steps20.json
python bench.py --workload gtr_g4_1000x10k_rescaled --steps 300 --warmup 10 --no-cpu-baseline 2>&1 | tail -1 > gpurun_out/${R}_bench_cfg2_rescaled.json
python bench.py --workload codon_mg94_500x5k --steps 100 --warmup 5 --cpu-budget 8 2>&1 | tail -1 > gpurun_out/${R}_bench_codon.json
python bench.py --workload codon_mg94_500x5k_g4 --steps 30 --warmup 5 --no-cpu-baseline 2>&1 | tail -1 > gpurun_out/${R}_bench_codon_g4.json
python bench.py --workload aa20_g4_500x5k --steps 100 --warmup 5 --no-cpu-baseline 2>&1 | tail -1 > gpurun_out/${R}_bench_aa20.json
python bench.py --workload hky_1441x593 --steps 1000 --warmup 10 --cpu-budget 4 2>&1 | tail -1 > gpurun_out/${R}_bench_hky1441.json
python bench.py --workload makona_like_1610x6k --steps 300 --warmup 10 --cpu-budget 6 2>&1 | tail -1 > gpurun_out/${R}_bench_makona_like.json
python bench.py --workload benchmark1_xml --steps 1000 --warmup 10 --cpu-budget 4 2>&1 | tail -1 > gpurun_out/${R}_bench_benchmark1_xml.json
python bench.py --workload benchmark2_xml --steps 1000 --warmup 10 --cpu-budget 4 2>&1 | tail -1 > gpurun_out/${R}_bench_benchmark2_xml.json
python tools/bench_gradient.py > /dev/null 2>&1
WORKLOAD=codon_mg94_500x5k STEPS=5 python tools/bench_gradient.py > /dev/null 2>&1
STEPS=100 python tools/bench_partitions.py 2>&1 | tail -1 > gpurun_out/${R}_bench_partitions.json
python tools/bench_patterns.py 2>&1 | tail -1 > gpurun_out/${R}_bench_patterns.json
bash tools/sanitize.sh > gpurun_out/${R}_sanitizer.txt 2>&1; tail -5 gpurun_out/${R}_sanitizer.txt
for f in gpurun_out/${R}_bench_*.json; do python - $f <<'PY'
import json, sys
try:
    d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
    r = d.get("roofline", {}); c = d.get("cpu_baseline") or {}
    print(sys.argv[1].split("/")[-1], "value %.1f e2e %.1f ms/step %.4f" % (d["value"], d["e2e"]["value"], d["ms_per_step"]),
          "partials_ms", r.get("partials_ms_per_step"), "frac", r.get("frac"), "gflops", r.get("gflops"),
          "cpu %s (%s thr)" % (c.get("value"), c.get("cores")), "inc_us", (d.get("incremental") or {}).get("us_per_eval"))
except Exception as e:
    print(sys.argv[1], "UNREADABLE", e)
PY
done
