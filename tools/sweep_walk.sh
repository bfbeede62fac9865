#!/bin/bash
# Kernel-variant sweep for the 4-state walk (run on the GPU box): one bench line per setting.
# columns: reorder phaseT(0=auto) R(patterns/thread) Tmin oversub
mkdir -p gpurun_out
python bench.py --steps 5 --warmup 3 --no-cpu-baseline > /dev/null 2>&1   # builds the alignment cache
CFGS=${CFGS:-"1 0 2 4 3;1 0 2 4 2;1 0 2 8 2;1 0 4 4 2;1 0 2 16 2;1 0 2 4 1"}
IFS=';' read -ra LIST <<< "$CFGS"
for cfg in "${LIST[@]}"; do
  set -- $cfg
  echo "reorder=$1 phaseT=$2 R=$3 Tmin=$4 oversub=$5"
  B200_REORDER=$1 B200_PHASE_T=$2 B200_WALK_R=$3 B200_PHASE_TMIN=$4 B200_PHASE_OVERSUB=$5 \
    python bench.py --steps ${STEPS:-100} --warmup 5 --no-cpu-baseline $BENCH_ARGS 2>&1 | python -c "
import sys, json
for l in sys.stdin:
    if l.startswith('{'):
        d = json.loads(l)
        r = d['roofline']
        print('  value %.1f evals/s  e2e %.1f  ms/step %.4f  partials %.4f ms/step (%d launches/step)  %.0f GB/s (frac %.3f)  %.1f GF/s  mat %.4f root %.4f logL %.6f' % (
            d['value'], d['e2e']['value'], d['ms_per_step'], r['partials_ms_per_step'], r['launches_per_step'], r['achieved'], r['frac'], r['gflops'],
            r['other_kernels_ms_per_step']['transition_matrices'], r['other_kernels_ms_per_step']['root'], d['logL']))
    else:
        sys.stdout.write(l)
"
done 2>&1 | tee gpurun_out/sweep_walk.txt
