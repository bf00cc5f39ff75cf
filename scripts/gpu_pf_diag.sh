#!/bin/bash
# PF kernel diagnostics: time per launch vs particle count and vs landmark count
OUT=gpurun_out; mkdir -p $OUT
run() { CRB_BENCH_PF_N=$1 CRB_BENCH_PF_LM=$2 python bench.py --steps 50 --warmup 5 --no-cpu --workload pf 2>/dev/null | \
    python -c "import json,sys; d=json.loads(sys.stdin.readline()); d=d.get('extra',{}).get('pf',d); print('PF n=$1 lm=$2', 'us/launch %.2f' % (d['ms_per_step']*1e3), 'GB/s %.0f frac %.3f' % (d['roofline']['achieved'], d['roofline']['frac']))"; }
( for n in 262144 524288 1048576 2097152 4194304 16777216; do run $n 8; done
  for lm in 0 1 2 4 8 16; do run 1048576 $lm; done ) | tee $OUT/pf_diag.txt
