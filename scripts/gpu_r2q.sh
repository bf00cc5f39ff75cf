#!/bin/bash
# MPC hinted order with one bin for the short problems.
OUT=gpurun_out; mkdir -p $OUT
timeout 600 python -m pytest tests/test_gpu_parity.py -x -q -k "hinted" > $OUT/q_pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/q_pytest.log
timeout 400 python bench.py --workload mpc --no-cpu --steps 20 --warmup 5 > $OUT/q_mpc.json 2> $OUT/q_mpc.err
tail -3 $OUT/q_pytest.log
python scripts/show_bench.py $OUT/q_mpc.json 2>&1 | grep "MPC" || tail -20 $OUT/q_mpc.err
