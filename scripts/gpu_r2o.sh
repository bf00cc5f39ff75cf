#!/bin/bash
# MPC hinted order: parity subset + timing.
OUT=gpurun_out; mkdir -p $OUT
[ -n "$SKIP_PYTEST" ] || timeout 600 python -m pytest tests/test_gpu_parity.py -x -q -k "pf_step or hinted or pf_sharded or resample" > $OUT/o_pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/o_pytest.log
timeout 400 python bench.py --workload mpc --no-cpu --steps 20 --warmup 5 > $OUT/o_mpc.json 2> $OUT/o_mpc.err
tail -4 $OUT/o_pytest.log
python scripts/show_bench.py $OUT/o_mpc.json 2>&1 | grep "MPC" || tail -20 $OUT/o_mpc.err
