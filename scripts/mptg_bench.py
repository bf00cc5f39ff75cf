"""Throughput of crb_mptg_optimize_batched (TrajectoryOptimizer::optimizer_traj, include/trajectory_optimizer.h
:53-128) on the GPU, and of the CPU checker on every host core in the same run.  Writes one JSON file.

  python scripts/mptg_bench.py --out DIR

Sizes: n in {2^16, 2^20} problems of synth.mptg_inputs (targets around the demo's, its max_iter / cost_th / h_step),
no trajectory output.  Each size is warmed up, then timed with CUDA events over at least --min-seconds of
back-to-back launches (param is restored before every launch).  problems/s counts problems per second;
rollouts/s counts the roll-outs the reference itself would make for the same results: per iteration one
nominal, six for the Jacobian and two for the line search (9 per update, plus the nominal of the last iteration
when it stops there).  The status histogram, including how often CRB_MPTG_OUT_OF_RANGE fires, is reported for
each size.  Needs a CUDA device: there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, synth  # noqa: E402
from oracle import mptg as OM  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def reference_rollouts(status, iters):
    """Roll-outs optimizer_traj makes: 9 per update, plus the last iteration's nominal unless max_iter ran out."""
    iters = iters.astype(np.int64)
    return int((9 * iters + (status != OM.MAX_ITER_REACHED)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--cpu-problems", type=int, default=65536)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mptg_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    p = eng.mptg_default_params()
    res = dict(gpu=gpu_info(), host_cores=OM.num_threads(), cells=[])
    for n in (1 << 16, 1 << 20):
        st, tg, pa = synth.mptg_inputs(n)
        sd, td, qd0 = (torch.from_numpy(v).to(dev) for v in (st, tg, pa))
        qd = qd0.clone()
        status = torch.empty(n, dtype=torch.int32, device=dev)
        iters = torch.empty(n, dtype=torch.int32, device=dev)
        for _ in range(2):   # warm-up (module load, first launch of the shape)
            qd.copy_(qd0)
            eng.mptg_optimize(sd, td, qd, p, status=status, iters=iters)
        torch.cuda.synchronize()
        reps, ms = 1, 0.0
        while True:
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(reps):
                qd.copy_(qd0)
                eng.mptg_optimize(sd, td, qd, p, status=status, iters=iters)
            t1.record()
            t1.synchronize()
            ms = t0.elapsed_time(t1)
            if ms >= 1000.0 * a.min_seconds:
                break
            reps = max(reps * 2, int(reps * 1000.0 * a.min_seconds / max(ms, 1e-3) * 1.2))
        per = ms / 1000.0 / reps
        s, it = status.cpu().numpy(), iters.cpu().numpy()
        ro = reference_rollouts(s, it)
        corner = (np.arange(n) % 64) <= 5
        hist = np.bincount(s, minlength=5).tolist()
        cell = dict(n=n, reps=reps, seconds=ms / 1000.0, call_ms=per * 1e3, problems_per_s=n / per,
                    rollouts_per_call=ro, rollouts_per_s=ro / per, mean_iters=float(it.mean()),
                    status_hist=dict(zip(["converged", "max_iter_reached", "empty_traj", "step_cap", "out_of_range"],
                                         hist)),
                    out_of_range_outside_corner_cases=int(((s == OM.OUT_OF_RANGE) & ~corner).sum()))
        if n <= a.cpu_problems:
            OM.optimize(st[:, :64], tg[:, :64], pa[:, :64], p)
            t = time.perf_counter()
            o = OM.optimize(st, tg, pa, p)
            dt = time.perf_counter() - t
            assert np.array_equal(o["status"], s) and np.array_equal(o["iters"], it)
            cell.update(cpu_problems=n, cpu_seconds=dt, cpu_problems_per_s=n / dt, cpu_rollouts_per_s=ro / dt,
                        speedup_vs_cpu=(n / per) / (n / dt))
        res["cells"].append(cell)
        print(json.dumps(cell), flush=True)
    eng.close()
    with open(os.path.join(a.out, "mptg_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
