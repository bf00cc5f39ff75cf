"""Throughput of crb_dwa_control_batched (dwa_control, src/dynamic_window_approach.cpp:148-155) on the GPU, and of
the CPU oracle on every host core in the same run.  Writes one JSON file.

  python scripts/dwa_bench.py --out DIR

Sizes: n in {4096, 65536, 262144} robots x {10 (the demo's), 64} obstacles, the reference's Config.  Each cell is
warmed up, then timed with CUDA events over at least --min-seconds of back-to-back launches.  decisions/s counts
robots per second; rollouts/s counts the samples of every robot's dynamic window, taken from the grid the oracle
computes (the `best` index space: Nv x Ny per robot).  Needs a CUDA device: there is no CPU fallback."""
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
from oracle import dwa as OD  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def samples_per_robot(x, params):
    """Nv x Ny of each robot's window (calc_dynamic_window :52-60, the loops :126-127) in float32."""
    f = np.float32
    p = params
    dw0 = np.maximum(x[3] - f(p.max_accel * p.dt), f(p.min_speed))
    dw1 = np.minimum(x[3] + f(p.max_accel * p.dt), f(p.max_speed))
    dw2 = np.maximum(x[4] - f(p.max_dyawrate * p.dt), f(-p.max_yawrate))
    dw3 = np.minimum(x[4] + f(p.max_dyawrate * p.dt), f(p.max_yawrate))

    def count(lo, hi, step, cap):
        v, k = lo.copy(), np.zeros(lo.shape, np.int64)
        for _ in range(cap):
            ok = v <= hi
            k += ok
            v = np.where(ok, (v + f(step)).astype(np.float32), v)
        return k
    return count(dw0, dw1, p.v_reso, 64) * count(dw2, dw3, p.yawrate_reso, 512)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--cpu-robots", type=int, default=16384)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dwa_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    p = OD.dwa_params()
    res = dict(gpu=gpu_info(), host_cores=OD.num_threads(), cells=[])
    for k in (10, 64):
        ob = synth.DWA_DEMO_OBSTACLES if k == 10 else synth.dwa_obstacles(k)
        obd = torch.from_numpy(ob).to(dev)
        for n in (4096, 65536, 262144):
            x, u, g = synth.dwa_inputs(n)
            xd, ud0, gd = (torch.from_numpy(v).to(dev) for v in (x, u, g))
            ud = ud0.clone()
            cost = torch.empty(n, dtype=torch.float32, device=dev)
            rollouts = int(samples_per_robot(x, p).sum())
            for _ in range(3):   # warm-up (module load, first launch of the shape)
                eng.dwa_control(xd, ud, gd, obd, cost=cost)
            torch.cuda.synchronize()
            reps, ms = 1, 0.0
            while True:
                ud.copy_(ud0)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(reps):
                    eng.dwa_control(xd, ud, gd, obd, cost=cost)
                t1.record()
                t1.synchronize()
                ms = t0.elapsed_time(t1)
                if ms >= 1000.0 * a.min_seconds:
                    break
                reps = max(reps * 2, int(reps * 1000.0 * a.min_seconds / max(ms, 1e-3) * 1.2))
            per = ms / 1000.0 / reps
            cell = dict(n=n, n_ob=k, reps=reps, seconds=ms / 1000.0, call_ms=per * 1e3, decisions_per_s=n / per,
                        rollouts_per_call=rollouts, rollouts_per_s=rollouts / per)
            if n == 4096 or n == 65536:
                m = min(n, a.cpu_robots)
                OD.dwa_control(x[:, :64], u[:, :64], g[:, :64], ob, p, traj=False)
                t = time.perf_counter()
                OD.dwa_control(np.ascontiguousarray(x[:, :m]), np.ascontiguousarray(u[:, :m]),
                              np.ascontiguousarray(g[:, :m]), ob, p, traj=False)
                dt = time.perf_counter() - t
                frac = int(samples_per_robot(x[:, :m], p).sum())
                cell.update(cpu_robots=m, cpu_seconds=dt, cpu_decisions_per_s=m / dt, cpu_rollouts_per_s=frac / dt,
                            speedup_vs_cpu=(n / per) / (m / dt))
            res["cells"].append(cell)
            print(json.dumps(cell), flush=True)
    eng.close()
    with open(os.path.join(a.out, "dwa_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
