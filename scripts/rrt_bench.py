"""Throughput of RRT planning on the GPU (crb_rrt_plan_batched) against the CPU checker on every host core, in the same
run.  Writes one JSON file.

  python scripts/rrt_bench.py --out DIR [--reps 5]

Maps: the demo (src/rrt.cpp: six circles, rand_area [-2, 15], expand_dis 0.5) and a dense seeded map of 64 circles over
[-20, 40)^2 (synth.rrt_scatter_obstacles, expand_dis 1.0), each with synth.rrt_inputs queries; fleets of 2^12 and 2^16
queries; max_iter 4096, far above the demo's longest run (about 1,600 draws), so that the cap is rare: the count of
MAX_ITER_REACHED queries is reported.  Each cell is timed with CUDA events over --reps launches after one warm-up
launch.  Reported: ms per launch, queries/s, accepted nodes/s (the sum of n_nodes) and loop passes/s (the sum of
n_iter), the status counts, the checker's time for the same queries on every host core and whether every GPU output is
bit-identical to it, and the card name and power limit read in the same run.  Needs a CUDA device: there is no CPU
fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, rrt_default_params, synth  # noqa: E402
from oracle import rrt as OR  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rrt_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    res = dict(gpu=gpu_info(), host_cores=OR.num_threads(), reps=a.reps, cells=[])
    d = synth.RRT_DEMO
    maps = {"demo": (synth.rrt_demo_obstacles(), d["rand_min"], d["rand_max"], d["expand_dis"]),
            "dense64": (synth.rrt_scatter_obstacles(64, -20.0, 40.0), -20.0, 40.0, 1.0)}
    max_pts, max_nodes = 128, 1024
    for name, (ob, lo, hi, e) in maps.items():
        p = rrt_default_params()
        p.rand_min, p.rand_max, p.expand_dis, p.max_iter = lo, hi, e, 4096
        prm = dict(rand_min=p.rand_min, rand_max=p.rand_max, expand_dis=p.expand_dis,
                   goal_sample_rate=p.goal_sample_rate, max_iter=p.max_iter)
        obd = torch.from_numpy(ob).to(dev)
        for nq in (1 << 12, 1 << 16):
            se, seed = synth.rrt_inputs(nq, ob, lo, hi)
            sed, sdd = torch.from_numpy(se).to(dev), torch.from_numpy(seed.view(np.int32)).to(dev)
            out = eng.rrt_plan(obd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes)   # warm-up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                eng.rrt_plan(obd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes, **out)
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            g = {k: v.cpu().numpy() for k, v in out.items()}
            t = time.perf_counter()
            o = OR.plan(prm, ob, se, seed, max_pts=max_pts, max_nodes=max_nodes)
            cpu_s = time.perf_counter() - t
            nodes, iters = int(g["n_nodes"].astype(np.int64).sum()), int(g["n_iter"].astype(np.int64).sum())
            cell = dict(map=name, queries=nq, max_iter=p.max_iter, gpu_ms=ms, gpu_queries_per_s=nq / (ms / 1e3),
                        gpu_nodes_per_s=nodes / (ms / 1e3), gpu_iterations_per_s=iters / (ms / 1e3),
                        cpu_seconds=cpu_s, cpu_queries_per_s=nq / cpu_s, gpu_over_cpu=cpu_s / (ms / 1e3),
                        nodes=nodes, iterations=iters,
                        status_hist=dict(zip(["found", "max_iter_reached", "bad_input"],
                                             np.bincount(g["status"], minlength=3).tolist())),
                        bit_identical=all(same(g[k], o[k]) for k in ("path", "path_len", "tree", "parent", "n_nodes",
                                                                     "n_iter", "status")))
            res["cells"].append(cell)
            print(json.dumps(cell), flush=True)
    eng.close()
    with open(os.path.join(a.out, "rrt_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
