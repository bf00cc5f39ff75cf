"""Throughput of the grid planners on the GPU (crb_grid_plan_batched, A* and Dijkstra) against the CPU checker on
every host core, in the same run.  Writes one JSON file.

  python scripts/grid_bench.py --out DIR [--reps 10]

Maps: the demo's walls (60 x 60 cells) and the seeded 128 x 128 scatter (synth.grid_scatter_obstacles(128)), each with
synth.grid_inputs queries; fleets of 2^12 and 2^16 queries.  Each cell is timed with CUDA events over --reps launches
after one warm-up launch (which also allocates the workspace).  Reported: ms per launch, queries/s, visited cells/s
(the sum of n_visited over the launch's queries), the slots (concurrent searches) used, the status counts, the
checker's time for the same queries on every host core and whether the GPU outputs are bit-identical to it, and the
card name and power limit read in the same run.  Needs a CUDA device: there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, GridBox, synth  # noqa: E402
from oracle import grid as OG  # noqa: E402


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
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("grid_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    res = dict(gpu=gpu_info(), host_cores=OG.num_threads(), reps=a.reps, cells=[])
    d = synth.GRID_DEMO
    maps = {"demo60": (*synth.grid_demo_obstacles(), d["reso"], d["rr"]),
            "scatter128": (*synth.grid_scatter_obstacles(128), 1.0, 1.0)}
    max_pts = 64
    for name, (ox, oy, reso, rr) in maps.items():
        gb = OG.box_of_obstacles(ox, oy, reso)
        box = GridBox(*[int(v) for v in gb])
        md = eng.grid_obstacle_map(torch.from_numpy(ox).to(dev), torch.from_numpy(oy).to(dev), reso, rr, box)
        m = md.cpu().numpy()
        for algo, aname in ((OG.ASTAR, "astar"), (OG.DIJKSTRA, "dijkstra")):
            for nq in (1 << 12, 1 << 16):
                sg = synth.grid_inputs(nq, gb, m, reso)
                sgd = torch.from_numpy(sg).to(dev)
                out = eng.grid_plan(algo, box, md, reso, sgd, max_pts=max_pts)   # warm-up, allocates the workspace
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    eng.grid_plan(algo, box, md, reso, sgd, max_pts=max_pts, **out)
                e1.record()
                e1.synchronize()
                ms = e0.elapsed_time(e1) / a.reps
                g = {k: v.cpu().numpy() for k, v in out.items()}
                t = time.perf_counter()
                o = OG.plan(algo, gb, m, reso, sg, max_pts=max_pts)
                cpu_s = time.perf_counter() - t
                visited = int(g["n_visited"].astype(np.int64).sum())
                cell = dict(map=name, algo=aname, queries=nq, slots=eng.grid_plan_slots(algo, box, nq), gpu_ms=ms,
                            gpu_queries_per_s=nq / (ms / 1e3), gpu_visited_cells_per_s=visited / (ms / 1e3),
                            cpu_seconds=cpu_s, cpu_queries_per_s=nq / cpu_s, cpu_visited_cells_per_s=visited / cpu_s,
                            gpu_over_cpu=(nq / (ms / 1e3)) / (nq / cpu_s), visited_cells=visited,
                            status_hist=dict(zip(["found", "no_path", "start_outside", "bad_point"],
                                                 np.bincount(g["status"], minlength=4).tolist())),
                            bit_identical=all(same(g[k], o[k]) for k in ("path", "path_len", "cost", "n_visited",
                                                                         "status")))
                res["cells"].append(cell)
                print(json.dumps(cell), flush=True)
    eng.close()
    with open(os.path.join(a.out, "grid_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
