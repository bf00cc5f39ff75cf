"""Throughput of RRT planning on the GPU (crb_rrt_plan_batched) against the CPU checker on every host core, in the same
run.  Writes one JSON file.

  python scripts/rrt_bench.py --out DIR [--reps 5] [--cells shared|many|all]

Maps: the demo (src/rrt.cpp: six circles, rand_area [-2, 15], expand_dis 0.5) and a dense seeded map of 64 circles over
[-20, 40)^2 (synth.rrt_scatter_obstacles, expand_dis 1.0), each with synth.rrt_inputs queries; fleets of 2^12 and 2^16
queries; max_iter 4096, far above the demo's longest run (about 1,600 draws), so that the cap is rare: the count of
MAX_ITER_REACHED queries is reported.  Each cell is timed with CUDA events over --reps launches after one warm-up
launch.  Reported: ms per launch, queries/s, accepted nodes/s (the sum of n_nodes) and loop passes/s (the sum of
n_iter), the status counts, the checker's time for the same queries on every host core and whether every GPU output is
bit-identical to it, and the card name and power limit read in the same run.

Obstacle list per query (crb_rrt_plan_many_batched), 2^16 queries, max_iter 4096 (`many_*` cells):
  a  the demo map through crb_rrt_plan_many_batched (one list, ob_of all 0) and through crb_rrt_plan_batched,
     alternated over --reps rounds; the median and spread of each
  b  1024 scattered maps of 0 to 64 circles over the demo's area (synth.rrt_fleet_obstacles), queries shuffled over
     them, against one crb_rrt_plan_batched launch per map
Every output is compared bitwise with the shared-list launches.  Needs a CUDA device: there is no CPU fallback."""
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


def _events_ms(fn, reps):
    import torch
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


KEYS = ("path", "path_len", "tree", "parent", "n_nodes", "n_iter", "status")


def many_cells(eng, res, reps):
    """The `many_*` cells of the module docstring."""
    import torch
    dev = torch.device("cuda:0")
    d = synth.RRT_DEMO
    lo, hi = d["rand_min"], d["rand_max"]
    p = rrt_default_params()
    p.rand_min, p.rand_max, p.expand_dis, p.max_iter = lo, hi, d["expand_dis"], 4096
    nq, max_pts, max_nodes = 1 << 16, 128, 1024
    host = lambda r: {k: r[k].cpu().numpy() for k in KEYS}  # noqa: E731

    # a: the demo map, both paths alternated
    ob = synth.rrt_demo_obstacles()
    se, seed = synth.rrt_inputs(nq, ob, lo, hi)
    obd, sed, sdd = (torch.from_numpy(v).to(dev) for v in (ob, se, seed.view(np.int32)))
    off = torch.tensor([0, len(ob)], dtype=torch.int64, device=dev)
    of = torch.zeros(nq, dtype=torch.int32, device=dev)
    osh = eng.rrt_plan(obd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes)
    om = eng.rrt_plan_many((obd, off), of, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes)
    torch.cuda.synchronize()
    ts, tm = [], []
    for _ in range(reps):
        ts.append(_events_ms(lambda: eng.rrt_plan(obd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes, **osh), 1))
        tm.append(_events_ms(lambda: eng.rrt_plan_many((obd, off), of, sed, sdd, p, max_pts=max_pts,
                                                       max_nodes=max_nodes, **om), 1))
    gs, gm = host(osh), host(om)
    cell = dict(cell="many_a_demo_one_list", queries=nq, max_iter=p.max_iter, rounds=reps,
                many_ms=float(np.median(tm)), many_ms_min=min(tm), many_ms_max=max(tm), shared_ms=float(np.median(ts)),
                shared_ms_min=min(ts), shared_ms_max=max(ts), many_over_shared=float(np.median(tm) / np.median(ts)),
                many_queries_per_s=nq / (np.median(tm) / 1e3), bit_identical=all(same(gm[k], gs[k]) for k in KEYS))
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)

    # b: 1024 scattered maps, queries shuffled, against one launch per map
    maps = synth.rrt_fleet_obstacles(1024, lo=lo, hi=hi)
    obn, offn = synth.pack_obstacles(maps, 3)
    ofn = np.random.default_rng(0xB).integers(0, len(maps), nq).astype(np.int32)
    se, seed = np.zeros((4, nq), np.float32), np.zeros(nq, np.uint32)
    for s in range(len(maps)):
        sel = np.nonzero(ofn == s)[0]
        se[:, sel], seed[sel] = synth.rrt_inputs(sel.size, maps[s], lo, hi, seed=s)
    obs = (torch.from_numpy(obn).to(dev), torch.from_numpy(offn).to(dev))
    ofd, sed, sdd = (torch.from_numpy(v).to(dev) for v in (ofn, se, seed.view(np.int32)))
    om = eng.rrt_plan_many(obs, ofd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes)
    torch.cuda.synchronize()
    ms = _events_ms(lambda: eng.rrt_plan_many(obs, ofd, sed, sdd, p, max_pts=max_pts, max_nodes=max_nodes, **om), reps)
    gm = host(om)
    per = []
    for s in range(len(maps)):
        sel = np.nonzero(ofn == s)[0]
        if sel.size:
            per.append((sel, torch.from_numpy(maps[s]).to(dev),
                        torch.from_numpy(np.ascontiguousarray(se[:, sel])).to(dev),
                        torch.from_numpy(np.ascontiguousarray(seed[sel]).view(np.int32)).to(dev)))
    outs = [eng.rrt_plan(o, a_, b_, p, max_pts=max_pts, max_nodes=max_nodes) for _, o, a_, b_ in per]   # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    for (_, o, a_, b_), r in zip(per, outs):
        eng.rrt_plan(o, a_, b_, p, max_pts=max_pts, max_nodes=max_nodes, **r)
    torch.cuda.synchronize()
    per_ms = (time.perf_counter() - t) * 1e3
    ok = True
    for (sel, _, _, _), r in zip(per, outs):
        h = host(r)
        ok = ok and all(same(gm[k][..., sel], h[k]) for k in KEYS)
    nodes, iters = int(gm["n_nodes"].astype(np.int64).sum()), int(gm["n_iter"].astype(np.int64).sum())
    cell = dict(cell="many_b_1024_maps_0_64", queries=nq, maps=len(maps), rows=int(offn[-1]), max_iter=p.max_iter,
                many_ms=ms, many_queries_per_s=nq / (ms / 1e3), many_nodes_per_s=nodes / (ms / 1e3),
                many_iterations_per_s=iters / (ms / 1e3), per_map_launches=len(per), per_map_ms=per_ms,
                status_hist=dict(zip(["found", "max_iter_reached", "bad_input", "bad_obstacles"],
                                     np.bincount(gm["status"], minlength=4).tolist())),
                bit_identical=bool(ok))
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cells", choices=("shared", "many", "all"), default="all")
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
    for name, (ob, lo, hi, e) in (maps.items() if a.cells != "many" else ()):
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
    if a.cells != "shared":
        many_cells(eng, res, a.reps)
    eng.close()
    with open(os.path.join(a.out, "rrt_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
