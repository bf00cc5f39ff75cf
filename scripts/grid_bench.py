"""Throughput of the grid planners on the GPU (crb_grid_plan_batched, A* and Dijkstra) against the CPU checker on
every host core, in the same run.  Writes one JSON file.

  python scripts/grid_bench.py --out DIR [--reps 10]

Maps: the demo's walls (60 x 60 cells) and the seeded 128 x 128 scatter (synth.grid_scatter_obstacles(128)), each with
synth.grid_inputs queries; fleets of 2^12 and 2^16 queries.  Each cell is timed with CUDA events over --reps launches
after one warm-up launch (which also allocates the workspace).  Reported: ms per launch, queries/s, visited cells/s
(the sum of n_visited over the launch's queries), the slots (concurrent searches) used, the status counts, the
checker's time for the same queries on every host core and whether the GPU outputs are bit-identical to it, and the
card name and power limit read in the same run.  Needs a CUDA device: there is no CPU fallback.

A map per query (crb_grid_obstacle_map_many, crb_grid_plan_many_batched), cells with "kind":
  mixed_maps     2^16 queries shuffled over 1024 synth.grid_fleet_maps: one many-map launch against one
                 crb_grid_plan_batched launch per map on the same queries, and one many-map build against 1024
                 crb_grid_obstacle_map launches
  local_windows  2^14 robots, each in its own 64 x 64 window of one shared obstacle field (synth.grid_local_windows)
  one_map        2^16 queries all on the demo map through the many-map entry point, beside crb_grid_plan_batched
  slot_cap       the mixed maps with one 1024 x 1024 map among them: max_cells, and so the slot count, is set by it
Each reports ms per launch, queries/s, slots, the status counts, and whether the outputs are bitwise the per-map path
and the checker (oracle/grid_many.py)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, GridBox, grid_map_table, synth  # noqa: E402
from oracle import grid as OG  # noqa: E402
from oracle import grid_many as GM  # noqa: E402


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
    many_cells(eng, dev, a.reps, res)
    eng.close()
    with open(os.path.join(a.out, "grid_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


STATUS = ["found", "no_path", "start_outside", "bad_point", "bad_map"]
KEYS = ("path", "path_len", "cost", "n_visited", "status")


def timed(fn, reps):
    """ms per call of fn over reps calls, after one warm-up call"""
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def many_cells(eng, dev, reps, res):
    """The map-per-query cells (see the module docstring)."""
    import torch
    max_pts = 64

    def d(x):
        return torch.from_numpy(np.ascontiguousarray(x)).to(dev)

    def build(f):
        table = grid_map_table(f["boxes"], f["reso"])
        ob, off = synth.pack_obstacles(f["lists"], 2)
        dt = tuple(d(x) for x in table[:3]) + (table[3],)
        args = ((d(ob), d(off)), d(f["ob_of"]), d(f["rr"]), dt)
        maps = torch.zeros(int(table[2][-1]), dtype=torch.uint8, device=dev)
        ms = timed(lambda: eng.grid_obstacle_map_many(*args, maps=maps), reps)
        return table, dt, (ob, off), maps, ms

    def per_map_maps(f, table, store):
        """crb_grid_obstacle_map once per map: the maps and ms for the whole set of launches"""
        ob, off = store
        dev_lists = [(d(ob[off[s]:off[s + 1], 0]), d(ob[off[s]:off[s + 1], 1])) for s in range(len(off) - 1)]
        out = torch.zeros(int(table[2][-1]), dtype=torch.uint8, device=dev)
        views = [out[table[2][m]:table[2][m + 1]].view(*OG.dims(table[0][m])) for m in range(len(table[1]))]
        boxes = [GridBox(*[int(v) for v in b]) for b in table[0]]

        def run():
            for m in range(len(table[1])):
                x, y = dev_lists[f["ob_of"][m]]
                eng.grid_obstacle_map(x, y, float(table[1][m]), float(f["rr"][m]), boxes[m], map=views[m])
        return out, timed(run, max(1, reps // 3))

    def plan_cell(kind, algo, aname, table, dt, maps_d, map_of, sg, per_map=True, extra=None, n_reps=None):
        n = sg.shape[1]
        n_reps = reps if n_reps is None else n_reps
        maps = maps_d.cpu().numpy()
        sgd, mod = d(sg), d(map_of)
        out = eng.grid_plan_many(algo, dt, maps_d, mod, sgd, max_pts=max_pts)
        ms = timed(lambda: eng.grid_plan_many(algo, dt, maps_d, mod, sgd, max_pts=max_pts, **out), n_reps)
        g = {k: v.cpu().numpy() for k, v in out.items()}
        cell = dict(kind=kind, algo=aname, queries=n, reps=n_reps, maps=len(table[1]), max_cells=int(table[3]),
                    slots=eng.grid_plan_many_slots(algo, table[3], n), many_ms=ms, many_queries_per_s=n / (ms / 1e3),
                    status_hist=dict(zip(STATUS, np.bincount(g["status"], minlength=5).tolist())))
        if per_map:
            # one crb_grid_plan_batched per map on its own queries, gathered beforehand
            order = np.argsort(map_of, kind="stable")
            cuts = np.searchsorted(map_of[order], np.arange(len(table[1]) + 1))
            jobs = []
            for m in range(len(table[1])):
                sel = order[cuts[m]:cuts[m + 1]]
                if sel.size == 0:
                    continue
                W, H = OG.dims(table[0][m])
                o = dict(path=torch.full((2 * max_pts, sel.size), float("nan"), device=dev),
                         path_len=torch.empty(sel.size, dtype=torch.int32, device=dev),
                         cost=torch.empty(sel.size, device=dev),
                         n_visited=torch.empty(sel.size, dtype=torch.int32, device=dev),
                         status=torch.empty(sel.size, dtype=torch.int32, device=dev))
                jobs.append((sel, GridBox(*[int(v) for v in table[0][m]]),
                             maps_d[table[2][m]:table[2][m + 1]].view(W, H), float(table[1][m]), d(sg[:, sel]), o))

            def run():
                for _, box, mp, r, s_, o in jobs:
                    eng.grid_plan(algo, box, mp, r, s_, max_pts=max_pts, **o)
            pm = timed(run, max(1, reps // 3))
            ref = {k: np.zeros_like(g[k]) for k in KEYS}
            for sel, *_, o in jobs:
                for k in KEYS:
                    ref[k][..., sel] = o[k].cpu().numpy()
            cell.update(per_map_launches=len(jobs), per_map_ms=pm, per_map_queries_per_s=n / (pm / 1e3),
                        per_map_over_many=pm / ms, bit_identical_per_map=all(same(g[k], ref[k]) for k in KEYS))
        if extra:
            cell.update(extra)
        t = time.perf_counter()
        o = GM.plan_many(algo, *table[:3], maps, table[3], map_of, sg, max_pts=max_pts)
        cell["cpu_seconds"] = time.perf_counter() - t
        cell["bit_identical_checker"] = all(same(g[k], o[k]) for k in KEYS)
        cell["bit_identical"] = cell["bit_identical_checker"] and cell.get("bit_identical_per_map", True)
        res["cells"].append(cell)
        print(json.dumps(cell), flush=True)

    algos = ((OG.ASTAR, "astar"), (OG.DIJKSTRA, "dijkstra"))
    # mixed maps
    f = synth.grid_fleet_maps(1024)
    table, dt, store, maps_d, build_ms = build(f)
    one_maps, per_build_ms = per_map_maps(f, table, store)
    want, _ = GM.obstacle_map_many(*store, f["ob_of"], f["rr"], *table[:3], int(table[2][-1]), table[3])
    got = maps_d.cpu().numpy()
    bcell = dict(kind="mixed_maps_build", maps=1024, cells=int(table[2][-1]), many_ms=build_ms,
                 per_map_launches=1024, per_map_ms=per_build_ms, per_map_over_many=per_build_ms / build_ms,
                 bit_identical=same(got, one_maps.cpu().numpy()) and same(got, want))
    res["cells"].append(bcell)
    print(json.dumps(bcell), flush=True)
    map_of, sg = synth.grid_fleet_inputs(1 << 16, table[0], table[1], got, table[2])
    for algo, aname in algos:
        plan_cell("mixed_maps", algo, aname, table, dt, maps_d, map_of, sg)
    # local windows
    w = synth.grid_local_windows(1 << 14)
    tw, dtw, _, mw_d, wbuild_ms = build(w)
    mw = mw_d.cpu().numpy()
    sgw = np.concatenate([synth.grid_inputs(1, tw[0][m], mw[tw[2][m]:tw[2][m + 1]].reshape(64, 64), 1.0, seed=m)
                          for m in range(1 << 14)], axis=1)
    for algo, aname in algos:
        plan_cell("local_windows", algo, aname, tw, dtw, mw_d, np.arange(1 << 14, dtype=np.int32), sgw,
                  per_map=False, extra=dict(build_ms=wbuild_ms))
    # one map: the demo map through both entry points
    ox, oy = synth.grid_demo_obstacles()
    gd = synth.GRID_DEMO
    gb = OG.box_of_obstacles(ox, oy, gd["reso"])
    one = dict(lists=[np.ascontiguousarray(np.stack([ox, oy], 1))], ob_of=np.int32([0]), boxes=gb[None],
               reso=np.float32([gd["reso"]]), rr=np.float32([gd["rr"]]))
    to, dto, _, mo_d, _ = build(one)
    sgo = synth.grid_inputs(1 << 16, gb, mo_d.cpu().numpy().reshape(*OG.dims(gb)), gd["reso"])
    for algo, aname in algos:
        plan_cell("one_map", algo, aname, to, dto, mo_d, np.zeros(1 << 16, np.int32), sgo)

    # slot cap: the same maps and one 1024 x 1024 map among them
    fx = synth.grid_fleet_maps(1023)
    bx, by = synth.grid_scatter_obstacles(1024)
    fx["lists"].append(np.ascontiguousarray(np.stack([bx, by], 1)))
    fx["ob_of"] = np.append(fx["ob_of"], len(fx["lists"]) - 1).astype(np.int32)
    fx["boxes"] = np.concatenate([fx["boxes"], np.int32([[0, 0, 1024, 1024]])])
    fx["reso"] = np.append(fx["reso"], np.float32(1.0)).astype(np.float32)
    fx["rr"] = np.append(fx["rr"], np.float32(1.0)).astype(np.float32)
    tx, dtx, _, mx_d, _ = build(fx)
    mof, sgx = synth.grid_fleet_inputs(1 << 16, tx[0], tx[1], mx_d.cpu().numpy(), tx[2])
    for algo, aname in algos:
        # a search on the large map takes seconds, so one timed launch and no per-map comparison
        plan_cell("slot_cap", algo, aname, tx, dtx, mx_d, mof, sgx, per_map=False, n_reps=1,
                  extra=dict(slots_without_large_map=eng.grid_plan_many_slots(algo, table[3], 1 << 16),
                             queries_on_large_map=int((mof == 1023).sum())))


if __name__ == "__main__":
    main()
