"""Throughput of crb_dwa_control_batched (dwa_control, src/dynamic_window_approach.cpp:148-155) on the GPU, and of
the CPU oracle on every host core in the same run; then crb_dwa_control_many_batched (an obstacle list per robot).
Writes one JSON file.

  python scripts/dwa_bench.py --out DIR [--cells shared|many|all]

Sizes: n in {4096, 65536, 262144} robots x {10 (the demo's), 64} obstacles, the reference's Config.  Each cell is
warmed up, then timed with CUDA events over at least --min-seconds of back-to-back launches.  decisions/s counts
robots per second; rollouts/s counts the samples of every robot's dynamic window, taken from the grid the oracle
computes (the `best` index space: Nv x Ny per robot).

Obstacle list per robot, 2^18 robots, the reference's Config (`many_*` cells):
  a  every robot on the demo's 10 obstacles, through crb_dwa_control_many_batched (one list, ob_of all 0) and through
     crb_dwa_control_batched, alternated in --rounds rounds of back-to-back launches; the median and spread of each
  b  4096 lists of 0 to 64 obstacles (synth.dwa_obstacles-like arenas), robots shuffled over them, against one
     crb_dwa_control_batched launch per list (what a caller without the many entry point does)
  c  a fleet that avoids itself: the robots of synth.dwa_inputs moved by up to 512 m (about 1 robot per m^2), each
     list the demo's obstacles plus the robots within 5 m, nearest first, capped at 256 (synth.dwa_neighbour_obstacles)
Every output of a and b is compared bitwise with the shared-list launches; in c a seeded sample of 4096 robots is
compared with one shared-list launch each.  Needs a CUDA device: there is no CPU fallback."""
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


def _events_ms(fn, reps):
    import torch
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


def _bits(t):
    a = t.cpu().numpy()
    return a.view(np.uint32) if a.dtype == np.float32 else a


def many_cells(eng, res, rounds):
    """The `many_*` cells of the module docstring."""
    import torch
    dev = torch.device("cuda:0")
    n = 1 << 18
    x, u, g = synth.dwa_inputs(n)
    xd, gd, ud0 = (torch.from_numpy(v).to(dev) for v in (x, g, u))
    i32 = lambda: torch.empty(n, dtype=torch.int32, device=dev)  # noqa: E731
    out = lambda: dict(u=ud0.clone(), cost=torch.empty(n, device=dev), best=i32())  # noqa: E731

    def many(o, ob, off, of, status=None):
        return lambda: eng.dwa_control_many(xd, o["u"], gd, (ob, off), of, cost=o["cost"], best=o["best"],
                                            status=status)

    def same(o1, o2):
        return all(np.array_equal(_bits(o1[k]), _bits(o2[k])) for k in ("u", "cost", "best"))

    # a: one list for everyone, both kernels alternated
    ob = torch.from_numpy(synth.DWA_DEMO_OBSTACLES).to(dev)
    off = torch.tensor([0, 10], dtype=torch.int64, device=dev)
    of = torch.zeros(n, dtype=torch.int32, device=dev)
    om, osh = out(), out()
    fm = many(om, ob, off, of)
    fs = lambda: eng.dwa_control(xd, osh["u"], gd, ob, cost=osh["cost"], best=osh["best"])  # noqa: E731
    for f in (fm, fs):
        f()
    torch.cuda.synchronize()
    reps = max(1, int(0.2 / max(_events_ms(fs, 1) / 1e3, 1e-6)))
    tm, ts = [], []
    for _ in range(rounds):
        ts.append(_events_ms(fs, reps))
        tm.append(_events_ms(fm, reps))
    om, osh = out(), out()
    many(om, ob, off, of)()
    eng.dwa_control(xd, osh["u"], gd, ob, cost=osh["cost"], best=osh["best"])
    cell = dict(cell="many_a_demo_one_list", n=n, rounds=rounds, reps=reps, many_ms=float(np.median(tm)),
                many_ms_min=min(tm), many_ms_max=max(tm), shared_ms=float(np.median(ts)), shared_ms_min=min(ts),
                shared_ms_max=max(ts), many_over_shared=float(np.median(tm) / np.median(ts)),
                many_decisions_per_s=n / (np.median(tm) / 1e3), bit_identical=same(om, osh))
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)

    # b: 4096 lists of 0..64 obstacles, robots shuffled, against one shared launch per list
    rng = np.random.default_rng(0xB)
    lists = [synth.dwa_obstacles(int(k), seed=s) for s, k in enumerate(rng.integers(0, 65, 4096))]
    obn, offn = synth.pack_obstacles(lists, 2)
    ofn = rng.integers(0, len(lists), n).astype(np.int32)
    obd, offd, ofd = (torch.from_numpy(v).to(dev) for v in (obn, offn, ofn))
    om = out()
    st = i32()
    fm = many(om, obd, offd, ofd, st)
    fm()
    torch.cuda.synchronize()
    ms = _events_ms(fm, 10)
    om = out()
    many(om, obd, offd, ofd, st)()
    order = np.argsort(ofn, kind="stable")
    bounds = np.searchsorted(ofn[order], np.arange(len(lists) + 1))
    xs, us, gs = (np.ascontiguousarray(v[:, order]) for v in (x, u, g))
    xsd, gsd = torch.from_numpy(xs).to(dev), torch.from_numpy(gs).to(dev)
    lists_d = [torch.from_numpy(o).to(dev) for o in lists]
    osh = dict(u=torch.from_numpy(us).to(dev), cost=torch.empty(n, device=dev), best=i32())
    views = [(slice(int(bounds[s]), int(bounds[s + 1])), s) for s in range(len(lists)) if bounds[s + 1] > bounds[s]]
    per = [(xsd[:, sl].contiguous(), gsd[:, sl].contiguous(), osh["u"][:, sl].contiguous(), s, sl) for sl, s in views]

    def per_list():
        for xl, gl, ul, s, sl in per:
            eng.dwa_control(xl, ul, gl, lists_d[s], cost=osh["cost"][sl], best=osh["best"][sl])
    per_list()
    torch.cuda.synchronize()
    t = time.perf_counter()
    per_list()
    torch.cuda.synchronize()
    per_ms = (time.perf_counter() - t) * 1e3
    for xl, gl, ul, s, sl in per:   # fresh inputs: u is in/out
        ul.copy_(torch.from_numpy(np.ascontiguousarray(us[:, sl])).to(dev))
    per_list()
    torch.cuda.synchronize()
    got_u = torch.empty_like(osh["u"])
    for xl, gl, ul, s, sl in per:
        got_u[:, sl] = ul
    osh["u"] = got_u
    ok = all(np.array_equal(_bits(om[k])[..., order], _bits(osh[k])) for k in ("u", "cost", "best"))
    cell = dict(cell="many_b_4096_lists_0_64", n=n, lists=len(lists), rows=int(offn[-1]), many_ms=ms,
                many_decisions_per_s=n / (ms / 1e3), per_list_launches=len(per), per_list_ms=per_ms,
                bit_identical=bool(ok and (st == 0).all().item()))
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)

    # c: the fleet avoids itself
    xc = x.copy()
    xc[:2] += np.random.default_rng(0xC).uniform(0.0, 512.0, (2, n)).astype(np.float32)
    gc = g + (xc[:2] - x[:2])
    t = time.perf_counter()
    obc, offc = synth.dwa_neighbour_obstacles(xc, synth.DWA_DEMO_OBSTACLES, 5.0, 256)
    build_s = time.perf_counter() - t
    xcd, gcd = torch.from_numpy(xc).to(dev), torch.from_numpy(np.ascontiguousarray(gc)).to(dev)
    obcd, offcd = torch.from_numpy(obc).to(dev), torch.from_numpy(offc).to(dev)
    ofc = torch.arange(n, dtype=torch.int32, device=dev)
    om = out()
    fm = lambda: eng.dwa_control_many(xcd, om["u"], gcd, (obcd, offcd), ofc, cost=om["cost"], best=om["best"],  # noqa
                                      status=st)
    fm()
    torch.cuda.synchronize()
    ms = _events_ms(fm, 10)
    om = out()
    fm()
    torch.cuda.synchronize()
    sample = np.random.default_rng(0xC1).choice(n, 4096, replace=False)
    ok = bool((st == 0).all().item())
    gu, gcst, gb = om["u"].cpu().numpy(), om["cost"].cpu().numpy(), om["best"].cpu().numpy()
    for i in sample:
        ud = torch.from_numpy(np.ascontiguousarray(u[:, i:i + 1])).to(dev)
        cst, bst = torch.empty(1, device=dev), torch.empty(1, dtype=torch.int32, device=dev)
        eng.dwa_control(xcd[:, i:i + 1].contiguous(), ud, gcd[:, i:i + 1].contiguous(),
                        obcd[int(offc[i]):int(offc[i + 1])], cost=cst, best=bst)
        ok = ok and np.array_equal(_bits(ud)[:, 0], gu[:, i].view(np.uint32)) and \
            _bits(cst)[0] == gcst[i:i + 1].view(np.uint32)[0] and int(bst.item()) == int(gb[i])
    lens = np.diff(offc)
    cell = dict(cell="many_c_neighbours_5m_cap_256", n=n, rows=int(offc[-1]), list_rows_mean=float(lens.mean()),
                list_rows_max=int(lens.max()), lists_at_cap=int((lens == 256).sum()), build_seconds=build_s,
                many_ms=ms, many_decisions_per_s=n / (ms / 1e3), checked_robots=len(sample), bit_identical=ok)
    res["cells"].append(cell)
    print(json.dumps(cell), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--cpu-robots", type=int, default=16384)
    ap.add_argument("--cells", choices=("shared", "many", "all"), default="all")
    ap.add_argument("--rounds", type=int, default=10)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dwa_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    p = OD.dwa_params()
    res = dict(gpu=gpu_info(), host_cores=OD.num_threads(), cells=[])
    for k in ((10, 64) if a.cells != "many" else ()):
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
    if a.cells != "shared":
        many_cells(eng, res, a.rounds)
    eng.close()
    with open(os.path.join(a.out, "dwa_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
