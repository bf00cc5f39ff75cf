"""Throughput of LQR path tracking on the GPU (crb_lqr_steering_control_batched, both programs) against the CPU checker
on every host core, in the same run.  Writes one JSON file.

  python scripts/lqr_track_bench.py --out DIR [--reps 20]

Cells: nx 4 (lqr_steer_control) and 5 (lqr_speed_steer_control); fleets of 2^16 and 2^20 vehicles; the demo-shaped
course (synth.lqr_course("demo"), ~430 points) and an 8192-point course (the sine course resampled); vehicles from
synth.lqr_track_inputs at their mixed speeds ("demo speeds") or all stopped (v = 0: solve_DARE runs its 150 iterations,
the worst case).  Each cell is timed with CUDA events over --reps launches after one warm-up launch.  Reported per cell:
ms per launch, calls/s, the mean and max DARE iterations, the same launch on a 1-point course (the DARE without the
scan), achieved FP32 FLOP/s with the flops counted from the executed iterations and the course length, against
crb_probe_fp32_peak measured in the same run, the checker's calls/s on every host core (on 2^16 vehicles) and whether
the GPU outputs are bit-identical to it.

Many-course cells (crb_lqr_steering_control_many_batched, a course per vehicle), both nx, 2^16 and 2^20 vehicles at the
demo speeds: "one_course" (every vehicle on the demo-shaped course, timed next to the shared-course entry point on the
same inputs), "4096x430" (4096 demo-length courses, the demo course rotated and moved) and "64x8192" (64 courses of the
8192-point course, rotated and moved), vehicles shuffled across the courses.  Reported per cell: ms per launch and
calls/s, the same fleet as one shared-course launch per course (the host loop a caller would otherwise write), and
whether the outputs are bitwise those per-course launches.  Then the MPC lookup
(crb_mpc_calc_ref_trajectory_many_batched, T = 20) at 2^20 agents on the 4096 courses, next to the single-course lookup
on one course.

The card's name and power limit are read in the same run.  Needs a CUDA device: there is no CPU fallback."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, synth  # noqa: E402
from oracle import lqrt as OL  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def mm(ra, ca, cb):
    return ra * cb * (2 * ca - 1)


def dare_flops(nx):
    """FP32 operations of one solve_DARE iteration as crb_lqr_dare.cuh executes it (products, the inverse or the
    division, Xn and the error)."""
    nu = 1 if nx == 4 else 2
    f = 4 * mm(nx, nx, nx) + mm(nx, nx, nu) + mm(nu, nx, nx) + mm(nu, nx, nu) + mm(nx, nu, nx) + 3 * nx * nx
    f += (1 + nx) if nu == 1 else (4 + 3 + 1 + 4 + mm(nx, 2, 2))
    return f


def tail_flops(nx):
    nu = 1 if nx == 4 else 2
    return mm(nu, nx, nx) + mm(nu, nx, nu) + mm(nu, nx, nx) + (2 * nx if nu == 1 else 12 + mm(2, 2, nx)) + 2 * nu * nx


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def moved(course, rng):
    """course rotated by a random angle (cyaw turns with it) and moved by up to 500 m."""
    th = rng.uniform(-np.pi, np.pi)
    tx, ty = rng.uniform(-500.0, 500.0, 2)
    x, y = course[0].astype(np.float64), course[1].astype(np.float64)
    return tuple(np.ascontiguousarray(v, np.float32) for v in (
        np.cos(th) * x - np.sin(th) * y + tx, np.sin(th) * x + np.cos(th) * y + ty,
        course[2].astype(np.float64) + th, course[3], course[4]))


def event_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(torch.cuda.current_stream())
    for _ in range(reps):
        fn()
    e1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def many_courses(a, eng, res, dev, base):
    """The many-course cells (see the module docstring)."""
    import torch
    rng = np.random.default_rng(0x4A7)
    sets = {"one_course": [base["demo"]],
            "4096x430": [moved(base["demo"], rng) for _ in range(4096)],
            "64x8192": [moved(base["course8192"], rng) for _ in range(64)]}
    res["many_cells"] = []
    for cname, courses in sets.items():
        packed = synth.pack_courses(courses)
        dpk = [torch.from_numpy(x).to(dev) for x in packed]
        dsingle = [[torch.from_numpy(x).to(dev) for x in c] for c in courses]
        for nx in (4, 5):
            nu = 1 if nx == 4 else 2
            dcs = dpk[:4] + dpk[5:] if nx == 4 else dpk
            for log2n in (16, 20):
                n = 1 << log2n
                course_of = rng.integers(0, len(courses), n).astype(np.int32)
                st = np.zeros((4, n), np.float32)
                ind, pe, pth = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.float32)
                groups = [np.nonzero(course_of == c)[0] for c in range(len(courses))]
                for c, sel in enumerate(groups):
                    if sel.size:
                        st[:, sel], ind[sel], pe[sel], pth[sel] = synth.lqr_track_inputs(sel.size, courses[c],
                                                                                         seed=log2n * 10007 + c)
                dst, dof = torch.from_numpy(st).to(dev), torch.from_numpy(course_of).to(dev)
                dind, dpe, dpth = (torch.from_numpy(x.copy()).to(dev) for x in (ind, pe, pth))
                u = torch.empty((nu, n), dtype=torch.float32, device=dev)
                it = torch.empty(n, dtype=torch.int32, device=dev)
                stt = torch.empty(n, dtype=torch.int32, device=dev)
                # the scan and the DARE depend on x only; ind, pe, pth_e are replaced by every call
                ms = event_ms(lambda: eng.lqr_steering_control_many(nx, dst, dcs, dof, dind, dpe, dpth, u=u, iters=it,
                                                                    status=stt), a.reps)
                # the same fleet, one shared-course launch per course on that course's vehicles (gathered beforehand)
                per = []
                for c, sel in enumerate(groups):
                    if sel.size:
                        ts = [torch.from_numpy(np.ascontiguousarray(x)).to(dev)
                              for x in (st[:, sel], ind[sel], pe[sel], pth[sel])]
                        per.append((c, sel, ts, torch.empty((nu, sel.size), dtype=torch.float32, device=dev),
                                    torch.empty(sel.size, dtype=torch.int32, device=dev),
                                    torch.empty(sel.size, dtype=torch.int32, device=dev)))

                def per_course():
                    for c, sel, ts, pu, pit, pst in per:
                        eng.lqr_steering_control(nx, ts[0], dsingle[c][: 4 if nx == 4 else 5], ts[1], ts[2], ts[3],
                                                 u=pu, iters=pit, status=pst)
                ms_per = event_ms(per_course, max(1, a.reps // 5))
                # bitwise: one fresh call of each on the original inputs
                dind, dpe, dpth = (torch.from_numpy(x.copy()).to(dev) for x in (ind, pe, pth))
                eng.lqr_steering_control_many(nx, dst, dcs, dof, dind, dpe, dpth, u=u, iters=it, status=stt)
                for c, sel, ts, pu, pit, pst in per:
                    for t, x in zip(ts[1:], (ind[sel], pe[sel], pth[sel])):
                        t.copy_(torch.from_numpy(x))
                per_course()
                torch.cuda.synchronize()
                got = [x.cpu().numpy() for x in (u, dind, dpe, dpth, it, stt)]
                want = [np.zeros_like(x) for x in got]
                for c, sel, ts, pu, pit, pst in per:
                    for w, x in zip(want, (pu, ts[1], ts[2], ts[3], pit, pst)):
                        w[..., sel] = x.cpu().numpy()
                cell = dict(nx=nx, courses=cname, n_courses=len(courses), points=int(packed[0].size), n=n, ms=ms,
                            calls_per_s=n / (ms * 1e-3), ms_launch_per_course=ms_per,
                            launches_per_course=len(per),
                            bit_identical_to_per_course=bool(all(same(g, w) for g, w in zip(got, want))))
                if cname == "one_course":
                    ms1 = event_ms(lambda: eng.lqr_steering_control(nx, dst, dsingle[0][: 4 if nx == 4 else 5], dind,
                                                                    dpe, dpth, u=u, iters=it, status=stt), a.reps)
                    cell.update(ms_shared_course_kernel=ms1, shared_course_calls_per_s=n / (ms1 * 1e-3))
                res["many_cells"].append(cell)
                print(json.dumps(cell), flush=True)
    # the MPC lookup at 2^20 agents on the 4096 courses, next to the single-course lookup on the demo course
    T, n = 20, 1 << 20
    courses = sets["4096x430"]
    packed = synth.pack_courses(courses)
    dpk = [torch.from_numpy(x).to(dev) for x in packed]
    course_of = rng.integers(0, len(courses), n).astype(np.int32)
    lens = np.diff(packed[5])
    local = rng.integers(0, lens[course_of]).astype(np.int32)
    gidx = packed[5][course_of] + local
    st = np.stack([packed[0][gidx] + rng.uniform(-1, 1, n), packed[1][gidx] + rng.uniform(-1, 1, n),
                   packed[2][gidx], rng.uniform(0, 5, n)]).astype(np.float32)
    dst, dof = torch.from_numpy(st).to(dev), torch.from_numpy(course_of).to(dev)
    ti0 = torch.from_numpy(np.maximum(local - 3, 0).astype(np.int32)).to(dev)
    dti = ti0.clone()
    xr = torch.empty((4 * T, n), dtype=torch.float32, device=dev)
    stt = torch.empty(n, dtype=torch.int32, device=dev)

    def many():
        dti.copy_(ti0)
        eng.calc_ref_trajectory_many(dst, (dpk[0], dpk[1], dpk[2], dpk[4], dpk[5]), dof, 1.0, dti, xr, T, status=stt)
    d1 = [torch.from_numpy(x).to(dev) for x in base["demo"]]
    st1 = st.copy()
    st1[:2] -= packed[0][gidx] - base["demo"][0][local], packed[1][gidx] - base["demo"][1][local]
    dst1 = torch.from_numpy(np.ascontiguousarray(st1)).to(dev)

    def single():
        dti.copy_(ti0)
        eng.calc_ref_trajectory(dst1, d1[0], d1[1], d1[2], d1[4], 1.0, dti, xr, T)
    copy_ms = event_ms(lambda: dti.copy_(ti0), a.reps)
    ms_many, ms_single = event_ms(many, a.reps) - copy_ms, event_ms(single, a.reps) - copy_ms
    cell = dict(kernel="mpc_lookup", T=T, n=n, n_courses=len(courses), ms=ms_many, calls_per_s=n / (ms_many * 1e-3),
                ms_single_course=ms_single, single_course_calls_per_s=n / (ms_single * 1e-3))
    res["mpc_lookup"] = cell
    print(json.dumps(cell), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lqr_track_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    peak = C.c_double(0.0)
    eng.lib.crb_probe_fp32_peak(eng.ctx, C.byref(peak))
    res = dict(gpu=gpu_info(), host_cores=OL.num_threads(), reps=a.reps, fp32_peak_tflops=peak.value, cells=[])
    sine = synth.lqr_course("sine", ds=60.0 / 8192)
    courses = {"demo": synth.lqr_course("demo"), "course8192": tuple(x[:8192] for x in sine)}
    one = tuple(x[:1] for x in courses["demo"])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(nx, dst, dcourse, dind, dpe, dpth, u, it, stt):
        def launch():
            eng.lqr_steering_control(nx, dst, dcourse, dind, dpe, dpth, u=u, iters=it, status=stt)
        launch()
        torch.cuda.synchronize()
        ev0.record(torch.cuda.current_stream())
        for _ in range(a.reps):
            launch()
        ev1.record(torch.cuda.current_stream())
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / a.reps

    for nx in (4, 5):
        nu = 1 if nx == 4 else 2
        for cname, course in courses.items():
            dcourse = [torch.from_numpy(x).to(dev) for x in course][: 4 if nx == 4 else 5]
            d1 = [torch.from_numpy(x).to(dev) for x in one][: 4 if nx == 4 else 5]
            for log2n in (16, 20):
                n = 1 << log2n
                for speeds in ("demo", "stopped"):
                    st, ind, pe, pth = synth.lqr_track_inputs(n, course, seed=log2n)
                    if speeds == "stopped":
                        st[3] = 0.0
                    dst = torch.from_numpy(st).to(dev)
                    # ind, pe, pth_e are replaced by every call; the timed launches start from the same inputs as
                    # the first (the scan and the DARE do not depend on them, only x does)
                    dind, dpe, dpth = (torch.from_numpy(x.copy()).to(dev) for x in (ind, pe, pth))
                    u = torch.empty((nu, n), dtype=torch.float32, device=dev)
                    it = torch.empty(n, dtype=torch.int32, device=dev)
                    stt = torch.empty(n, dtype=torch.int32, device=dev)
                    ms = timed(nx, dst, dcourse, dind, dpe, dpth, u, it, stt)
                    iters = it.cpu().numpy()
                    ms1 = timed(nx, dst, d1, dind.zero_(), dpe, dpth, u, it, stt)
                    flops = float(iters.astype(np.float64).sum()) * dare_flops(nx) + n * tail_flops(nx) \
                        + 5.0 * n * len(course[0])
                    cell = dict(nx=nx, course=cname, ncourse=len(course[0]), n=n, speeds=speeds, ms=ms,
                                calls_per_s=n / (ms * 1e-3), dare_iters_mean=float(iters.mean()),
                                dare_iters_max=int(iters.max()), ms_one_point_course=ms1,
                                achieved_tflops=flops / (ms * 1e-3) / 1e12,
                                fraction_of_fp32_peak=flops / (ms * 1e-3) / 1e12 / peak.value if peak.value else None)
                    if log2n == 16:
                        dind2, dpe2, dpth2 = (torch.from_numpy(x.copy()).to(dev) for x in (ind, pe, pth))
                        r = eng.lqr_steering_control(nx, dst, dcourse, dind2, dpe2, dpth2)
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        o = OL.control(nx, st, course, ind, pe, pth)
                        tc = time.perf_counter() - t0
                        cell.update(checker_s=tc, checker_calls_per_s=n / tc, speedup_vs_checker=tc / (ms * 1e-3),
                                    bit_identical=bool(all(same(g.cpu().numpy(), o[k]) for g, k in (
                                        (r["u"], "u"), (dind2, "ind"), (dpe2, "pe"), (dpth2, "pth_e"),
                                        (r["iters"], "iters"), (r["status"], "status")))))
                    res["cells"].append(cell)
                    print(json.dumps(cell), flush=True)
    many_courses(a, eng, res, dev, courses)
    eng.close()
    path = os.path.join(a.out, "lqr_track_bench.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
