"""Throughput of the fleet particle filter (crb_pf_step_many_batched) on the GPU.  Writes one JSON file.

  python scripts/pf_fleet_bench.py --out DIR [--reps 20]

Cells: 2^14, 2^16 and 2^18 robots x np = 100 with the demo's lists (synth.pf_fleet_inputs: the tags of the four RFID
marks within 20 m, 1 to 4 rows) and with 16-row lists, and 2^22 particles as 2^12 x 1024, 2^11 x 2048, 2^10 x 4096 and
2^9 x 8192 (demo lists): above np = 1157 fewer than 8 robots (warps) fit a CTA, at 8192 one.  Each cell is timed
with CUDA events over --reps ping-pong steps after two warm-up steps, with noise and uniforms drawn in the kernel.
Beside each cell:
  per_robot    one crb_pf_step per robot, the fleet's only route without this entry point: timed over a sample of
               64 robots and scaled to the fleet;
  one_filter   crb_pf_step on ONE filter of the same total particle count, as particles/s.
Reported: ms per step, particles/s, achieved bytes/s from the algorithmic bytes per particle (px read and written, 16
+ 16, pw read and written, 4 + 4, px_next written, 16: 56 bytes, plus the robot's observation rows, u and its result
column once per robot), and
the card name and power limit read in the same run.  Needs a CUDA device: there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, pf_default_params, synth  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def timed(torch, fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def fleet_cell(torch, eng, nr, npr, rows, reps):
    f = synth.pf_fleet_inputs(nr, npr, seed=nr + npr + (4 if rows == "demo" else int(rows)))
    if rows != "demo":
        lm = synth.pf_landmarks(int(rows), seed=7)
        f["z"], f["z_off"] = synth.pack_obstacles([lm], 3)
        f["z_of"][:] = 0
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    st = dict(x=d(f["px"]), xn=torch.empty(4, nr * npr, device="cuda"), t=0)
    w, u, z, zo, zof = d(f["pw"]), d(f["u"]), d(f["z"]), d(f["z_off"]), d(f["z_of"])
    res = torch.empty(24, nr, dtype=torch.float64, device="cuda")

    def step():
        st["t"] += 1
        eng.pf_step_many(npr, st["x"], w, st["xn"], u, (z, zo), zof, seed=st["t"], resample_seed=st["t"], result=res)
        st["x"], st["xn"] = st["xn"], st["x"]

    ms = timed(torch, step, reps)
    n = nr * npr
    nrows = int(f["z_off"][-1]) if rows == "demo" else int(rows) * nr
    byts = 56 * n + 12 * nrows + nr * (8 + 8 + 4 + 24 * 8)
    resampled = int(res[22].sum().item())

    # one crb_pf_step per robot on a sample of 64 robots, scaled
    k = 64
    sx = [d(f["px"][:, r * npr:(r + 1) * npr]) for r in range(k)]
    sw = [d(f["pw"][r * npr:(r + 1) * npr]) for r in range(k)]
    sn = [torch.empty(4, npr, device="cuda") for _ in range(k)]
    sres = torch.empty(24, dtype=torch.float64, device="cuda")
    lists = [f["z"][f["z_off"][f["z_of"][r]]:f["z_off"][f["z_of"][r] + 1]] for r in range(k)]
    prms = []
    for r in range(k):
        p = pf_default_params()
        p.u[0], p.u[1] = float(f["u"][0, r]), float(f["u"][1, r])
        prms.append(p)

    def per_robot():
        for r in range(k):
            eng.pf_step(sx[r], sw[r], sn[r], None, lists[r], params=prms[r], seed=r, resample_seed=r, result=sres)

    ms_per = timed(torch, per_robot, max(2, reps // 4)) * nr / k

    # one filter of the same particle count
    one = synth.pf_inputs(n)
    ox, ow, on = d(one[0]), d(one[1]), torch.empty(4, n, device="cuda")
    lm = lists[0]
    ost = dict(x=ox, xn=on, t=0)

    def one_filter():
        ost["t"] += 1
        eng.pf_step(ost["x"], ow, ost["xn"], None, lm, seed=ost["t"], resample_seed=ost["t"], result=sres)
        ost["x"], ost["xn"] = ost["xn"], ost["x"]

    ms_one = timed(torch, one_filter, reps)
    return dict(robots=nr, np=npr, rows=rows, ms=ms, particles_per_s=n / (ms * 1e-3),
                gbytes_per_s=byts / (ms * 1e-3) / 1e9, resampled_last_step=resampled,
                per_robot_ms_scaled=ms_per, speedup_vs_per_robot=ms_per / ms,
                one_filter_ms=ms_one, one_filter_particles_per_s=n / (ms_one * 1e-3),
                ratio_vs_one_filter=(n / (ms * 1e-3)) / (n / (ms_one * 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    eng = Engine(0)
    cells = []
    for nr in (1 << 14, 1 << 16, 1 << 18):
        for rows in ("demo", 16):
            cells.append(fleet_cell(torch, eng, nr, 100, rows, a.reps))
            print(json.dumps(cells[-1]))
    for npr in (1024, 2048, 4096, 8192):
        cells.append(fleet_cell(torch, eng, (1 << 22) // npr, npr, "demo", a.reps))
        print(json.dumps(cells[-1]))
    out = dict(gpu=gpu_info(), cells=cells)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "pf_fleet_bench.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(out["gpu"]))
    eng.close()


if __name__ == "__main__":
    main()
