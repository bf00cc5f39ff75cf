"""What a noise model per agent costs the EKF step, and what it saves a fleet that mixes sensors.

Times, alternately and in one process, with 3 rotating buffer sets and 30 launches captured in a CUDA graph as
scripts/ekf_ceiling.py does, at 2^20 and 2^24 agents:
  baseline     crb_ekf_step_batched, one model for the whole batch;
  many_1       crb_ekf_step_many_batched with a one-model table;
  many_8       8 models, agents shuffled over them;
  many_4096    4096 models, shuffled;
  many_n       one model per agent (a shuffled permutation);
  gather_8     what a caller does without the model table for 8 classes: per class, gather its agents (torch
               index_select), one crb_ekf_step_batched, scatter back (index_copy_), timed end to end;
and, at 2^20 agents with pinned z / u, 50 ticks of the resident track: crb_ekf_track_step against
crb_ekf_track_step_many with 8 models (x_out every tick, async, two host buffers in rotation).
G updates/s and TB/s per form; the byte count is algorithmic: 176 B per update for the baseline and gather_8 (the
filter's own traffic; gather_8's index passes come on top), 180 B for the model-table forms (the 4-byte index), 268 B
for many_n (its 88-byte record too).  Prints the card's name and power limit read in the same run, and one JSON record
as the last line, also written to --out (default: a temporary directory).

  python scripts/ekf_many_bench.py [--rounds 5] [--reps 3] [--sizes 20,24] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS = 30
TRACK_N = 1 << 20
TRACK_TICKS = 50
BYTES = {"baseline": 176, "many_1": 180, "many_8": 180, "many_4096": 180, "many_n": 268, "gather_8": 176}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return {"error": str(exc)[:120]}
    f = [c.strip() for c in out.split(",")]
    return dict(zip(["name", "power_limit", "sm_clock", "sm_clock_max"], f)) if len(f) == 4 else {"raw": out}


def model_of(torch, n, m, dev, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randperm(n, generator=g) % m
    return ids.to(torch.int32).to(dev)


def graph_forms(args, torch, eng, n):
    import numpy as np
    from cpprobotics_b200 import ekf_models, synth
    dev = torch.device("cuda", 0)
    f = synth.ekf_fleet_inputs(min(n, 4096), 4096, seed=0xBE)
    host = synth.ekf_inputs(n, seed=0xBE)
    pristine = [torch.from_numpy(a).to(dev) for a in host]
    sets = [[t.clone() for t in pristine] for _ in range(3)]

    def table(m):
        k = np.arange(m) % f["dt"].size
        return torch.from_numpy(ekf_models(f["dt"][k], f["Q"][k], f["R"][k])).to(dev)
    tabs = {m: (table(m), model_of(torch, n, m, dev, m)) for m in (1, 8, 4096, n)}
    # gather / scatter by class: per class its sorted agent indices and gather buffers
    cls = tabs[8][1].long()
    groups = []
    for c in range(8):
        idx = torch.nonzero(cls == c).flatten()
        groups.append((idx, [torch.empty((t.shape[0], idx.numel()), device=dev) for t in pristine]))
    prm = [None] * 8   # the class's params: the same records as the table, as EkfParams
    from cpprobotics_b200 import EkfParams
    for c in range(8):
        p = EkfParams()
        p.dt = float(f["dt"][c])
        p.Q[:] = [float(v) for v in f["Q"][c]]
        p.R[:] = [float(v) for v in f["R"][c]]
        prm[c] = p

    def gather(k):
        x, P, z, u = sets[k % 3]
        for (idx, b), p in zip(groups, prm):
            for src, dst in zip((x, P, z, u), b):
                torch.index_select(src, 1, idx, out=dst)
            eng.ekf_estimation(*b, params=p)
            x.index_copy_(1, idx, b[0])
            P.index_copy_(1, idx, b[1])

    forms = {
        "baseline": lambda k: eng.ekf_estimation(*sets[k % 3]),
        "many_1": lambda k: eng.ekf_estimation_many(*sets[k % 3], *tabs[1]),
        "many_8": lambda k: eng.ekf_estimation_many(*sets[k % 3], *tabs[8]),
        "many_4096": lambda k: eng.ekf_estimation_many(*sets[k % 3], *tabs[4096]),
        "many_n": lambda k: eng.ekf_estimation_many(*sets[k % 3], *tabs[n]),
        "gather_8": gather,
    }
    graphs = {}
    for name, step in forms.items():
        for k in range(3):        # warm up outside the capture
            step(k)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            eng.bind_current_stream()
            for k in range(STEPS):
                step(k)
        eng.bind_current_stream()
        g.replay()
        graphs[name] = g
    torch.cuda.synchronize()
    ms = {name: [] for name in graphs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        for s in sets:   # the same state every round: no drift in the filters' inputs
            for t, p in zip(s, pristine):
                t.copy_(p)
        order = list(graphs) if r % 2 == 0 else list(reversed(list(graphs)))
        for name in order:
            graphs[name].replay()
            for _ in range(args.reps):
                torch.cuda.synchronize()
                e0.record()
                graphs[name].replay()
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1))
    res = {}
    for name, ts in ms.items():
        med = statistics.median(ts)
        ups = n * STEPS / (med * 1e-3)
        res[name] = dict(gups=ups / 1e9, tbs=ups * BYTES[name] / 1e12, us_per_launch=med * 1e3 / STEPS,
                         gups_min=n * STEPS / (max(ts) * 1e-3) / 1e9, gups_max=n * STEPS / (min(ts) * 1e-3) / 1e9,
                         bytes_per_update=BYTES[name], samples=len(ts))
    base = res["baseline"]["gups"]
    for v in res.values():
        v["vs_baseline"] = v["gups"] / base
    del graphs, sets, tabs, groups
    torch.cuda.empty_cache()
    return res


def track_forms(args, torch, eng):
    from cpprobotics_b200 import ekf_models, synth
    dev = torch.device("cuda", 0)
    n = TRACK_N
    f = synth.ekf_fleet_inputs(n, 8, seed=0xBF, n_steps=2)
    tab = torch.from_numpy(ekf_models(f["dt"], f["Q"], f["R"])).to(dev)
    mof = torch.from_numpy(f["model_of"]).to(dev)
    z = [torch.from_numpy(f["z"][2 * k:2 * k + 2].copy()).pin_memory() for k in range(2)]
    u = [torch.from_numpy(f["u"][2 * k:2 * k + 2].copy()).pin_memory() for k in range(2)]
    out = [torch.empty((4, n)).pin_memory() for _ in range(2)]
    torch.cuda.synchronize()
    trk = {"track_step": eng.ekf_track_open(f["x"], f["P"]), "track_step_many": eng.ekf_track_open(f["x"], f["P"])}
    steps = {"track_step": lambda t, k: eng.ekf_track_step(t, z[k % 2], u[k % 2], x_out=out[k % 2], async_=True),
             "track_step_many": lambda t, k: eng.ekf_track_step_many(t, z[k % 2], u[k % 2], tab, mof,
                                                                     x_out=out[k % 2], async_=True)}
    ms = {name: [] for name in steps}
    try:
        for name in steps:   # warm-up
            for k in range(4):
                steps[name](trk[name], k)
            eng.ekf_track_sync(trk[name])
        for r in range(args.rounds):
            order = list(steps) if r % 2 == 0 else list(reversed(list(steps)))
            for name in order:
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    for k in range(TRACK_TICKS):
                        steps[name](trk[name], k)
                    eng.ekf_track_sync(trk[name])
                    ms[name].append((time.perf_counter() - t0) * 1e3)
    finally:
        for t in trk.values():
            eng.ekf_track_close(t)
    res = {}
    for name, ts in ms.items():
        med = statistics.median(ts)
        res[name] = dict(gups=n * TRACK_TICKS / (med * 1e-3) / 1e9, us_per_tick=med * 1e3 / TRACK_TICKS,
                         us_per_tick_min=min(ts) * 1e3 / TRACK_TICKS, us_per_tick_max=max(ts) * 1e3 / TRACK_TICKS,
                         samples=len(ts))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="timed graph replays (track: timed 50-tick runs) per form and "
                                                         "round")
    ap.add_argument("--sizes", default="20,24", help="log2 of the agent counts")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ekf_many_bench.json"))
    args = ap.parse_args()

    import torch
    from cpprobotics_b200 import Engine
    if not torch.cuda.is_available():
        raise SystemExit("ekf_many_bench.py measures the GPU: no CUDA device")
    torch.cuda.set_device(0)
    eng = Engine(0)
    before = card()
    rec = dict(card_before=before, launches_per_graph=STEPS, rounds=args.rounds, reps=args.reps, sizes={})
    for lg in (int(s) for s in args.sizes.split(",")):
        res = graph_forms(args, torch, eng, 1 << lg)
        rec["sizes"][f"2^{lg}"] = res
        for name, v in res.items():
            print(f"2^{lg} {name:10s} {v['gups']:6.2f} G updates/s  {v['tbs']:5.2f} TB/s  "
                  f"{v['us_per_launch']:8.1f} us/launch  [{v['gups_min']:.2f} .. {v['gups_max']:.2f}]  "
                  f"x{v['vs_baseline']:.3f} of baseline", flush=True)
    rec["track_2^20_pinned"] = track_forms(args, torch, eng)
    for name, v in rec["track_2^20_pinned"].items():
        print(f"track 2^20 {name:16s} {v['gups']:6.3f} G updates/s  {v['us_per_tick']:7.1f} us/tick  "
              f"[{v['us_per_tick_min']:.1f} .. {v['us_per_tick_max']:.1f}]", flush=True)
    rec["card_after"] = card()
    eng.close()
    print(f"card: {before}  after: {rec['card_after']}")
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
