"""How far the EKF step sits from what the H100 can do with its access pattern.

Times, alternately and in one process, with 3 rotating buffer sets and 30 launches captured in a CUDA graph as
bench.py does (2^20 agents, 176 algorithmic bytes per update, 184.5 MB per launch):
  (a) the EKF step, crb_ekf_step_batched;
  (b) crb_probe_ekf_pattern: the same 24-load / 20-store SoA layout, access width, launch shape and PDL, trivial arithmetic,
      i.e. the ceiling for this access pattern;
  (c) a plain device copy (torch copy_) of 92.3 MB, i.e. the same 184.5 MB read plus written.
(a) against (b) is the kernel's own cost; (b) against (c) is the cost of the pattern and the launch boundaries.
Prints GB/s and us per launch for each, with the card's name, power limit and SM clocks, and writes the record
to --out (default: a temporary directory).

  python scripts/ekf_ceiling.py [--rounds 3] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 1 << 20
STEPS = 30
BYTES = 176 * N


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return {"error": str(exc)[:120]}
    f = [c.strip() for c in out.split(",")]
    return dict(zip(["name", "power_limit", "sm_clock", "sm_clock_max"], f)) if len(f) == 4 else {"raw": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3, help="timed graph replays per form and round")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ekf_ceiling.json"))
    args = ap.parse_args()

    import torch
    from cpprobotics_b200 import Engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("ekf_ceiling.py measures the GPU: no CUDA device")
    torch.cuda.set_device(0)
    eng = Engine(0)
    dev = torch.device("cuda", 0)
    host = synth.ekf_inputs(N)
    pristine = [torch.from_numpy(a).to(dev) for a in host]
    ekf_sets = [[t.clone() for t in pristine] for _ in range(3)]
    pat_sets = [[t.clone() for t in pristine] for _ in range(3)]
    copy_sets = [(torch.ones(BYTES // 8, device=dev), torch.empty(BYTES // 8, device=dev)) for _ in range(3)]

    forms = {
        "a_ekf_step": lambda k: eng.ekf_estimation(*ekf_sets[k % 3]),
        "b_pattern": lambda k: eng.probe_ekf_pattern(*pat_sets[k % 3]),
        "c_copy": lambda k: copy_sets[k % 3][1].copy_(copy_sets[k % 3][0]),
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

    before = card()
    ms = {name: [] for name in graphs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        for sets in (ekf_sets, pat_sets):   # the same state every round: no drift in the EKF's inputs
            for s in sets:
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
    after = card()
    eng.close()

    res = {}
    for name, ts in ms.items():
        med = statistics.median(ts)
        res[name] = dict(gbs=BYTES * STEPS / (med * 1e-3) / 1e9, us_per_launch=med * 1e3 / STEPS,
                         gbs_min=BYTES * STEPS / (max(ts) * 1e-3) / 1e9,
                         gbs_max=BYTES * STEPS / (min(ts) * 1e-3) / 1e9, samples=len(ts))
    a, b, c = (res[k]["gbs"] for k in ("a_ekf_step", "b_pattern", "c_copy"))
    rec = dict(card_before=before, card_after=after, agents=N, launches_per_graph=STEPS,
               bytes_per_launch=BYTES, forms=res, a_over_b=a / b, b_over_c=b / c, a_over_c=a / c)
    print(f"card: {before}")
    for name, v in res.items():
        print(f"{name:12s} {v['gbs']:7.0f} GB/s  {v['us_per_launch']:6.2f} us/launch  "
              f"[{v['gbs_min']:.0f} .. {v['gbs_max']:.0f}], {v['samples']} graph replays")
    print(f"(a)/(b) {a / b:.3f}   (b)/(c) {b / c:.3f}   (a)/(c) {a / c:.3f}   card after: {after}")
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
