"""Throughput of the state lattice planner on the GPU: the biased sampler (crb_slp_sample_states_batched), the
lookup-table search (crb_slp_search_nearest_batched) and the optimizer (crb_mptg_optimize_batched) for fleets of
queries, and of the CPU checker on every host core in the same run.  Writes one JSON file.

  python scripts/slp_bench.py --out DIR

Each query is one robot's planning step: the demo's biased sampler (nxy 30, nh 2, ns 100, d 20: 58 states per
query), each state seeded from synth.slp_table(24) and optimised with the planner's settings.  Fleets of 2^12, 2^14
and 2^16 queries.  Each stage is timed with CUDA events over --reps back-to-back runs after a warm-up.  Reported:
stage times, queries/s and problems/s (one problem = one state), the status counts, a histogram of iteration counts
(the optimizer launch lasts as long as its slowest problem), and the card name and power limit read in the same
run.  Needs a CUDA device: there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cpprobotics_b200 import Engine, SlpSampler, synth  # noqa: E402
from oracle import mptg as OM  # noqa: E402
from oracle import slp as OS  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-queries", type=int, default=1 << 12)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("slp_bench.py needs a CUDA device (libcrb has no CPU fallback)")
    os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    eng = Engine(0)
    prm, v = eng.slp_default_params()
    tb = synth.slp_table(24)
    tbd = torch.from_numpy(tb).to(dev)
    res = dict(gpu=gpu_info(), host_cores=OM.num_threads(), table_rows=int(tb.shape[0]), cells=[])
    for nq in (1 << 12, 1 << 14, 1 << 16):
        fields, qp = synth.slp_inputs(nq, OS.BIASED)
        s = SlpSampler(fields["kind"], fields["nxy"], fields["nh"], fields["ns"], fields["d"])
        S = eng.slp_states_per_query(s)
        n = nq * S
        qd = torch.from_numpy(qp).to(dev)
        tgt = torch.empty((3, n), dtype=torch.float32, device=dev)
        nst, sst = (torch.empty(nq, dtype=torch.int32, device=dev) for _ in range(2))
        param = torch.empty((4, n), dtype=torch.float32, device=dev)
        row = torch.empty(n, dtype=torch.int32, device=dev)
        q0 = torch.empty_like(param)
        state = torch.zeros((4, n), dtype=torch.float32, device=dev)
        state[3] = v
        st, it = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ms = np.zeros(3)
        for rep in range(a.reps + 1):   # the first round is the warm-up
            ev[0].record()
            eng.slp_sample_states(s, qd, tgt, nst, sst)
            ev[1].record()
            eng.slp_search_nearest(tgt, tbd, param=q0, row=row)
            ev[2].record()
            param.copy_(q0)
            eng.mptg_optimize(state, tgt, param, prm, status=st, iters=it)
            ev[3].record()
            ev[3].synchronize()
            if rep:
                ms += [ev[k].elapsed_time(ev[k + 1]) for k in range(3)]
        ms /= a.reps
        total = ms.sum() / 1e3
        status, iters = st.cpu().numpy(), it.cpu().numpy()
        cell = dict(queries=nq, problems=n, sample_ms=ms[0], search_ms=ms[1], optimize_ms=ms[2],
                    queries_per_s=nq / total, problems_per_s=n / total,
                    status_hist=dict(zip(["converged", "max_iter_reached", "empty_traj", "step_cap", "out_of_range"],
                                         np.bincount(status, minlength=5).tolist())),
                    iters_hist={int(k): int(c) for k, c in zip(*np.unique(iters, return_counts=True))},
                    sampler_out_of_range=int((sst.cpu().numpy() != 0).sum()))
        if nq <= a.cpu_queries:
            osmp = OS.sample(OS.sampler(fields["kind"], fields["nxy"], fields["nh"], fields["ns"], fields["d"]), qp)
            t = time.perf_counter()
            osmp = OS.sample(OS.sampler(fields["kind"], fields["nxy"], fields["nh"], fields["ns"], fields["d"]), qp)
            og = OS.generate_path(osmp["target"], tb)
            dt = time.perf_counter() - t
            assert np.array_equal(og["status"], status) and np.array_equal(og["iters"], iters)
            cell.update(cpu_queries=nq, cpu_seconds=dt, cpu_queries_per_s=nq / dt, cpu_problems_per_s=n / dt)
        res["cells"].append(cell)
        print(json.dumps(cell), flush=True)
    eng.close()
    with open(os.path.join(a.out, "slp_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
