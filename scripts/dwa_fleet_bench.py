"""What a Config per robot costs dwa_control, and what it saves a fleet that mixes robot types.

2^18 robots (--log2n), each among one of 4096 obstacle lists (synth.dwa_fleet_obstacles), robots shuffled over lists
and classes.  Each cell times two forms alternately in one process, with CUDA events around --reps launches after
warm-up, over --rounds rounds, and reports the median ms per launch and the spread ((max - min) / median):
  a. one_record    every robot on the reference Config: crb_dwa_control_fleet_batched with a one-record table against
                   crb_dwa_control_many_batched (the cost of the record load and the per-warp record check);
  b. eight_classes 8 robot classes (synth.dwa_fleet_configs): one fleet launch against what a caller does without the
                   table: per class, gather its robots (torch index_select), one crb_dwa_control_many_batched launch,
                   scatter u, cost, best and traj back (index_copy_), all inside the timed window;
  c. heavy_class   b's classes plus tests/dwa_cases.py's both_caps_2_steps (both sample grids near their caps) as a
                   ninth: the same two forms, and the fleet launch again with the robots sorted by class (a block keeps
                   its shared memory until its slowest warp ends, so a heavy robot holds its neighbours' slots).
Every form writes u, cost, best and traj; each cell compares every output of its forms bitwise (sorted robots after
un-sorting).  Prints the card's name, power limit and clocks read in the same run, and one JSON record as the last
line, also written to --out (default: a temporary directory).

  python scripts/dwa_fleet_bench.py [--log2n 18] [--rounds 5] [--reps 3] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_LISTS = 4096


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return {"error": str(exc)[:120]}
    f = [c.strip() for c in out.split(",")]
    return dict(zip(["name", "power_limit", "sm_clock", "sm_clock_max"], f)) if len(f) == 4 else {"raw": out}


def timed(torch, fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def same(torch, a, b):
    """Bitwise equal, any NaN equal to any NaN."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if not a.dtype.is_floating_point:
        return bool(torch.equal(a, b))
    na, nb = torch.isnan(a), torch.isnan(b)
    return bool(torch.equal(na, nb)) and bool(torch.equal(a.view(torch.int32)[~na], b.view(torch.int32)[~nb]))


class Fleet:
    """One cell's robots on the device and the output buffers of each form."""

    def __init__(self, torch, eng, configs, config_of, ob_of, store, seed):
        import numpy as np
        from cpprobotics_b200 import dwa_config_table, synth
        dev = torch.device("cuda", 0)
        self.torch, self.eng, self.configs = torch, eng, configs
        self.n = n = config_of.size
        x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=seed)
        pts = [eng.dwa_rollout_points(p) for p in configs]
        self.max_pts = max(pts)
        self.pts = pts
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        self.x, self.u0, self.g, self.ob_of, self.config_of = t(x), t(u), t(g), t(ob_of), t(config_of)
        self.store = (t(store[0]), t(store[1]))
        self.table = t(dwa_config_table(configs))
        self.sel = [torch.nonzero(self.config_of == c).flatten() for c in range(len(configs))]
        self.out = {}

    def buffers(self, form):
        torch, n = self.torch, self.n
        if form not in self.out:
            dev = self.x.device
            self.out[form] = dict(u=self.u0.clone(), cost=torch.empty(n, device=dev),
                                  best=torch.empty(n, dtype=torch.int32, device=dev),
                                  traj=torch.zeros((5 * self.max_pts, n), device=dev))
        return self.out[form]

    def fleet(self, form="fleet"):
        b = self.buffers(form)
        b["u"].copy_(self.u0)
        self.eng.dwa_control_fleet(self.x, b["u"], self.g, self.store, self.ob_of, self.table, self.config_of,
                                   max_pts=self.max_pts, cost=b["cost"], best=b["best"], traj=b["traj"])

    def composed(self, form="composed"):
        """Per class: gather, one crb_dwa_control_many_batched, scatter back."""
        torch = self.torch
        b = self.buffers(form)
        b["u"].copy_(self.u0)
        for c, idx in enumerate(self.sel):
            m = idx.numel()
            if m == 0:
                continue
            ub = self.u0.index_select(1, idx)
            cost = torch.empty(m, device=idx.device)
            best = torch.empty(m, dtype=torch.int32, device=idx.device)
            traj = torch.empty((5 * self.pts[c], m), device=idx.device)
            self.eng.dwa_control_many(self.x.index_select(1, idx), ub, self.g.index_select(1, idx), self.store,
                                      self.ob_of.index_select(0, idx), self.configs[c], cost=cost, best=best,
                                      traj=traj, status=torch.empty(m, dtype=torch.int32, device=idx.device))
            b["u"].index_copy_(1, idx, ub)
            b["cost"].index_copy_(0, idx, cost)
            b["best"].index_copy_(0, idx, best)
            b["traj"][:5 * self.pts[c]].index_copy_(1, idx, traj)

    def sorted_view(self):
        """The same robots sorted by class (stable), and the permutation."""
        order = self.torch.sort(self.config_of, stable=True).indices
        s = Fleet.__new__(Fleet)
        s.__dict__.update(self.__dict__)
        s.x, s.u0, s.g = self.x[:, order].contiguous(), self.u0[:, order].contiguous(), self.g[:, order].contiguous()
        s.ob_of, s.config_of = self.ob_of[order].contiguous(), self.config_of[order].contiguous()
        s.out = {}
        return s, order


def compare(torch, got, want, order=None):
    ok = {}
    for k in ("u", "cost", "best", "traj"):
        a = got[k]
        if order is not None:
            inv = torch.empty_like(order)
            inv[order] = torch.arange(order.numel(), device=order.device)
            a = a.index_select(a.dim() - 1, inv)
        ok[k] = same(torch, a, want[k])
    return ok


def run_cell(args, torch, forms):
    """forms: {name: callable}, timed in alternated rounds.  The warm-up launches leave the outputs the cell
    compares."""
    for f in forms.values():
        f()
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in forms}
    for r in range(args.rounds):
        names = list(forms) if r % 2 == 0 else list(reversed(list(forms)))
        for k in names:
            times[k].append(timed(torch, forms[k], args.reps))
    res = {}
    for k, v in times.items():
        med = statistics.median(v)
        res[k] = dict(ms_median=round(med, 4), spread=round((max(v) - min(v)) / med, 4),
                      ms_rounds=[round(t, 4) for t in v])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2n", type=int, default=18)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "dwa_fleet_bench.json"))
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dwa_fleet_bench needs a CUDA device")
    import dwa_cases as D
    from cpprobotics_b200 import Engine, dwa_default_params, synth
    from cpprobotics_b200._lib import DwaParams
    eng = Engine(0)
    n = 1 << args.log2n
    rng = np.random.default_rng(0xBE7C)
    store = synth.pack_obstacles(synth.dwa_fleet_obstacles(N_LISTS, seed=0xB0B), 2)
    ob_of = rng.integers(0, N_LISTS, n).astype(np.int32)
    rec = dict(bench="dwa_fleet", n=n, n_lists=N_LISTS, rounds=args.rounds, reps=args.reps, card=card(), cells={})

    # a. one record
    ref = dwa_default_params()
    fa = Fleet(torch, eng, [ref], np.zeros(n, np.int32), ob_of, store, seed=0xA)

    def many():
        b = fa.buffers("many")
        b["u"].copy_(fa.u0)
        eng.dwa_control_many(fa.x, b["u"], fa.g, fa.store, fa.ob_of, ref, cost=b["cost"], best=b["best"],
                             traj=b["traj"], status=None)
    res = run_cell(args, torch, {"fleet": fa.fleet, "many": many})
    res["bitwise"] = compare(torch, fa.out["fleet"], fa.out["many"])
    res["fleet_over_many"] = round(res["fleet"]["ms_median"] / res["many"]["ms_median"], 4)
    rec["cells"]["a_one_record"] = res
    del fa
    torch.cuda.empty_cache()

    # b. eight classes
    classes = synth.dwa_fleet_configs(8, seed=0xC1A55)
    cof = rng.integers(0, 8, n).astype(np.int32)
    fb = Fleet(torch, eng, classes, cof, ob_of, store, seed=0xB)
    res = run_cell(args, torch, {"fleet": fb.fleet, "composed": fb.composed})
    res["bitwise"] = compare(torch, fb.out["fleet"], fb.out["composed"])
    res["composed_over_fleet"] = round(res["composed"]["ms_median"] / res["fleet"]["ms_median"], 4)
    res["points"] = fb.pts
    rec["cells"]["b_eight_classes"] = res
    del fb
    torch.cuda.empty_cache()

    # c. one heavy class among them
    heavy = DwaParams(*[getattr(D.config("both_caps_2_steps"), k) for k, _ in DwaParams._fields_])
    cof = rng.integers(0, 9, n).astype(np.int32)
    fc = Fleet(torch, eng, classes + [heavy], cof, ob_of, store, seed=0xC)
    fs, order = fc.sorted_view()
    res = run_cell(args, torch, {"fleet": fc.fleet, "composed": fc.composed, "fleet_sorted": fs.fleet})
    res["bitwise"] = compare(torch, fc.out["fleet"], fc.out["composed"])
    res["bitwise_sorted"] = compare(torch, fs.out["fleet"], fc.out["fleet"], order)
    res["composed_over_fleet"] = round(res["composed"]["ms_median"] / res["fleet"]["ms_median"], 4)
    res["sorted_over_fleet"] = round(res["fleet_sorted"]["ms_median"] / res["fleet"]["ms_median"], 4)
    res["heavy_samples"] = "both_caps_2_steps: up to 62 x 510 samples, 2 steps"
    rec["cells"]["c_heavy_class"] = res
    rec["all_bitwise"] = all(all(v.values()) for cell in rec["cells"].values()
                             for k, v in cell.items() if k.startswith("bitwise"))
    eng.close()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(f"card: {rec['card']}")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
