"""Writes tests/golden/slp_golden.npz: the reference's OWN src/state_lattice_planner.cpp (compiled against oracle/shim
into oracle/_ref/libref_slp.so) on tests/golden/lookuptable.csv: the three demo scenarios end to end (every
trajectory whole, max_pts 256), and a seeded set of queries per sampler with the search and generate_path of their
states.  The fixture keeps the pin where neither the reference nor oracle/_ref exists.
Run: python tests/golden/make_slp_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import slp_cases as SC  # noqa: E402
from cpprobotics_b200 import synth  # noqa: E402
from oracle import mptg as OM  # noqa: E402
from oracle import slp as OS  # noqa: E402

MAX_PTS = 256
N_SEEDED = 24   # queries per sampler; generate_path runs on the first states of the valid ones


def main():
    L = SC.ref_lib()
    tb = SC.table()
    out = dict(table=tb)
    for kind, name in ((0, "uniform"), (1, "biased"), (2, "lane")):
        traj, ln = SC.ref_demo(L, kind, tb, MAX_PTS)
        out[f"demo_{name}_traj"], out[f"demo_{name}_len"] = traj, ln
        fields, qp = synth.slp_inputs(N_SEEDED, kind, seed=0x601D + kind)
        s = SC.sampler_of(fields)
        target, cnt = SC.ref_sample(L, s, qp)
        out[f"seeded_{name}_qp"], out[f"seeded_{name}_target"], out[f"seeded_{name}_n_states"] = qp, target, cnt
        # the search and generate_path of the states the reference defines: finite (no csv_file[-1]), and with an
        # optimization that ends CONVERGED or MAX_ITER_REACHED by the checker (no back() of an empty trajectory)
        # (and not of a query the checker refuses as outside the exact sin / cos range)
        valid = np.repeat(OS.sample(s, qp)["status"] == OS.OK, OS.states_per_query(s))
        fin = np.flatnonzero(np.isfinite(target).all(axis=0) & valid)
        ok = OS.generate_path(np.ascontiguousarray(target[:, fin]), tb)["status"] <= OM.MAX_ITER_REACHED
        fin = fin[ok][:64]
        t = np.ascontiguousarray(target[:, fin])
        out[f"seeded_{name}_cols"] = fin.astype(np.int32)
        out[f"seeded_{name}_param"] = SC.ref_search(L, t, tb)
        out[f"seeded_{name}_traj"], out[f"seeded_{name}_len"] = SC.ref_generate_path(L, t, tb, 0.0, MAX_PTS)
    np.savez_compressed(os.path.join(HERE, "slp_golden.npz"), **out)


if __name__ == "__main__":
    main()
