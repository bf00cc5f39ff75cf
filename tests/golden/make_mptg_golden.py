"""Writes tests/golden/mptg_golden.npz: optimizer_traj() of the reference's OWN text (include/trajectory_optimizer.h
compiled against oracle/shim into oracle/_ref/libref_mptg.so) on seeded problems and the corner cases of
tests/mptg_cases.py.  The fixture keeps the pin where neither the reference nor oracle/_ref exists.
Run: python tests/golden/make_mptg_golden.py"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import mptg_cases  # noqa: E402
from cpprobotics_b200 import synth  # noqa: E402
from oracle import mptg as OM  # noqa: E402

N = 96
MAX_PTS = 128


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def reference(lib, state, target, param, params, max_pts):
    """The reference's optimizer_traj per problem: param [4,n], traj [3*max_pts,n] (NaN beyond the returned Traj),
    traj_len [n], cost [n] of the returned Traj's last point (NaN when it is empty)."""
    n = state.shape[1]
    q = np.ascontiguousarray(param, np.float32).copy()
    traj = np.full((3 * max_pts, n), np.nan, np.float32)
    tl = np.zeros(n, np.int32)
    cost = np.zeros(n, np.float32)
    h = (C.c_float * 3)(*params.h_step)
    for i in range(n):
        s, t, qi = (np.ascontiguousarray(a[:, i], np.float32) for a in (state, target, q))
        tr = np.full(3 * max_pts, np.nan, np.float32)
        k, c = C.c_int(0), C.c_float(0.0)
        lib.ref_mptg_optimize(_vp(s), _vp(t), _vp(qi), C.c_float(params.base_l), C.c_float(params.ds),
                              C.c_int(params.max_iter), C.c_float(params.cost_th), h, _vp(tr), C.c_int(max_pts),
                              C.byref(k), C.byref(c))
        q[:, i], traj[:, i], tl[i], cost[i] = qi, tr, k.value, c.value
    return q, traj, tl, cost


def golden_sets():
    st, tg, pa = synth.mptg_inputs(4 * N, seed=0x6A7)
    keep = OM.optimize(st, tg, pa)["status"] <= OM.MAX_ITER_REACHED   # only what the reference defines
    sel = np.flatnonzero(keep)[:N]
    sets = [("synth", *(np.ascontiguousarray(a[:, sel]) for a in (st, tg, pa)), OM.mptg_params())]
    return sets + mptg_cases.quirk_sets()


def main():
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_mptg.so"))
    out = {}
    for name, st, tg, pa, prm in golden_sets():
        q, traj, tl, cost = reference(lib, st, tg, pa, prm, MAX_PTS)
        out.update({f"{name}_state": st, f"{name}_target": tg, f"{name}_param_in": pa,
                    f"{name}_prm": np.array([prm.base_l, prm.ds, prm.max_iter, prm.cost_th, *prm.h_step], np.float64),
                    f"{name}_param": q, f"{name}_traj": traj, f"{name}_traj_len": tl, f"{name}_cost": cost})
    np.savez_compressed(os.path.join(HERE, "mptg_golden.npz"), names=np.array([s[0] for s in golden_sets()]), **out)


if __name__ == "__main__":
    main()
