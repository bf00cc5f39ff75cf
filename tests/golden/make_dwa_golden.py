"""Writes tests/golden/dwa_golden.npz: dwa_control() and motion() of the reference's OWN text
(src/dynamic_window_approach.cpp compiled against oracle/shim into oracle/_ref/libref_dwa.so) on seeded robots and
the quirk robots of tests/dwa_cases.py, with no obstacles, the demo's 10 and 64 random ones.  The fixture keeps the
pin where neither the reference nor oracle/_ref exists.  Run: python tests/golden/make_dwa_golden.py"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import dwa_cases  # noqa: E402
from cpprobotics_b200 import synth  # noqa: E402
from oracle import dwa as OD  # noqa: E402

N = 128
OBSTACLE_SETS = {"none": np.zeros((0, 2), np.float32), "demo": synth.DWA_DEMO_OBSTACLES,
                 "random64": synth.dwa_obstacles(64, seed=5)}


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def reference(lib, x, u, goal, ob, params):
    """The reference's dwa_control per robot: u [2,n], cost [n], traj [5*n_pts,n] (NaN when it returns an empty
    Traj), and motion(x, u_new, dt) [5,n]."""
    n, n_pts = x.shape[1], OD.dwa_rollout_points(params)
    cfg = np.array([getattr(params, k) for k, _ in params._fields_], np.float32)
    uo = np.ascontiguousarray(u, np.float32).copy()
    cost = np.zeros(n, np.float32)
    traj = np.full((5 * n_pts, n), np.nan, np.float32)
    nxt = np.zeros((5, n), np.float32)
    ob = np.ascontiguousarray(ob, np.float32)
    for i in range(n):
        xi, ui, gi = (np.ascontiguousarray(a[:, i]) for a in (x, uo, goal))
        t = np.zeros(5 * n_pts, np.float32)
        k, c = C.c_int(0), C.c_float(0.0)
        lib.ref_dwa_control(_vp(xi), _vp(ui), _vp(gi), _vp(ob), C.c_int(len(ob)), _vp(cfg), _vp(t), C.byref(k),
                            C.byref(c))
        uo[:, i], cost[i] = ui, c.value
        if k.value:
            assert k.value == n_pts
            traj[:, i] = t
        o = np.zeros(5, np.float32)
        lib.ref_dwa_motion(_vp(xi), _vp(ui), C.c_float(params.dt), _vp(o))
        nxt[:, i] = o
    return uo, cost, traj, nxt


def main():
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_dwa.so"))
    p = OD.dwa_params()
    out = {}
    for name, ob in OBSTACLE_SETS.items():
        x, u, g = dwa_cases.batch(N, ob, seed=0xD3A)
        qx, qu, qg = dwa_cases.quirk_agents(ob, p)
        x, u, g = (np.ascontiguousarray(np.concatenate(a, axis=1)) for a in ((x, qx), (u, qu), (g, qg)))
        uo, cost, traj, nxt = reference(lib, x, u, g, ob, p)
        out.update({f"{name}_ob": ob, f"{name}_x": x, f"{name}_u_in": u, f"{name}_goal": g, f"{name}_u": uo,
                    f"{name}_cost": cost, f"{name}_traj": traj, f"{name}_motion": nxt})
    np.savez_compressed(os.path.join(HERE, "dwa_golden.npz"), **out)


if __name__ == "__main__":
    main()
