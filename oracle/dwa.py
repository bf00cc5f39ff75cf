"""ctypes wrapper of oracle/lib/liboracle_dwa.so — the CPU restatement of src/dynamic_window_approach.cpp
(dwa_control, motion, glibc's acosf).  Built by `make -C oracle` (python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from ._load import LIB_DIR, checker

LIB_PATH = os.path.join(LIB_DIR, "liboracle_dwa.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


PROTOTYPES = {
    "crb_oracle_num_threads": (C.c_int, []),
    "crb_oracle_libm_acosf": (C.c_float, [C.c_float]),
    "crb_oracle_libm_acosf_census": (C.c_int64, [C.c_uint32, C.c_uint32]),
    "crb_oracle_dwa_motion": (None, [C.c_int64, f32p, f32p, C.c_float, C.c_int]),
    "crb_oracle_dwa_control": (None, [C.c_int64, f32p, f32p, f32p, C.c_void_p, C.c_int, C.c_void_p, f32p, i32p,
                                      C.c_void_p, C.c_int]),
}


def lib() -> C.CDLL:
    return checker(LIB_PATH, PROTOTYPES)


def num_threads() -> int:
    return int(lib().crb_oracle_num_threads())


# ---- src/dynamic_window_approach.cpp -------------------------------------------------------------------------
class DwaParams(C.Structure):
    """Field-for-field the same as crb_dwa_params (include/crb.h) and the reference's class Config (:25-41)."""
    _fields_ = [(name, C.c_float) for name in (
        "max_speed", "min_speed", "max_yawrate", "max_accel", "robot_radius", "max_dyawrate",
        "v_reso", "yawrate_reso", "dt", "predict_time", "to_goal_cost_gain", "speed_cost_gain")]


def dwa_params(**over) -> DwaParams:
    """Config's initialisers (:27-40): double expressions with PI = 3.141592653 (:16) narrowed to float."""
    pi = 3.141592653
    d = dict(max_speed=1.0, min_speed=-0.5, max_yawrate=40.0 * pi / 180.0, max_accel=0.2, robot_radius=1.0,
             max_dyawrate=40.0 * pi / 180.0, v_reso=0.01, yawrate_reso=0.1 * pi / 180.0, dt=0.1, predict_time=3.0,
             to_goal_cost_gain=1.0, speed_cost_gain=1.0)
    d.update(over)
    p = DwaParams()
    for k, v in d.items():
        setattr(p, k, float(np.float32(v)))
    return p


def dwa_rollout_points(params=None) -> int:
    """Points of calc_trajectory's Traj (:63-74): the reference's float `time += dt` loop, plus the start."""
    p = params or dwa_params()
    t, k = np.float32(0.0), 0
    while t <= np.float32(p.predict_time) and k <= 1000:   # CRB_DWA_MAX_STEPS
        t = np.float32(t + np.float32(p.dt))
        k += 1
    return k + 1


def libm_acosf(x) -> float:
    return float(lib().crb_oracle_libm_acosf(float(x)))


def libm_acosf_census(lo_bits: int, hi_bits: int) -> int:
    """Number of bit patterns in [lo_bits, hi_bits), both signs, where the restatement differs from the host acosf."""
    return int(lib().crb_oracle_libm_acosf_census(int(lo_bits), int(hi_bits)))


def dwa_motion(x, u, dt=None, nthreads=0):
    """motion() :43-50 on a copy of x [5,n] with u [2,n]."""
    x = np.ascontiguousarray(x, np.float32).copy()
    lib().crb_oracle_dwa_motion(x.shape[1], x, np.ascontiguousarray(u, np.float32),
                                float(dwa_params().dt if dt is None else dt), nthreads)
    return x


def dwa_control(x, u, goal, ob, params=None, traj=True, nthreads=0):
    """dwa_control() :148-155 in the libcrb layout.  x [5,n], u [2,n] (u[1] read), goal [2,n], ob [n_ob,2].
    Returns dict(u [2,n], cost [n], best [n] int32, traj [5*n_pts,n] or None)."""
    p = params or dwa_params()
    x = np.ascontiguousarray(x, np.float32)
    n = x.shape[1]
    uo = np.ascontiguousarray(u, np.float32).copy()
    ob = np.ascontiguousarray(np.asarray(ob, np.float32).reshape(-1, 2))
    cost = np.zeros(n, np.float32)
    best = np.zeros(n, np.int32)
    tr = np.zeros((5 * dwa_rollout_points(p), n), np.float32) if traj else None
    lib().crb_oracle_dwa_control(n, x, uo, np.ascontiguousarray(goal, np.float32),
                                 ob.ctypes.data if ob.size else None, ob.shape[0], C.byref(p), cost, best,
                                 None if tr is None else tr.ctypes.data, nthreads)
    return dict(u=uo, cost=cost, best=best, traj=tr)
