"""MPC parameter sets away from the reference's constants, shared by the CPU and GPU tests.

The reference's weights come in equal pairs (w_x = w_y, w_yaw = w_v, w_a = w_delta), so a test at the defaults
cannot see two of them swapped.  W gives every weight its own value; B changes the model and the bounds so that
the speed bound is active (max_speed 4 m/s against starting speeds up to 5 m/s); S is a slow, long-step vehicle.
REVERSE asks for -2 m/s on a straight road with min_speed = -1, so the lower speed bound binds."""
from __future__ import annotations

import numpy as np

from cpprobotics_b200 import synth

W = dict(w_x=2.0, w_y=0.7, w_yaw=0.3, w_v=1.3, w_a=0.05, w_delta=0.002, w_da=0.2, w_ddelta=3.0)
B = dict(dt=0.1, wb=1.8, max_steer=0.3, max_accel=2.5, max_speed=4.0, min_speed=-1.0)
S = dict(dt=0.3, wb=4.0, max_steer=0.6, max_accel=0.4)
REVERSE = dict(min_speed=-1.0)
SETS = dict(W=W, B=B, S=S)

# the largest float below 0.5: roundf gives 0 here, floorf(q + 0.5f) gives 1
EDGE_Q = np.nextafter(np.float32(0.5), np.float32(0.0))


def set_params(target, over):
    """target (a ctypes MpcParams) with the fields of `over` set; returns target."""
    for k, v in over.items():
        setattr(target, k, v)
    return target


def f64_params(over):
    """The same constants for the float64 statement (oracle/ref_mpc_f64.py): the float32 values the solver sees."""
    return {k: (float(np.float32(v)) if isinstance(v, float) else v) for k, v in over.items()}


def case(n, T, seed=0xC0FFEE, dt=0.2):
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, seed=seed, course=course)
    xref, _ = synth.mpc_xref_numpy(st, pind, T, course=course, dt=dt)
    return st, xref


def reverse_case(n, T, dt=0.2):
    """Straight road along x driven backwards at -2 m/s, lateral offsets in [-0.5, 0.5] m, yaw 0 (the car
    faces +x), starting speeds in [-1, 0.5] m/s."""
    st = np.zeros((4, n), np.float32)
    st[1] = np.linspace(-0.5, 0.5, n)
    st[2] = np.linspace(-0.05, 0.05, n)[::-1]
    st[3] = np.linspace(-1.0, 0.5, n)
    xref = np.zeros((4 * T, n), np.float32)
    for t in range(T):
        xref[4 * t] = np.float32(-2.0 * dt * t)
        xref[4 * t + 3] = -2.0
    return st, xref


def travel_q(v, t, dl, DT):
    """travel / dl after t steps of calc_ref_trajectory's accumulation (:149-150) at speed v."""
    travel = np.float32(0.0)
    for _ in range(t):
        travel = np.float32(np.float64(travel) + np.float64(abs(np.float32(v))) * DT)
    return np.float32(travel / np.float32(dl))


def rounding_edge_speeds(dl, DT, t_max=32):
    """[(t, v)]: for each stage t in 1..t_max the smallest speed v >= 0 (if any) whose travel / dl after t steps
    is exactly EDGE_Q.  travel_q is monotone in v, so a bisection over the float bits of v finds it."""
    out = []
    for t in range(1, t_max + 1):
        lo, hi = 0, int(np.float32(100.0).view(np.int32))
        while lo < hi:   # smallest bit pattern with travel_q >= EDGE_Q
            mid = (lo + hi) // 2
            if travel_q(np.int32(mid).view(np.float32), t, dl, DT) >= EDGE_Q:
                hi = mid
            else:
                lo = mid + 1
        v = np.int32(lo).view(np.float32)
        if travel_q(v, t, dl, DT) == EDGE_Q:
            out.append((t, v))
    return out


def edge_states(speeds):
    """state [4, k] at (10, 20 sin 0.5, 0.5) on synth.mpc_course() with the given speeds (search from pind 5)."""
    k = len(speeds)
    st = np.empty((4, k), np.float32)
    st[0], st[1], st[2] = 10.0, np.float32(20.0 * np.sin(0.5)), 0.5
    st[3] = np.asarray(speeds, np.float32)
    return st, np.full(k, 5, np.int32)
