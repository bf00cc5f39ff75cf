"""Robots that reach the corners of dwa_control's semantics (src/dynamic_window_approach.cpp), for the DWA tests and
tests/golden/make_dwa_golden.py.  Each builder returns x [5,m], u [2,m], goal [2,m] (float32, libcrb layout)."""
import numpy as np

from cpprobotics_b200 import synth
from oracle import dwa as OD

f = np.float32


def _cols(rows):
    x = np.array([r[0] for r in rows], np.float32).T.copy()
    u = np.array([r[1] for r in rows], np.float32).T.copy()
    g = np.array([r[2] for r in rows], np.float32).T.copy()
    return x, u, g


def _rollout_end(x, v, w, params):
    s = np.asarray(x, np.float32).reshape(5, 1)
    uu = np.array([[v], [w]], np.float32)
    for _ in range(OD.dwa_rollout_points(params) - 1):
        s = OD.dwa_motion(s, uu, params.dt)
    return s[:, 0]


def _error(g, e):
    """calc_to_goal_cost's `error` (:105-108) in the reference's precisions."""
    gm = np.sqrt(f(g[0] * g[0]) + f(g[1] * g[1]), dtype=np.float32)
    tm = f(np.sqrt(np.float64(e[0]) ** 2 + np.float64(e[1]) ** 2))
    dot = f(f(g[0] * e[0]) + f(g[1] * e[1]))
    return f(dot / f(gm * tm))


def collinear_goal(x, params):
    """A goal on the line through the origin and the end of sample 0's rollout (v = dw[0], w = dw[2]) for which
    rounding puts `error` outside [-1, 1], so std::acos returns NaN and that sample's cost is NaN."""
    p = params
    v0 = max(f(x[3] - f(p.max_accel * p.dt)), f(p.min_speed))
    w0 = max(f(x[4] - f(p.max_dyawrate * p.dt)), f(-p.max_yawrate))
    e = _rollout_end(x, v0, w0, p)
    for k in range(1, 4000):
        c = f(0.37 + 0.0137 * k) * (1 if k % 2 else -1)
        g = (f(c * e[0]), f(c * e[1]))
        if abs(float(_error(g, e))) > 1.0:
            return g
    raise AssertionError("no collinear goal with |error| > 1 found")


def quirk_agents(ob, params=None):
    """Every sample colliding (robot on obstacle 0; only when there are obstacles), goal at the origin, a goal
    collinear with a rollout end (|error| > 1), windows clipped at each speed and yaw-rate limit, an empty window
    (v far above max_speed), the demo's start and goal, and an obstacle-free corner (subnormal obstacle cost)."""
    p = params or OD.dwa_params()
    rows = []
    if len(ob):
        rows.append(((ob[0][0], ob[0][1], 0.3, 0.5, 0.1), (0.5, 0.1), (10.0, 10.0)))
    rows.append(((3.0, 4.0, 0.2, 0.5, 0.0), (0.5, 0.0), (0.0, 0.0)))
    xc = (2.0, 3.0, 0.7, 0.5, 0.02)
    rows.append((xc, (0.5, 0.02), collinear_goal(np.array(xc, np.float32), p)))
    rows.append(((2.0, 7.0, 1.0, p.max_speed, p.max_yawrate), (p.max_speed, p.max_yawrate), (9.0, 1.0)))
    rows.append(((6.0, 1.0, -2.0, p.min_speed, -p.max_yawrate), (p.min_speed, -p.max_yawrate), (1.0, 9.0)))
    rows.append(((1.0, 1.0, 0.0, 5.0, 0.0), (0.0, 0.3), (10.0, 10.0)))
    rows.append((synth.DWA_DEMO_START, (0.0, 0.0), synth.DWA_DEMO_GOAL))
    rows.append(((-300.0, -300.0, 0.5, 0.2, 0.0), (0.2, 0.0), (-290.0, -310.0)))
    return _cols(rows)


def batch(n, ob, seed=0xC0FFEE, params=None):
    """n seeded robots with the quirk robots spread through the batch (every 97th slot)."""
    x, u, g = synth.dwa_inputs(n, seed=seed)
    qx, qu, qg = quirk_agents(ob, params)
    slots = np.arange(0, n, 97)[: qx.shape[1]]
    k = len(slots)
    x[:, slots], u[:, slots], g[:, slots] = qx[:, :k], qu[:, :k], qg[:, :k]
    return x, u, g
