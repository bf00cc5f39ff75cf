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
    """n seeded robots with the quirk robots spread through the batch (every 97th slot).  With params, the robots'
    speeds and yaw rates lie within (and one in four at) that configuration's limits."""
    if params is None:
        x, u, g = synth.dwa_inputs(n, seed=seed)
    else:
        x, u, g = synth.dwa_inputs(n, seed=seed, max_speed=params.max_speed, min_speed=params.min_speed,
                                   max_yawrate=params.max_yawrate)
    qx, qu, qg = quirk_agents(ob, params)
    slots = np.arange(0, n, 97)[: qx.shape[1]]
    k = len(slots)
    x[:, slots], u[:, slots], g[:, slots] = qx[:, :k], qu[:, :k], qg[:, :k]
    return x, u, g


# ---- configurations away from the reference's default Config --------------------------------------------------
# name -> (why, Config members that differ from the defaults, options).  Every one is accepted by
# crb_dwa_rollout_points.  Options: heavy (many samples or steps: small batches), yaw0 (start yaws put on every
# third robot).  The "*_cap" resolutions are the smallest floats the sample-count rule accepts for their windows.
CONFIGS = {
    "distinct": ("a realistic robot whose twelve members are all distinct, so a swapped field changes the result",
                 dict(max_speed=1.6, min_speed=-0.35, max_yawrate=0.9, max_accel=0.45, robot_radius=0.55,
                      max_dyawrate=1.3, v_reso=0.02, yawrate_reso=0.004, dt=0.05, predict_time=2.2,
                      to_goal_cost_gain=0.8, speed_cost_gain=1.15), {}),
    "speed_cap": ("the speed window at its cap (62 samples) at ordinary magnitudes",
                  dict(max_speed=2.0, min_speed=-1.0, max_accel=0.3, dt=0.1, v_reso=0.00096786505,
                       max_dyawrate=0.1, predict_time=1.0), {}),
    "yaw_cap": ("the yaw-rate window at its cap (510 samples) at ordinary magnitudes",
                dict(max_yawrate=1.0, max_dyawrate=2.0, dt=0.1, yawrate_reso=0.0007843736, v_reso=0.05,
                     predict_time=1.0), {}),
    "both_caps_2_steps": ("both windows at their caps (31,620 samples) with a two-step rollout",
                          dict(max_speed=2.0, min_speed=-1.0, max_accel=0.3, v_reso=0.00096786505, max_yawrate=1.0,
                               max_dyawrate=2.0, yawrate_reso=0.0007843736, dt=0.1, predict_time=0.1),
                          dict(heavy=True)),
    "both_caps_1_step": ("both windows at their caps with a one-step rollout: the last point is odd, never checked",
                         dict(max_speed=2.0, min_speed=-1.0, max_accel=0.3, v_reso=0.00096786505, max_yawrate=1.0,
                              max_dyawrate=2.0, yawrate_reso=0.0007843736, dt=0.1, predict_time=0.05),
                         dict(heavy=True)),
    "steps_1000": ("exactly CRB_DWA_MAX_STEPS rollout steps; the last point is even, an obstacle-check point",
                   dict(dt=0.0625, predict_time=62.4375, max_dyawrate=0.2), dict(heavy=True)),
    "steps_999": ("999 rollout steps; the last point is odd and not obstacle-checked",
                  dict(dt=0.0625, predict_time=62.375, max_dyawrate=0.2), dict(heavy=True)),
    "zero_steps": ("predict_time < 0: no rollout step, every sample ties and the last one in v-major order wins",
                   dict(predict_time=-1.0), {}),
    "one_step": ("predict_time in [0, dt): one rollout step", dict(predict_time=0.03), {}),
    "radius_zero": ("robot_radius = 0: only an obstacle exactly on a checked point collides",
                    dict(robot_radius=0.0), {}),
    "radius_negative": ("robot_radius < 0: nothing ever collides", dict(robot_radius=-1.0), {}),
    "radius_five": ("robot_radius = 5 with no rollout step, so 3-4-5 distances sit exactly on the radius",
                    dict(robot_radius=5.0, predict_time=-0.5), {}),
    "gains_zero": ("both gains 0: the obstacle cost alone decides", dict(to_goal_cost_gain=0.0, speed_cost_gain=0.0),
                   {}),
    "gains_negative": ("negative gains: the cost rewards turning away from the goal and slowing down",
                       dict(to_goal_cost_gain=-1.3, speed_cost_gain=-0.7), {}),
    "gains_overflow": ("gains near FLT_MAX: costs overflow to +-inf and inf - inf gives NaN",
                       dict(to_goal_cost_gain=3.0e38, speed_cost_gain=-3.0e38), {}),
    "speed_gain_above_min_cost": ("a speed gain that puts every cost above min_cost's initial 10000 (no sample lands "
                                  "on max_speed): best = -1, u = (0, u_prev[1])",
                                  dict(speed_cost_gain=1.0e30, max_speed=1.5, max_accel=0.25), {}),
    "empty_speed_window": ("min_speed > max_speed: the speed window is always empty",
                           dict(min_speed=0.5, max_speed=0.2), {}),
    "empty_yaw_window": ("max_yawrate < 0: the yaw-rate window is always empty", dict(max_yawrate=-0.3), {}),
    "yaw_past_120": ("yaw rates and a horizon that carry the yaw past 120 rad (sinf / cosf's large reduction), and "
                     "robots that start at |yaw| >= 120 and >= 2^20",
                     dict(max_yawrate=40.0, max_dyawrate=20.0, yawrate_reso=0.05, predict_time=4.0),
                     dict(yaw0=(130.25, -250.5, 1048576.5, -3.0e7, 119.99))),
    "speed_cap_large": ("speed 1.2e7 (ulp 1), v_reso 3 ulps: the widest speed window the rule accepts there",
                        dict(max_speed=1.2e7, min_speed=11999845.0, max_accel=1000.0, v_reso=3.0, predict_time=0.3),
                        {}),
    "yaw_cap_large": ("yaw rate 3e6 (ulp 0.25), yawrate_reso 3 ulps: the widest yaw window the rule accepts there",
                      dict(max_yawrate=3.0e6, max_dyawrate=1274.0, yawrate_reso=0.75, dt=0.125, predict_time=0.25),
                      {}),
}


def config(name):
    return OD.dwa_params(**CONFIGS[name][1])


def heavy(name):
    return CONFIGS[name][2].get("heavy", False)


def config_batch(name, n, ob, seed=0xC0FFEE):
    """batch() for the configuration `name`, its start yaws applied to every third robot."""
    p = config(name)
    x, u, g = batch(n, ob, seed=seed, params=p)
    yaw0 = CONFIGS[name][2].get("yaw0")
    if yaw0:
        k = np.arange(0, n, 3)
        x[2, k] = np.resize(np.float32(yaw0), len(k))
    return x, u, g
