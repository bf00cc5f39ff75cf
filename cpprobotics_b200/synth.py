"""Seeded, index-addressed synthetic inputs for the BASELINE.json configs (SURVEY.md §8 d-3..d-6).

Every value is a pure function of (seed, stream, global agent index), so a shard [i0, i0+n) holds
the same bits whatever the GPU count, and the CPU oracle and the GPU path consume identical arrays.
The reference itself seeds from std::random_device (src/extended_kalman_filter.cpp:163-164) and is
not reproducible; these generators replace its main()-level simulation, not any hot-path code.
numpy only (no torch, no oracle).
"""
from __future__ import annotations

import numpy as np

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)
_G = np.uint64(0x9E3779B97F4A7C15)


def splitmix64(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = (x + _G).astype(np.uint64)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def u01(seed: int, stream: int, idx: np.ndarray) -> np.ndarray:
    """float64 uniform in [0,1) for each global index."""
    with np.errstate(over="ignore"):
        key = splitmix64(np.array([np.uint64(seed) ^ (np.uint64(stream) * _G)], dtype=np.uint64))[0]
        h = splitmix64(idx.astype(np.uint64) ^ key)
    return (h >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def uniform(seed, stream, idx, lo, hi):
    return lo + (hi - lo) * u01(seed, stream, idx)


def normal(seed, stream, idx):
    """Box-Muller in float64 from two uniform streams (2*stream, 2*stream+1 of a private space)."""
    a = u01(seed, 1000 + 2 * stream, idx)
    b = u01(seed, 1001 + 2 * stream, idx)
    return np.sqrt(-2.0 * np.log(1.0 - a)) * np.cos(2.0 * np.pi * b)


# ---- config 2: batched EKF (SURVEY §8 d-3) ---------------------------------------------------------
def ekf_inputs(n: int, i0: int = 0, seed: int = 0xC0FFEE, n_steps: int = 1):
    """x [4,n], P [16,n] (column-major), z [2*n_steps,n], u [2*n_steps,n], all float32."""
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    x = np.empty((4, n), np.float64)
    x[0] = uniform(seed, 0, idx, -50.0, 50.0)
    x[1] = uniform(seed, 1, idx, -50.0, 50.0)
    x[2] = uniform(seed, 2, idx, -np.pi, np.pi)
    x[3] = uniform(seed, 3, idx, 0.0, 10.0)
    # P = L L^T + 0.1 I with L lower triangular, entries U(-0.5, 0.5): SPD, eigenvalues O(0.1..1)
    L = np.zeros((4, 4, n), np.float64)
    s = 10
    for r in range(4):
        for c in range(r + 1):
            L[r, c] = uniform(seed, s, idx, -0.5, 0.5)
            s += 1
    P = np.empty((16, n), np.float64)
    for c in range(4):
        for r in range(4):
            acc = 0.1 * (r == c)
            for k in range(4):
                acc = acc + L[r, k] * L[c, k]
            P[r + 4 * c] = acc
    z = np.empty((2 * n_steps, n), np.float64)
    u = np.empty((2 * n_steps, n), np.float64)
    for st in range(n_steps):
        u[2 * st + 0] = 1.0 + 0.5 * normal(seed, 40 + 4 * st, idx)
        u[2 * st + 1] = 0.1 + 0.1 * normal(seed, 41 + 4 * st, idx)
        z[2 * st + 0] = x[0] + 0.1 * st + 0.5 * normal(seed, 42 + 4 * st, idx)
        z[2 * st + 1] = x[1] + 0.5 * normal(seed, 43 + 4 * st, idx)
    f = np.float32
    return (np.ascontiguousarray(x.astype(f)), np.ascontiguousarray(P.astype(f)),
            np.ascontiguousarray(z.astype(f)), np.ascontiguousarray(u.astype(f)))


# ---- config 3: batched PF predict + weight (SURVEY §8 d-4) -------------------------------------------
PF_TRUTH = (2.0, -1.0, 0.3, 1.0)


def pf_landmarks(n_lm: int = 8, seed: int = 0xC0FFEE, radius: float = 15.0) -> np.ndarray:
    """rows (range, lx, ly) like the reference's observation items (src/particle_filter.cpp:263-266):
    landmarks on a circle, range = distance from the hidden truth pose + 0.04 * N(0,1)."""
    k = np.arange(n_lm, dtype=np.float64)
    lx = radius * np.cos(2.0 * np.pi * k / n_lm)
    ly = radius * np.sin(2.0 * np.pi * k / n_lm)
    d = np.sqrt((lx - PF_TRUTH[0]) ** 2 + (ly - PF_TRUTH[1]) ** 2)
    d = d + 0.04 * normal(seed, 90, np.arange(n_lm, dtype=np.uint64))
    return np.ascontiguousarray(np.stack([d, lx, ly], axis=1).astype(np.float32))


def pf_inputs(n: int, i0: int = 0, seed: int = 0xC0FFEE, n_total: int | None = None):
    """px [4,n], pw [n] (= 1/n_total), noise [2,n] (standard normal), float32."""
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    px = np.empty((4, n), np.float64)
    px[0] = PF_TRUTH[0] + 0.2 * normal(seed, 60, idx)
    px[1] = PF_TRUTH[1] + 0.2 * normal(seed, 61, idx)
    px[2] = uniform(seed, 62, idx, -np.pi, np.pi)
    px[3] = uniform(seed, 63, idx, 0.0, 2.0)
    noise = np.stack([normal(seed, 64, idx), normal(seed, 65, idx)], axis=0)
    pw = np.full(n, 1.0 / float(n_total if n_total else n), np.float64)
    f = np.float32
    return (np.ascontiguousarray(px.astype(f)), np.ascontiguousarray(pw.astype(f)),
            np.ascontiguousarray(noise.astype(f)))


# ---- configs 4/5: batched MPC (SURVEY §8 d-5) ------------------------------------------------------------
def mpc_course(length: float = 500.0, dl: float = 1.0):
    """Analytic course sampled every dl metres: cx = s, cy = 20 sin(s/20), cyaw = heading, sp = 10/3.6
    (the reference's target speed, src/model_predictive_control.cpp:488)."""
    s = np.arange(0.0, length, dl)
    cx = s
    cy = 20.0 * np.sin(s / 20.0)
    cyaw = np.arctan2(np.cos(s / 20.0), 1.0)
    sp = np.full_like(s, 10.0 / 3.6)
    f = np.float32
    return cx.astype(f), cy.astype(f), cyaw.astype(f), sp.astype(f)


def mpc_states(n: int, i0: int = 0, seed: int = 0xC0FFEE, course=None):
    """state [4,n] float32 and the integer course index each agent starts its search from [n] int32:
    a course point at s0 ~ U(0,400) displaced laterally by U(-1,1) m, yaw + U(-0.2,0.2), v ~ U(0,5)."""
    cx, cy, cyaw, _ = course if course is not None else mpc_course()
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    k = np.floor(uniform(seed, 80, idx, 0.0, 400.0)).astype(np.int64)
    lat = uniform(seed, 81, idx, -1.0, 1.0)
    st = np.empty((4, n), np.float64)
    st[0] = cx[k] - lat * np.sin(cyaw[k])
    st[1] = cy[k] + lat * np.cos(cyaw[k])
    st[2] = cyaw[k] + uniform(seed, 82, idx, -0.2, 0.2)
    st[3] = uniform(seed, 83, idx, 0.0, 5.0)
    pind = np.maximum(k - 5, 0).astype(np.int32)
    return np.ascontiguousarray(st.astype(np.float32)), np.ascontiguousarray(pind)


def mpc_xref_numpy(state, pind, T: int, course=None, dl: float = 1.0, dt: float = 0.2):
    """Vectorised restatement of calc_ref_trajectory / calc_nearest_index
    (src/model_predictive_control.cpp:107-170) used to synthesise the solver's xref input
    [4T, n] (field 4t+k).  float32 arithmetic where the reference uses float.  dt is the double DT of :149
    (for a crb_mpc_params.dt other than the default, the value libcrb promotes it to: the float's own value)."""
    cx, cy, cyaw, sp = course if course is not None else mpc_course()
    n = state.shape[1]
    nc = len(cx)
    win = np.minimum(pind[None, :].astype(np.int64) + np.arange(10)[:, None], nc - 1)
    dxw = cx[win] - state[0][None, :]
    dyw = cy[win] - state[1][None, :]
    d = (dxw * dxw + dyw * dyw).astype(np.float32)
    # first strict minimum inside the (clipped) window
    valid = (pind[None, :].astype(np.int64) + np.arange(10)[:, None]) < nc
    d = np.where(valid, d, np.float32(np.inf))
    ind = pind.astype(np.int64) + np.argmin(d, axis=0)
    ind = np.maximum(ind, pind.astype(np.int64))
    xref = np.empty((4 * T, n), np.float32)
    travel = np.zeros(n, np.float32)
    for i in range(T):
        travel = (travel.astype(np.float64) + np.abs(state[3]).astype(np.float64) * dt).astype(np.float32)
        q = (travel / np.float32(dl)).astype(np.float32)
        # roundf (:150): half away from zero.  q >= 0 and q < 2^23, so floor(q) and q - floor(q) are exact;
        # floor(q + 0.5f) is not (it rounds q = 0.49999997f up to 1)
        r = np.floor(q)
        dind = (r + (q - r >= np.float32(0.5))).astype(np.int64)
        j = np.minimum(ind + dind, nc - 1)
        xref[4 * i + 0] = cx[j]
        xref[4 * i + 1] = cy[j]
        xref[4 * i + 2] = cyaw[j]
        xref[4 * i + 3] = sp[j]
    return np.ascontiguousarray(xref), ind.astype(np.int32)


# ---- row f-4: batched LQR (lqr_steer_control.cpp / lqr_speed_steer_control.cpp) ----------------------------
def lqr_inputs(n: int, nx: int, i0: int = 0, seed: int = 0xC0FFEE, dt: float = 0.1, wheel_base: float = 0.5):
    """Per-agent (A, B) exactly as lqr_steering_control builds them from the vehicle speed
    (src/lqr_steer_control.cpp:104-112, src/lqr_speed_steer_control.cpp:116-126), v ~ U(0.3, 4) m/s, plus the
    reference's Q = I, R = I.  Column-major, float32: A [nx*nx, n], B [nx*nu, n], Q [nx*nx], R [nu*nu]."""
    assert nx in (4, 5)
    nu = 1 if nx == 4 else 2
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    v = uniform(seed, 95, idx, 0.3, 4.0).astype(np.float32)
    A = np.zeros((nx * nx, n), np.float32)
    B = np.zeros((nx * nu, n), np.float32)
    A[0 + nx * 0] = 1.0
    A[0 + nx * 1] = np.float32(dt)
    A[1 + nx * 2] = v
    A[2 + nx * 2] = 1.0
    A[2 + nx * 3] = np.float32(dt)
    B[3 + nx * 0] = v / np.float32(wheel_base)
    if nx == 5:
        A[4 + nx * 4] = 1.0
        B[4 + nx * 1] = np.float32(dt)
    return A, B, np.eye(nx, dtype=np.float32).reshape(-1), np.eye(nu, dtype=np.float32).reshape(-1)


# ---- dynamic window approach (src/dynamic_window_approach.cpp) --------------------------------------------
# main()'s obstacle list (:169-180), start state (:167) and goal (:168)
DWA_DEMO_OBSTACLES = np.array([[-1, -1], [0, 2], [4, 2], [5, 4], [5, 5], [5, 6], [5, 9], [8, 9], [7, 9], [12, 12]],
                              np.float32)
DWA_DEMO_START = (0.0, 0.0, 3.141592653 / 8.0, 0.0, 0.0)
DWA_DEMO_GOAL = (10.0, 10.0)


def dwa_inputs(n: int, seed: int = 0xC0FFEE, i0: int = 0, max_speed: float = 1.0, min_speed: float = -0.5,
               max_yawrate: float = 40.0 * 3.141592653 / 180.0):
    """x [5,n] (x, y, yaw, v, yawrate), u [2,n] (u[1] = the previous yaw rate), goal [2,n], float32.
    Robots in the demo's arena ([-2, 12]^2, goal anywhere in it), v and yaw rate inside the limits; one robot in
    four sits exactly at a speed limit and one in four at a yaw-rate limit, so its window is clipped (:55-58)."""
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    f = np.float32
    x = np.empty((5, n), np.float32)
    x[0] = uniform(seed, 110, idx, -2.0, 12.0)
    x[1] = uniform(seed, 111, idx, -2.0, 12.0)
    x[2] = uniform(seed, 112, idx, -np.pi, np.pi)
    x[3] = uniform(seed, 113, idx, min_speed, max_speed)
    x[4] = uniform(seed, 114, idx, -max_yawrate, max_yawrate)
    pick_v = u01(seed, 115, idx)
    pick_w = u01(seed, 116, idx)
    x[3] = np.where(pick_v < 0.125, f(max_speed), np.where(pick_v < 0.25, f(min_speed), x[3]))
    x[4] = np.where(pick_w < 0.125, f(max_yawrate), np.where(pick_w < 0.25, f(-max_yawrate), x[4]))
    u = np.empty((2, n), np.float32)
    u[0] = x[3]
    u[1] = x[4]
    goal = np.empty((2, n), np.float32)
    goal[0] = uniform(seed, 117, idx, -2.0, 12.0)
    goal[1] = uniform(seed, 118, idx, -2.0, 12.0)
    return np.ascontiguousarray(x), np.ascontiguousarray(u), np.ascontiguousarray(goal)


def dwa_obstacles(k: int, seed: int = 0xC0FFEE) -> np.ndarray:
    """[k, 2] rows (ox, oy), obstacle j a function of (seed, j, k) only: uniform in a square around the demo's
    arena that grows with k so that the density stays the demo's (10 in 14 m x 14 m) and most robots keep an
    admissible sample."""
    idx = np.arange(k, dtype=np.uint64)
    h = 7.0 * max(1.0, np.sqrt(k / 10.0))
    ob = np.stack([uniform(seed, 120, idx, 5.0 - h, 5.0 + h), uniform(seed, 121, idx, 5.0 - h, 5.0 + h)], axis=1)
    return np.ascontiguousarray(ob.astype(np.float32))


# ---- model-predictive trajectory generation (src/model_predictive_trajectory_generator.cpp) -------------------
# main()'s start state (:26, CONST_V 3.0), target (:27) and initial parameter (:30)
MPTG_DEMO_STATE = (0.0, 0.0, 0.0, 3.0)
MPTG_DEMO_TARGET = (5.0, 2.0, 0.0)
MPTG_DEMO_PARAM = (6.0, 0.0, 0.0, 0.0)


def mptg_inputs(n: int, seed: int = 0xC0FFEE, i0: int = 0):
    """state [4,n] (x, y, yaw, v), target [3,n] (x, y, yaw), param [4,n] (distance, steering_sequence[0..2]),
    float32; problem i a function of (seed, i0 + i) only.  Around the demo: start at the origin with v = 3, target
    x in [3, 8], y in [-3, 3], yaw in [-0.6, 0.6], initial parameter (hypot(x, y) + 1, {0, 0, 0}).  One problem in
    64 is a corner case, by index: distance -1 (an empty roll-out), steering[0] = 150 (tanf outside the exact
    range), distance 2000 (more than CRB_MPTG_MAX_STEPS steps), start yaw 200 (sinf / cosf outside the exact
    range), a target behind the start (rarely converges)."""
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    state = np.zeros((4, n), np.float32)
    state[3] = 3.0
    target = np.empty((3, n), np.float32)
    target[0] = uniform(seed, 130, idx, 3.0, 8.0)
    target[1] = uniform(seed, 131, idx, -3.0, 3.0)
    target[2] = uniform(seed, 132, idx, -0.6, 0.6)
    param = np.zeros((4, n), np.float32)
    param[0] = np.hypot(target[0].astype(np.float64), target[1].astype(np.float64)) + 1.0
    corner = idx % np.uint64(64)
    param[0] = np.where(corner == 1, np.float32(-1.0), param[0])
    param[1] = np.where(corner == 2, np.float32(150.0), param[1])
    param[0] = np.where(corner == 3, np.float32(2000.0), param[0])
    state[2] = np.where(corner == 4, np.float32(200.0), state[2])
    target[0] = np.where(corner == 5, np.float32(-4.0), target[0])
    return np.ascontiguousarray(state), np.ascontiguousarray(target), np.ascontiguousarray(param)


# src/state_lattice_planner.cpp:157-210: the demo's three scenarios.  Its float constants are double expressions
# narrowed to float (e.g. -45.0/180 * M_PI); lane_state_sample_test's int d = 10 becomes the float d parameter.
_DEG = np.pi / 180.0
SLP_DEMO = {
    0: dict(nxy=5, nh=3, ns=0, d=20, qp=(-45.0 / 180 * np.pi, 45.0 / 180 * np.pi, -45.0 / 180 * np.pi,
                                         45.0 / 180 * np.pi)),
    1: dict(nxy=30, nh=2, ns=100, d=20, qp=(0.0, -45.0 / 180 * np.pi, 45.0 / 180 * np.pi, -20.0 / 180 * np.pi,
                                            20.0 / 180 * np.pi)),
    2: dict(nxy=5, nh=1, ns=0, d=0, qp=(10.0, 90.0 / 180.0 * np.pi, 3.0, 1.0, 10.0)),
}


def slp_inputs(n_q: int, kind: int, seed: int = 0xC0FFEE, i0: int = 0):
    """(sampler fields dict(kind, nxy, nh, ns, d), qp [F, n_q] float32) for the state lattice planner's samplers
    (kind 0 uniform, 1 biased, 2 lane), the demo's integers; query i a function of (seed, i0 + i) only.  Query 0 is
    the demo's scenario for that kind; the others are random around it: polar angle ranges a_min in [-1.2, 0],
    a_max in [0, 1.2], heading ranges p_min in [-0.6, 0], p_max in [0, 0.6], goal_angle in [-1, 1]; lanes with
    l_center in [-15, 15], l_heading in [-pi, pi], l_width in [1, 6], v_width in [0.5, 2], d in [5, 20].  One query in
    64 is a corner case, by index:
      1  an angle outside the exact sinf / cosf range (a_min = -200, a_max = -150; l_heading = 130)
      2  a zero-width range (a_max = a_min; v_width = l_width)
      3  a NaN input (p_max; l_center)
      4  reversed ranges (a_max < a_min, p_max < p_min; negative d); biased: goal_angle 10, so every cnav sample is
         negative and cnav_max keeps its FLT_MIN start
      5  inf inputs (a_max = +inf: NaN angles; l_width = inf: NaN offsets)"""
    idx = np.arange(i0, i0 + n_q, dtype=np.uint64)
    demo = SLP_DEMO[kind]
    f = 4 if kind == 0 else 5
    qp = np.empty((f, n_q), np.float64)
    corner = idx % np.uint64(64)
    if kind == 2:
        qp[0] = uniform(seed, 140, idx, -15.0, 15.0)
        qp[1] = uniform(seed, 141, idx, -np.pi, np.pi)
        qp[2] = uniform(seed, 142, idx, 1.0, 6.0)
        qp[3] = uniform(seed, 143, idx, 0.5, 2.0)
        qp[4] = uniform(seed, 144, idx, 5.0, 20.0)
        qp[1] = np.where(corner == 1, 130.0, qp[1])
        qp[3] = np.where(corner == 2, qp[2], qp[3])
        qp[0] = np.where(corner == 3, np.nan, qp[0])
        qp[4] = np.where(corner == 4, -qp[4], qp[4])
        qp[2] = np.where(corner == 5, np.inf, qp[2])
    else:
        o = f - 4
        if o:
            qp[0] = uniform(seed, 145, idx, -1.0, 1.0)
            qp[0] = np.where(corner == 4, 10.0, qp[0])
        qp[o] = uniform(seed, 146, idx, -1.2, 0.0)
        qp[o + 1] = uniform(seed, 147, idx, 0.0, 1.2)
        qp[o + 2] = uniform(seed, 148, idx, -0.6, 0.0)
        qp[o + 3] = uniform(seed, 149, idx, 0.0, 0.6)
        qp[o] = np.where(corner == 1, -200.0, qp[o])
        qp[o + 1] = np.where(corner == 1, -150.0, qp[o + 1])
        qp[o + 1] = np.where(corner == 2, qp[o], qp[o + 1])
        qp[o + 3] = np.where(corner == 3, np.nan, qp[o + 3])
        rev = corner == 4
        qp[o], qp[o + 1] = np.where(rev, qp[o + 1], qp[o]), np.where(rev, qp[o], qp[o + 1])
        qp[o + 2], qp[o + 3] = np.where(rev, qp[o + 3], qp[o + 2]), np.where(rev, qp[o + 2], qp[o + 3])
        qp[o + 1] = np.where(corner == 5, np.inf, qp[o + 1])
    qp[:, idx == 0] = np.asarray(demo["qp"], np.float64)[:, None]
    fields = dict(kind=kind, nxy=demo["nxy"], nh=demo["nh"], ns=demo["ns"], d=demo["d"])
    return fields, np.ascontiguousarray(qp.astype(np.float32))


def slp_table(rows: int, seed: int = 0x51A7):
    """A lookup table [rows, 6] float32 (x, y, yaw, s, km, kf) in lookuptable.csv's ranges, made without it: targets
    x in [1, 30], y in [-8, 8], yaw in [-0.6, 0.6], s = |xy|, and the seeds km = kf = the curvature of the circle
    through the origin (heading 0) and (x, y)."""
    idx = np.arange(rows, dtype=np.uint64)
    t = np.empty((rows, 6), np.float64)
    t[:, 0] = uniform(seed, 150, idx, 1.0, 30.0)
    t[:, 1] = uniform(seed, 151, idx, -8.0, 8.0)
    t[:, 2] = uniform(seed, 152, idx, -0.6, 0.6)
    t[:, 3] = np.hypot(t[:, 0], t[:, 1])
    t[:, 4] = 2.0 * t[:, 1] / (t[:, 3] ** 2)
    t[:, 5] = t[:, 4]
    return np.ascontiguousarray(t.astype(np.float32))
