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


def ekf_fleet_inputs(n: int, n_models: int, seed: int = 0xC0FFEE, n_steps: int = 1):
    """ekf_inputs for a fleet whose agents each name one of n_models noise models.  Returns a dict with x, P, z, u as
    ekf_inputs gives them and the model table as arrays: dt float64 [m] in [0.02, 0.2], Q float32 [m, 16] and R
    float32 [m, 4] (column-major, as crb_ekf_params; pack them with engine.ekf_models), and model_of int32 [n], a
    shuffled assignment that uses every model when n >= n_models.  Q is the reference's diagonal scaled per model,
    with non-symmetric off-diagonal entries in every other model; R is a per-model diagonal, non-symmetric in every
    third model."""
    x, P, z, u = ekf_inputs(n, seed=seed, n_steps=n_steps)
    rng = np.random.default_rng([seed, n_models, 0xEF])
    m = int(n_models)
    dt = rng.uniform(0.02, 0.2, m)
    Q = np.zeros((m, 16), np.float64)
    Q[:, [0, 5, 15]] = 0.01 * rng.uniform(0.25, 4.0, (m, 3))
    Q[:, 10] = (np.pi / 180) ** 2 * rng.uniform(0.25, 4.0, m)
    off = [1, 2, 3, 4, 6, 7, 8, 9, 11, 12, 13, 14]
    Q[::2, off] = 1e-3 * rng.uniform(-1.0, 1.0, (len(range(0, m, 2)), len(off)))
    R = np.zeros((m, 4), np.float64)
    R[:, [0, 3]] = rng.uniform(0.1, 2.0, (m, 2))
    R[::3, 1:3] = rng.uniform(-0.05, 0.05, (len(range(0, m, 3)), 2))
    model_of = (rng.permutation(n) % m).astype(np.int32)
    return dict(x=x, P=P, z=z, u=u, dt=dt, Q=Q.astype(np.float32), R=R.astype(np.float32), model_of=model_of)


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


# src/a_star.cpp / src/dijkstra.cpp:247-286: the demo's walls (float loop counters, 60.0 - i narrowed to float), start
# (10, 10), goal (50, 50), grid_size 1, robot_size 1.  The box is [0, 60) x [0, 60): 60 x 60 cells.
GRID_DEMO = dict(sx=10.0, sy=10.0, gx=50.0, gy=50.0, reso=1.0, rr=1.0)


def grid_demo_obstacles():
    """(ox, oy) float32 in the demo's push_back order."""
    ox, oy = [], []
    for i in range(60):
        ox.append(i); oy.append(60.0)
    for i in range(60):
        ox.append(60.0); oy.append(i)
    for i in range(61):
        ox.append(i); oy.append(60.0)
    for i in range(61):
        ox.append(0.0); oy.append(i)
    for i in range(40):
        ox.append(20.0); oy.append(i)
    for i in range(40):
        ox.append(40.0); oy.append(60.0 - i)
    return np.float32(ox), np.float32(oy)


def grid_scatter_obstacles(side: int, reso: float = 1.0, per_cell: float = 1.0 / 40, seed: int = 0x6A1D):
    """(ox, oy) float32: obstacles at the corners (0, 0) and (side, side), which make the box [0, side)^2 cells, and
    round(side^2 * per_cell) obstacles scattered uniformly over it (coordinates in metres, cell * reso)."""
    k = int(round(side * side * per_cell))
    idx = np.arange(k, dtype=np.uint64)
    x = uniform(seed, 170, idx, 0.0, side * reso)
    y = uniform(seed, 171, idx, 0.0, side * reso)
    ox = np.concatenate([[0.0, side * reso], x]).astype(np.float32)
    oy = np.concatenate([[0.0, side * reso], y]).astype(np.float32)
    return ox, oy


def grid_inputs(n: int, box, grid_map, reso: float, seed: int = 0xC0FFEE, i0: int = 0):
    """sg [4, n] float32 (sx, sy, gx, gy) for the grid planners on one map (box (min_x, min_y, max_x, max_y), grid_map
    [W, H], nonzero = blocked); query i a function of (seed, i0 + i) and the map only.  Start and goal are free cells,
    given in metres with a jitter of up to 0.45 cell that the planners' rounding removes.  One query in 64 is a corner
    case, by index:
      1  the goal on a blocked cell (unreachable)      2  the start outside the box
      3  a NaN goal                                      4  start == goal
      5  the goal outside the box                        6  the start on a blocked cell (the reference expands it)"""
    idx = np.arange(i0, i0 + n, dtype=np.uint64)
    m = np.asarray(grid_map)
    W, H = m.shape
    free = np.flatnonzero(m.reshape(-1) == 0)
    blocked = np.flatnonzero(m.reshape(-1) != 0)
    if free.size == 0:
        raise ValueError("the map has no free cell")

    def pick(cells, stream):
        k = np.minimum((u01(seed, stream, idx) * cells.size).astype(np.int64), cells.size - 1)
        c = cells[k]
        return c // H + int(box[0]), c % H + int(box[1])

    sx, sy = pick(free, 180)
    gx, gy = pick(free, 181)
    corner = idx % np.uint64(64)
    if blocked.size:
        bx, by = pick(blocked, 182)
        gx, gy = np.where(corner == 1, bx, gx), np.where(corner == 1, by, gy)
        sx, sy = np.where(corner == 6, bx, sx), np.where(corner == 6, by, sy)
    sx = np.where(corner == 2, int(box[0]) - 3, sx)
    gx, gy = np.where(corner == 4, sx, gx), np.where(corner == 4, sy, gy)
    gy = np.where(corner == 5, int(box[3]) + 2, gy)
    jit = [uniform(seed, 183 + j, idx, -0.45, 0.45) for j in range(4)]
    sg = np.stack([(sx + jit[0]) * reso, (sy + jit[1]) * reso, (gx + jit[2]) * reso, (gy + jit[3]) * reso])
    sg[2] = np.where(corner == 3, np.nan, sg[2])
    return np.ascontiguousarray(sg.astype(np.float32))


# src/rrt.cpp: the demo's six circular obstacles (x, y, r), start (0, 0), goal (6, 9), rand_area {-2, 15}, expand_dis 0.5
# (RRT's other constructor arguments take their defaults: goal_sample_rate 5).
RRT_DEMO = dict(sx=0.0, sy=0.0, gx=6.0, gy=9.0, rand_min=-2.0, rand_max=15.0, expand_dis=0.5)


def rrt_demo_obstacles():
    """ob [6, 3] float32 rows (x, y, r) in the demo's order."""
    return np.float32([[5, 5, 1], [3, 6, 2], [3, 8, 2], [3, 10, 2], [7, 5, 2], [9, 5, 2]])


def rrt_scatter_obstacles(k: int, lo: float, hi: float, r_min: float = 0.3, r_max: float = 1.2, seed: int = 0x5A77):
    """ob [k, 3] float32: k circles with centres uniform over [lo, hi)^2 and radii uniform in [r_min, r_max)."""
    idx = np.arange(k, dtype=np.uint64)
    return np.ascontiguousarray(np.stack([uniform(seed, 190, idx, lo, hi), uniform(seed, 191, idx, lo, hi),
                                          uniform(seed, 192, idx, r_min, r_max)], axis=1).astype(np.float32))


def rrt_inputs(n: int, ob, lo: float, hi: float, seed: int = 0xC0FFEE, i0: int = 0):
    """(se [4, n] float32 (sx, sy, gx, gy), seed [n] uint32) for RRT queries on one map ob [k, 3]: query i a function of
    (seed, i0 + i) and the map only.  Start and goal are uniform over [lo, hi)^2 outside every obstacle (a point inside
    one is redrawn from the next of 16 streams; after 16 tries it is kept).  One query in 64 is a corner case, by index:
      1  start == goal          2  the start inside an obstacle (the reference never checks it)"""
    o = np.asarray(ob, np.float32).reshape(-1, 3)
    idx = np.arange(i0, i0 + n, dtype=np.uint64)

    def point(stream):
        px, py = uniform(seed, stream, idx, lo, hi).astype(np.float32), uniform(seed, stream + 1, idx, lo, hi).astype(np.float32)
        for t in range(1, 16):
            inside = ((px[:, None] - o[:, 0]) ** 2 + (py[:, None] - o[:, 1]) ** 2 <= o[:, 2] ** 2).any(axis=1) \
                if o.size else np.zeros(n, bool)
            if not inside.any():
                break
            px = np.where(inside, uniform(seed, stream + 2 * t, idx, lo, hi), px).astype(np.float32)
            py = np.where(inside, uniform(seed, stream + 2 * t + 1, idx, lo, hi), py).astype(np.float32)
        return px, py

    sx, sy = point(200)
    gx, gy = point(240)
    corner = idx % np.uint64(64)
    gx, gy = np.where(corner == 1, sx, gx), np.where(corner == 1, sy, gy)
    if o.size:
        sx, sy = np.where(corner == 2, o[0, 0], sx), np.where(corner == 2, o[0, 1], sy)
    se = np.ascontiguousarray(np.stack([sx, sy, gx, gy]).astype(np.float32))
    seeds = (splitmix64(idx ^ np.uint64(seed)) >> np.uint64(32)).astype(np.uint32)
    return se, seeds


# ---- LQR path tracking (src/lqr_steer_control.cpp, src/lqr_speed_steer_control.cpp) ------------------------------
# The demos' waypoints (main() of each program); the course is input data, so a float64 natural cubic spline here
# stands in for the reference's Spline2D (its bits are not reproduced, only its shape).
LQR_DEMO_WAYPOINTS = {
    "demo": ([0.0, 6.0, 12.5, 10.0, 7.5, 3.0, -1.0], [0.0, -3.0, -5.0, 6.5, 3.0, 5.0, -2.0]),          # lqr_steer
    "demo_speed": ([0.0, 6.0, 12.5, 10.0, 17.5, 20.0, 25.0], [0.0, -3.0, -5.0, 6.5, 3.0, 0.0, 0.0]),  # speed+steer
}
LQR_KINDS = ("straight", "circle", "sine", "scurve", "demo", "demo_speed")
LQR_TARGET_SPEED = 10.0 / 3.6


def _natural_spline(t, v):
    """Coefficients of the natural cubic spline through (t, v): value, first and second derivative callables."""
    t, v = np.asarray(t, np.float64), np.asarray(v, np.float64)
    h = np.diff(t)
    m = len(t)
    A = np.zeros((m, m))
    r = np.zeros(m)
    A[0, 0] = A[-1, -1] = 1.0
    for i in range(1, m - 1):
        A[i, i - 1], A[i, i], A[i, i + 1] = h[i - 1], 2.0 * (h[i - 1] + h[i]), h[i]
        r[i] = 3.0 * ((v[i + 1] - v[i]) / h[i] - (v[i] - v[i - 1]) / h[i - 1])
    c = np.linalg.solve(A, r)
    b = (v[1:] - v[:-1]) / h - h * (2.0 * c[:-1] + c[1:]) / 3.0
    d = (c[1:] - c[:-1]) / (3.0 * h)

    def seg(s):
        i = np.clip(np.searchsorted(t, s, side="right") - 1, 0, m - 2)
        return i, s - t[i]

    def f(s, der=0):
        i, x = seg(s)
        if der == 0:
            return v[i] + b[i] * x + c[i] * x ** 2 + d[i] * x ** 3
        if der == 1:
            return b[i] + 2.0 * c[i] * x + 3.0 * d[i] * x ** 2
        return 2.0 * c[i] + 6.0 * d[i] * x
    return f


def lqr_speed_profile(cyaw, target_speed: float = LQR_TARGET_SPEED) -> np.ndarray:
    """calc_speed_profile of src/lqr_steer_control.cpp:35-53 (the speed+steer program's version writes past the end
    of its vector): target_speed, its sign flipped after each 45-90 degree yaw step, 0 at those steps and at the end."""
    sp = np.full(len(cyaw), np.float32(target_speed), np.float32)
    direction = 1.0
    for i in range(len(cyaw) - 1):
        dyaw = abs(float(np.float32(cyaw[i + 1]) - np.float32(cyaw[i])))
        switch = (np.pi / 4.0 < dyaw) and (dyaw < np.pi / 2.0)
        if switch:
            direction = -direction
        sp[i] = target_speed * (-1 if direction != 1.0 else 1)
        if switch:
            sp[i] = 0.0
    sp[-1] = 0.0
    return sp


def lqr_course(kind: str, ds: float = 0.1):
    """A float32 course (cx, cy, cyaw, ck, sp) sampled every ds metres: "straight" (40 m along a slanted line),
    "circle" (radius 8, one lap), "sine" (amplitude 3, wavelength 20, 60 m), "scurve" (two opposite 10 m arcs), or the
    demos' waypoints through a float64 natural cubic spline over chord length ("demo" of lqr_steer_control, "demo_speed"
    of lqr_speed_steer_control).  sp is lqr_speed_profile of the yaw at the demos' 10 km/h."""
    if kind == "straight":
        s = np.arange(0.0, 40.0, ds)
        th = 0.3
        x, y = s * np.cos(th), s * np.sin(th)
        yaw, k = np.full_like(s, th), np.zeros_like(s)
    elif kind == "circle":
        r = 8.0
        s = np.arange(0.0, 2 * np.pi * r, ds)
        a = s / r
        x, y = r * np.sin(a), r - r * np.cos(a)
        yaw, k = a, np.full_like(s, 1.0 / r)
    elif kind == "sine":
        xs = np.arange(0.0, 60.0, ds)
        w = 2 * np.pi / 20.0
        x, y = xs, 3.0 * np.sin(w * xs)
        dy, ddy = 3.0 * w * np.cos(w * xs), -3.0 * w * w * np.sin(w * xs)
        yaw, k = np.arctan2(dy, 1.0), ddy / (1.0 + dy * dy) ** 1.5
    elif kind == "scurve":
        r = 10.0
        s = np.arange(0.0, np.pi * r, ds)
        a = s / r
        half = a < np.pi / 2
        a2 = a - np.pi / 2
        x = np.where(half, r * np.sin(a), r + r * np.sin(np.pi / 2 - a2))
        y = np.where(half, r - r * np.cos(a), r + r - r * np.cos(np.pi / 2 - a2))
        yaw = np.where(half, a, np.pi / 2 - a2)
        k = np.where(half, 1.0 / r, -1.0 / r)
    elif kind in LQR_DEMO_WAYPOINTS:
        wx, wy = (np.asarray(w, np.float64) for w in LQR_DEMO_WAYPOINTS[kind])
        t = np.concatenate([[0.0], np.cumsum(np.hypot(np.diff(wx), np.diff(wy)))])
        fx, fy = _natural_spline(t, wx), _natural_spline(t, wy)
        s = np.arange(0.0, t[-1], ds)
        x, y = fx(s), fy(s)
        dx, dy, ddx, ddy = fx(s, 1), fy(s, 1), fx(s, 2), fy(s, 2)
        yaw = np.arctan2(dy, dx)
        k = (ddy * dx - ddx * dy) / (dx * dx + dy * dy) ** 1.5
    else:
        raise ValueError(f"unknown course kind {kind!r}; one of {LQR_KINDS}")
    cx, cy, cyaw, ck = (np.ascontiguousarray(a, np.float32) for a in (x, y, yaw, k))
    return cx, cy, cyaw, ck, lqr_speed_profile(cyaw)


def lqr_track_inputs(n: int, course, seed: int = 0xC0FFEE):
    """n vehicles around a course: a random course point, up to 2 m off it (a tenth of them up to 30 m), yaw the
    course heading plus up to +-1 rad (a twentieth anywhere in +-200 rad), speed from {0, the demo's 10 km/h, 1, 0.3,
    -1.5} or uniform in [-3, 6]; pe, pth_e small and ind a random course index.  Returns (state [4, n] float32,
    ind [n] int32, pe [n] float32, pth_e [n] float32)."""
    cx, cy, cyaw = course[0], course[1], course[2]
    rng = np.random.default_rng(seed)
    nc = len(cx)
    j = rng.integers(0, nc, n)
    off = rng.uniform(-2.0, 2.0, (2, n))
    far = rng.random(n) < 0.1
    off[:, far] *= 15.0
    x = cx[j] + off[0]
    y = cy[j] + off[1]
    yaw = cyaw[j] + rng.uniform(-1.0, 1.0, n)
    wild = rng.random(n) < 0.05
    yaw[wild] = rng.uniform(-200.0, 200.0, int(wild.sum()))
    v = rng.uniform(-3.0, 6.0, n)
    pick = rng.integers(0, 6, n)
    table = np.array([0.0, LQR_TARGET_SPEED, 1.0, 0.3, -1.5])
    v = np.where(pick < 5, table[np.minimum(pick, 4)], v)
    state = np.ascontiguousarray(np.stack([x, y, yaw, v]).astype(np.float32))
    ind = rng.integers(0, nc, n).astype(np.int32)
    pe = rng.uniform(-1.0, 1.0, n).astype(np.float32)
    pth_e = rng.uniform(-0.5, 0.5, n).astype(np.float32)
    return state, ind, pe, pth_e


# ---- many courses: the *_many entry points (a course per vehicle) ---------------------------------------------------
def pack_courses(courses):
    """A list of courses (cx, cy, cyaw, ck, sp) -> (cx, cy, cyaw, ck, sp, course_off): each field of every course
    concatenated in list order (float32 [npts]) and course_off (int64 [n_courses + 1]), course c being
    [course_off[c], course_off[c + 1])."""
    lens = [len(c[0]) for c in courses]
    off = np.zeros(len(courses) + 1, np.int64)
    off[1:] = np.cumsum(lens)
    fields = tuple(np.ascontiguousarray(np.concatenate([np.asarray(c[f], np.float32).reshape(-1) for c in courses])
                                        if courses else np.zeros(0, np.float32)) for f in range(5))
    return fields + (off,)


def _mpc_course_with_curvature():
    cx, cy, cyaw, sp = mpc_course()
    s = np.arange(0.0, 500.0, 1.0)
    dy, ddy = np.cos(s / 20.0), -np.sin(s / 20.0) / 20.0
    return cx, cy, cyaw, (ddy / (1.0 + dy * dy) ** 1.5).astype(np.float32), sp


def fleet_courses(n_courses: int, seed: int = 0xF1EE7):
    """n_courses varied courses (cx, cy, cyaw, ck, sp) for a fleet: each a random stretch of one of the LQR_KINDS
    courses or the MPC course (mpc_course, with its curvature), rotated by a random angle (cyaw turns with it) and
    moved by up to 500 m.  Lengths run from 2 points to the whole base course; every 16th course (the second, the
    eighteenth, ...) and about one in twenty others have a single point.  Deterministic for a seed."""
    rng = np.random.default_rng(seed)
    bases = [lqr_course(k) for k in LQR_KINDS] + [_mpc_course_with_curvature()]
    out = []
    for c in range(n_courses):
        b = bases[int(rng.integers(0, len(bases)))]
        nb = len(b[0])
        if c % 16 == 1 or rng.random() < 0.05:
            ln = 1
        else:
            ln = int(rng.integers(2, nb + 1))
        s0 = int(rng.integers(0, nb - ln + 1))
        th = rng.uniform(-np.pi, np.pi)
        tx, ty = rng.uniform(-500.0, 500.0, 2)
        x, y = (np.asarray(a[s0:s0 + ln], np.float64) for a in b[:2])
        ct, st = np.cos(th), np.sin(th)
        out.append(tuple(np.ascontiguousarray(a, np.float32) for a in (
            ct * x - st * y + tx, st * x + ct * y + ty, np.asarray(b[2][s0:s0 + ln], np.float64) + th,
            b[3][s0:s0 + ln], b[4][s0:s0 + ln])))
    return out


# ---- an obstacle list per robot: crb_dwa_control_many_batched, crb_rrt_plan_many_batched --------------------------
def pack_obstacles(lists, k: int):
    """A list of obstacle lists ([m_s, k] rows each, m_s >= 0) -> (ob, ob_off): every list's rows back to back in list
    order (float32 [n_rows, k]) and ob_off (int64 [n_sets + 1]), list s being rows [ob_off[s], ob_off[s + 1])."""
    rows = [np.asarray(o, np.float32).reshape(-1, k) for o in lists]
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    ob = np.concatenate(rows) if rows else np.zeros((0, k), np.float32)
    return np.ascontiguousarray(ob, np.float32).reshape(-1, k), off


def dwa_fleet_obstacles(n_sets: int, seed: int = 0x0B57):
    """n_sets varied DWA obstacle lists ([m, 2] float32 rows (ox, oy)): list s is empty when s % 16 == 0, one row when
    s % 16 == 1, CRB_DWA_MAX_OBSTACLES rows when s % 16 == 2, and otherwise 2 to 64 rows.  Each list lies in its own
    arena: a square of half-width 3 to 30 m around a centre up to 5 m from the demo's (5, 5), so that robots drawn by
    dwa_inputs see near, sparse and dense obstacles.  Deterministic for a seed."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n_sets):
        m = {0: 0, 1: 1, 2: 256}.get(s % 16, int(rng.integers(2, 65)))
        h = float(rng.uniform(3.0, 30.0))
        cx, cy = 5.0 + rng.uniform(-5.0, 5.0, 2)
        out.append(np.ascontiguousarray(np.stack([rng.uniform(cx - h, cx + h, m), rng.uniform(cy - h, cy + h, m)],
                                                 axis=1).astype(np.float32).reshape(m, 2)))
    return out


# ---- a Config per robot: crb_dwa_control_fleet_batched ------------------------------------------------------------
# Robot classes: the Config members each one sets apart from the reference's (:27-40).  Window sizes (speed x yaw-rate
# samples) and rollout steps are at most about 2/3 of CRB_DWA_MAX_SPEED_SAMPLES, CRB_DWA_MAX_YAWRATE_SAMPLES and
# CRB_DWA_MAX_STEPS, so that dwa_fleet_configs' +-15 % changes to every member stay within the limits.
DWA_ROBOT_CLASSES = (
    ("reference", {}),                                             # 5 x 80 samples, 30 steps
    ("small_fast", dict(max_speed=2.0, min_speed=-0.3, max_yawrate=2.0, max_accel=1.0, robot_radius=0.3,
                        max_dyawrate=3.0, v_reso=0.02, yawrate_reso=0.02, dt=0.1, predict_time=1.5,
                        to_goal_cost_gain=1.2, speed_cost_gain=0.6)),      # 11 x 31, 15 steps
    ("large_slow", dict(max_speed=0.4, min_speed=-0.1, max_yawrate=0.3, max_accel=0.05, robot_radius=2.0,
                        max_dyawrate=0.2, v_reso=0.005, yawrate_reso=0.002, dt=0.2, predict_time=5.0,
                        to_goal_cost_gain=0.7, speed_cost_gain=1.5)),      # 5 x 41, 26 steps
    ("coarse_grid", dict(max_accel=0.5, v_reso=0.05, yawrate_reso=0.02)),  # 3 x 7, 30 steps
    ("fine_grid", dict(max_accel=0.3, max_dyawrate=0.6, v_reso=0.002, yawrate_reso=0.0005, predict_time=2.0)),
    ("short_horizon", dict(max_accel=0.4, dt=0.05, predict_time=0.6)),    # 5 x 40, 13 steps
    ("long_horizon", dict(predict_time=8.0, robot_radius=0.5)),           # 5 x 80, 81 steps
    ("no_reverse", dict(max_speed=1.2, min_speed=0.0, max_yawrate=1.0, max_accel=0.3, robot_radius=0.6,
                        max_dyawrate=1.5, v_reso=0.015, yawrate_reso=0.01, dt=0.08, predict_time=2.4,
                        to_goal_cost_gain=1.0, speed_cost_gain=0.8)),     # 4 x 25, 31 steps
)


def dwa_fleet_configs(n_configs: int, seed: int = 0xC1A55):
    """n_configs robot classes (DwaParams): class k is DWA_ROBOT_CLASSES[k % 8] (the fine grid has 31 x 241 samples and
    21 steps), exactly for k < 8 and with every member scaled by its own factor in [0.85, 1.15] from k = 8 on.
    Every class is inside crb.h's limits.  Deterministic for a seed."""
    from ._lib import DwaParams
    pi = 3.141592653
    ref = dict(max_speed=1.0, min_speed=-0.5, max_yawrate=40.0 * pi / 180.0, max_accel=0.2, robot_radius=1.0,
               max_dyawrate=40.0 * pi / 180.0, v_reso=0.01, yawrate_reso=0.1 * pi / 180.0, dt=0.1, predict_time=3.0,
               to_goal_cost_gain=1.0, speed_cost_gain=1.0)
    names = [k for k, _ in DwaParams._fields_]
    out = []
    for k in range(n_configs):
        d = dict(ref, **DWA_ROBOT_CLASSES[k % len(DWA_ROBOT_CLASSES)][1])
        if k >= len(DWA_ROBOT_CLASSES):
            scale = uniform(seed, 130, np.arange(k * 12, k * 12 + 12, dtype=np.uint64), 0.85, 1.15)
            d = {m: d[m] * float(scale[j]) for j, m in enumerate(names)}
        out.append(DwaParams(*(float(np.float32(d[m])) for m in names)))
    return out


def dwa_fleet_inputs(configs, config_of, seed: int = 0xC0FFEE):
    """x [5,n], u [2,n], goal [2,n] for robots on classes configs[config_of[i]]: the robots of class c are
    dwa_inputs(m_c, seed + c) with that class's speed and yaw-rate limits, so each sits within its own limits and one
    in four sits at a speed limit and one in four at a yaw-rate limit.  Deterministic for a seed."""
    config_of = np.asarray(config_of)
    n = config_of.size
    x, u, g = np.empty((5, n), np.float32), np.empty((2, n), np.float32), np.empty((2, n), np.float32)
    for c in np.unique(config_of):
        sel = np.nonzero(config_of == c)[0]
        p = configs[int(c)]
        x[:, sel], u[:, sel], g[:, sel] = dwa_inputs(sel.size, seed=seed + int(c), max_speed=p.max_speed,
                                                     min_speed=p.min_speed, max_yawrate=p.max_yawrate)
    return x, u, g


def rrt_fleet_obstacles(n_sets: int, seed: int = 0x5CA7, lo: float = -2.0, hi: float = 15.0, max_k: int = 64):
    """n_sets scattered RRT maps ([m, 3] float32 rows (x, y, r)) over one planning area [lo, hi)^2: map s has 0 to max_k
    circles (rrt_scatter_obstacles, radii 0.3 to 1.2) from a seed of its own; every 16th map (s % 16 == 0) is empty.
    Deterministic for a seed."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n_sets):
        m = 0 if s % 16 == 0 else int(rng.integers(0, max_k + 1))
        out.append(rrt_scatter_obstacles(m, lo, hi, seed=int(rng.integers(1 << 31))))
    return out


def dwa_neighbour_obstacles(x, static_ob, radius: float, cap: int = 256, chunk: int = 16384):
    """The obstacle lists of a fleet that avoids itself: robot i's list is the static obstacles static_ob [m, 2], then
    the positions (x[0], x[1]) of the other robots within `radius` of it (squared distance in float64 <= radius^2),
    nearest first (ties by robot index), the whole list cut at `cap` rows.  x [5, n] (or [2+, n]) float32.  Returns
    (ob, ob_off) as pack_obstacles, list i being robot i's (so ob_of = arange(n)).  Built in numpy on a hash grid of
    radius-sized cells, `chunk` robots at a time: for tests and benchmarks."""
    px, py = np.asarray(x[0], np.float32), np.asarray(x[1], np.float32)
    n = px.size
    st = np.asarray(static_ob, np.float32).reshape(-1, 2)[:cap]
    room = cap - len(st)
    pos = np.stack([px, py], axis=1)
    gx = np.floor(px.astype(np.float64) / radius).astype(np.int64)
    gy = np.floor(py.astype(np.float64) / radius).astype(np.int64)
    gx -= gx.min() - 1
    gy -= gy.min() - 1
    span = int(gy.max()) + 2
    key = gx * span + gy
    order = np.argsort(key, kind="stable")
    skey = key[order]
    counts = np.zeros(n, np.int64)
    nbr = []
    r2 = float(radius) * float(radius)
    for c0 in range(0, n, chunk):
        ii = np.arange(c0, min(n, c0 + chunk))
        pi, pj = [], []
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                t = key[ii] + dx * span + dy
                lo_, hi_ = np.searchsorted(skey, t, "left"), np.searchsorted(skey, t, "right")
                cnt = hi_ - lo_
                rep = np.repeat(np.arange(ii.size), cnt)
                start = np.repeat(lo_ - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
                pi.append(ii[rep])
                pj.append(order[start + np.arange(rep.size)])
        i, j = np.concatenate(pi), np.concatenate(pj)
        d2 = (px[j].astype(np.float64) - px[i]) ** 2 + (py[j].astype(np.float64) - py[i]) ** 2
        keep = (i != j) & (d2 <= r2)
        i, j, d2 = i[keep], j[keep], d2[keep]
        o = np.lexsort((j, d2, i))
        i, j = i[o], j[o]
        first = np.searchsorted(i, ii, "left")
        rank = np.arange(i.size) - np.repeat(first, np.bincount(i - c0, minlength=ii.size))
        take = rank < room
        counts[ii] = np.minimum(np.bincount(i - c0, minlength=ii.size), max(room, 0))
        nbr.append(j[take])
    nbr = np.concatenate(nbr) if nbr else np.zeros(0, np.int64)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(counts + len(st))
    ob = np.empty((int(off[-1]), 2), np.float32)
    row = np.arange(int(off[-1])) - np.repeat(off[:-1], counts + len(st))
    is_st = row < len(st)
    ob[is_st] = st[row[is_st]]
    ob[~is_st] = pos[nbr]
    return ob, off


# ---- a map per query: crb_grid_obstacle_map_many, crb_grid_plan_many_batched ----------------------------------------
def _grid_cells(o, reso):
    """(int)round(o * 1.0 / reso) in double, as the planners round obstacles"""
    return np.round(np.asarray(o, np.float32).astype(np.float64) * 1.0 / np.float64(np.float32(reso))).astype(np.int64)


def grid_fleet_maps(n_maps: int, seed: int = 0x6F1E):
    """n_maps varied grid maps over shared obstacle lists: dict(lists ([k, 2] float32 rows (ox, oy)), ob_of int32
    [n_maps], boxes int32 [n_maps, 4], reso float32 [n_maps], rr float32 [n_maps]).  Every list is scattered over a
    window of up to 60 x 60 cells at a base resolution between 10^-2 and 10^1.7 and offset up to 40 cells from the
    origin; list s is empty when s % 16 == 0.  About four maps share each list, each at the base resolution or 1.5 or
    2 times it, with rr 0, 0.5, 1 or 2 times its resolution.  By map index: m % 8 == 1 is a single cell, m % 8 == 2 a
    rectangular window cut from the list's box, m % 8 == 3 that box grown by 3 cells on each side, otherwise the box of
    its list's window.  Deterministic for a seed."""
    rng = np.random.default_rng(seed)
    n_lists = max(1, (n_maps + 3) // 4)
    lists, base = [], []
    for s in range(n_lists):
        r0 = float(np.float32(10.0 ** rng.uniform(-2.0, 1.69)))
        W0, H0 = int(rng.integers(2, 61)), int(rng.integers(2, 61))
        x0, y0 = int(rng.integers(-40, 41)), int(rng.integers(-40, 41))
        k = 0 if s % 16 == 0 else int(rng.integers(1, max(2, W0 * H0 // 6)))
        cx, cy = x0 + rng.uniform(0.0, W0, k), y0 + rng.uniform(0.0, H0, k)
        lists.append(np.ascontiguousarray(np.stack([cx * r0, cy * r0], axis=1).astype(np.float32).reshape(k, 2)))
        base.append((r0, x0, y0, W0, H0))
    ob_of = np.zeros(n_maps, np.int32)
    boxes = np.zeros((n_maps, 4), np.int32)
    reso = np.zeros(n_maps, np.float32)
    rr = np.zeros(n_maps, np.float32)
    for m in range(n_maps):
        s = int(rng.integers(n_lists)) if m >= n_lists else m
        r0, x0, y0, W0, H0 = base[s]
        r = np.float32(r0 * (1.0, 1.0, 1.5, 2.0)[int(rng.integers(4))])
        bx0, by0 = int(np.floor(x0 * r0 / r)), int(np.floor(y0 * r0 / r))
        W, H = max(1, int(np.ceil(W0 * r0 / r))), max(1, int(np.ceil(H0 * r0 / r)))
        kind = m % 8
        if kind == 1:
            bx0, by0, W, H = bx0 + int(rng.integers(W)), by0 + int(rng.integers(H)), 1, 1
        elif kind == 2:
            w, h = int(rng.integers(1, W + 1)), int(rng.integers(1, H + 1))
            bx0, by0, W, H = bx0 + int(rng.integers(W - w + 1)), by0 + int(rng.integers(H - h + 1)), w, h
        elif kind == 3:
            bx0, by0, W, H = bx0 - 3, by0 - 3, W + 6, H + 6
        ob_of[m], reso[m] = s, r
        boxes[m] = (bx0, by0, bx0 + W, by0 + H)
        rr[m] = np.float32(r * (0.0, 0.5, 1.0, 2.0)[int(rng.integers(4))])
    return dict(lists=lists, ob_of=ob_of, boxes=boxes, reso=reso, rr=rr)


def grid_local_windows(n_robots: int, side: int = 256, win: int = 64, reso: float = 1.0, rr: float = 1.0,
                       seed: int = 0x10CA):
    """A fleet in one obstacle field, each robot planning in its own win x win window: the field is
    grid_scatter_obstacles(side, reso) and every window a box of cells at a seeded offset inside [0, side)^2.  Returns
    the dict of grid_fleet_maps, with one list that every window shares (ob_of all 0), reso and rr the same for all."""
    ox, oy = grid_scatter_obstacles(side, reso)
    rng = np.random.default_rng(seed)
    x0 = rng.integers(0, side - win + 1, n_robots)
    y0 = rng.integers(0, side - win + 1, n_robots)
    boxes = np.ascontiguousarray(np.stack([x0, y0, x0 + win, y0 + win], axis=1).astype(np.int32))
    return dict(lists=[np.ascontiguousarray(np.stack([ox, oy], axis=1))], ob_of=np.zeros(n_robots, np.int32),
                boxes=boxes, reso=np.full(n_robots, reso, np.float32), rr=np.full(n_robots, rr, np.float32))


def grid_fleet_inputs(n: int, boxes, reso, maps, map_off, seed: int = 0xC0FFEE):
    """(map_of int32 [n], sg float32 [4, n]) for n queries over the maps of a table (boxes [n_maps, 4], reso, the byte
    store maps and map_off): every query on a map drawn uniformly, in shuffled order, and the queries of map m
    grid_inputs(k, boxes[m], map m, reso[m], seed, i0 = (57 + m) % 64), so that each map's first queries are
    grid_inputs' corner cases.  A map with no free cell takes its queries as if every cell were free.  Deterministic for
    a seed."""
    rng = np.random.default_rng(seed)
    n_maps = len(reso)
    map_of = rng.integers(0, n_maps, n).astype(np.int32)
    sg = np.zeros((4, n), np.float32)
    order = np.argsort(map_of, kind="stable")
    cuts = np.searchsorted(map_of[order], np.arange(n_maps + 1))
    for m in range(n_maps):
        sel = order[cuts[m]:cuts[m + 1]]
        if sel.size == 0:
            continue
        b = boxes[m]
        W, H = int(b[2]) - int(b[0]), int(b[3]) - int(b[1])
        mm = np.asarray(maps[int(map_off[m]):int(map_off[m + 1])]).reshape(W, H)
        if not (mm == 0).any():
            mm = np.zeros_like(mm)
        sg[:, sel] = grid_inputs(sel.size, b, mm, float(reso[m]), seed=seed, i0=(57 + m) % 64)
    return map_of, sg


PF_RFID = ((10.0, 0.0), (10.0, 10.0), (0.0, 15.0), (-5.0, 20.0))   # the demo's tags, src/particle_filter.cpp:192-196
PF_MAX_RANGE = 20.0                                                  # :20


def pf_fleet_inputs(n_robots: int, np_per_robot: int, seed: int = 0xF1EE7, tags=PF_RFID,
                    max_range: float = PF_MAX_RANGE, spread: float = 10.0):
    """A fleet of particle filters for crb_pf_step_many_batched: robot r has its own hidden true pose (within `spread`
    m of the origin), its own particles (a 0.2 m cloud around that pose, random yaw and speed), its own control u
    (speed 0.5..1.5, yaw rate -0.3..0.3) and its own observation list built as the demo builds z (:257-268): the tags
    of the shared set `tags` ([k, 2], the demo's four by default) within max_range of the true pose, each as a row
    (range + 0.04 N(0,1), lx, ly).  Lists are packed with pack_obstacles(lists, 3), one list per robot.
    Returns dict(px [4,n], pw [n] (= 1/np), u [2,n_robots], z [n_rows,3], z_off [n_robots+1], z_of [n_robots],
    noise [2,n], uniforms [n] in [1,2), truth [4,n_robots]), float32 / int64 / int32, n = n_robots * np_per_robot."""
    nr, npr = int(n_robots), int(np_per_robot)
    n = nr * npr
    ridx = np.arange(nr, dtype=np.uint64)
    pidx = np.arange(n, dtype=np.uint64)
    truth = np.stack([uniform(seed, 70, ridx, -spread, spread), uniform(seed, 71, ridx, -spread, spread),
                      uniform(seed, 72, ridx, -np.pi, np.pi), uniform(seed, 73, ridx, 0.5, 1.5)])
    own = np.repeat(np.arange(nr), npr)
    px = np.empty((4, n), np.float64)
    px[0] = truth[0, own] + 0.2 * normal(seed, 74, pidx)
    px[1] = truth[1, own] + 0.2 * normal(seed, 75, pidx)
    px[2] = uniform(seed, 76, pidx, -np.pi, np.pi)
    px[3] = uniform(seed, 77, pidx, 0.0, 2.0)
    u = np.stack([uniform(seed, 78, ridx, 0.5, 1.5), uniform(seed, 79, ridx, -0.3, 0.3)])
    tg = np.asarray(tags, np.float32).reshape(-1, 2)
    tx, ty = truth[0].astype(np.float32), truth[1].astype(np.float32)
    d = np.sqrt((tx[:, None] - tg[None, :, 0]) ** 2 + (ty[:, None] - tg[None, :, 1]) ** 2).astype(np.float32)
    dn = (d + np.float32(0.04) * normal(seed, 80, np.arange(nr * len(tg), dtype=np.uint64)).reshape(nr, -1)
          .astype(np.float32)).astype(np.float32)
    seen = d <= np.float32(max_range)
    lists = [np.stack([dn[r, seen[r]], tg[seen[r], 0], tg[seen[r], 1]], axis=1) for r in range(nr)]
    z, z_off = pack_obstacles(lists, 3)
    f = np.float32
    return dict(px=np.ascontiguousarray(px.astype(f)), pw=np.full(n, 1.0 / npr, f),
                u=np.ascontiguousarray(u.astype(f)), z=z, z_off=z_off, z_of=np.arange(nr, dtype=np.int32),
                noise=np.ascontiguousarray(np.stack([normal(seed, 81, pidx), normal(seed, 82, pidx)]).astype(f)),
                uniforms=np.ascontiguousarray(uniform(seed, 83, pidx, 1.0, 2.0).astype(f)),
                truth=np.ascontiguousarray(truth.astype(f)))
