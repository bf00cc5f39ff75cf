"""Inputs for tests/test_lqr_track.py: corner cases of calc_nearest_index, lqr_steering_control and update of the two
LQR programs, and the test-driven closed loop."""
import numpy as np

from cpprobotics_b200 import synth

NAN, INF = float("nan"), float("inf")
MAX_STEER = 45.0 / 180 * np.pi


def corner_states(course):
    """(state [4, n], ind [n], pe [n], pth_e [n]) of the corner cases on a course: v = 0 (DARE_MAXITER), negative v,
    |yaw| > 120, states so far away that d_e overflows to inf (the incoming ind is kept), NaN and inf fields."""
    cx, cy, cyaw = course[0], course[1], course[2]
    nc = len(cx)
    rows = []
    m = min(nc, 7)
    for j in range(m):
        jj = (j * 37) % nc
        x, y = float(cx[jj]), float(cy[jj])
        for v in (0.0, -0.0, -1.5, -40.0, 2.7777777, 1e-3, 30.0):
            rows.append((x + 0.3, y - 0.2, float(cyaw[jj]) + 0.1, v))
        for yaw in (121.0, -150.5, 1e4, -3e5, 2 * np.pi, -np.pi, np.pi):
            rows.append((x, y, yaw, 1.0))
        rows.append((x, y, float(cyaw[jj]), 1.0))          # on the course: e = 0
    for far in (1e20, -1e20, 3e38, -3e38):                     # d_e = inf: no point wins, ind kept
        rows.append((far, 0.0, 0.5, 1.0))
        rows.append((0.0, far, -0.5, 2.0))
    for bad in ((NAN, 0.0, 0.0, 1.0), (0.0, NAN, 0.0, 1.0), (1.0, 1.0, NAN, 1.0), (1.0, 1.0, 0.0, NAN),
                (INF, 0.0, 0.0, 1.0), (1.0, 1.0, INF, 1.0), (1.0, 1.0, 0.0, INF), (1.0, 1.0, 0.0, -INF)):
        rows.append(bad)
    st = np.ascontiguousarray(np.array(rows, np.float32).T)
    n = st.shape[1]
    rng = np.random.default_rng(0x1A7)
    ind = rng.integers(0, nc, n).astype(np.int32)
    pe = rng.uniform(-1, 1, n).astype(np.float32)
    pth_e = rng.uniform(-1, 1, n).astype(np.float32)
    pe[::5] = 0.0
    pth_e[::7] = NAN
    return st, ind, pe, pth_e


def duplicate_course():
    """A course with repeated points (the first of equal minima must win), and points equidistant from a vehicle."""
    cx = np.float32([0, 1, 1, 1, 2, 3, 3, -1, 1, 5, 5])
    cy = np.float32([0, 0, 0, 0, 0, 0, 0, 2, 2, 0, 0])
    cyaw = np.float32([0, 0.1, 0.2, 0.3, 0, 0, -0.2, 1.0, 2.0, 3.0, -3.0])
    ck = np.float32([0, 0.5, -0.5, 1, 2, -2, 0.1, 1e-3, 100, -1e4, 3e38])
    sp = np.float32([1, 2, 3, -1, 0, 2.5, 2.5, 1, 1, 0, 0])
    st = np.float32([[1.0, 0.3, 0.0, 2.0], [2.0, 0.0, 0.0, 1.0], [0.0, 1.0, 0.5, 1.0],   # (0, 1): equidistant to 0 and 8
                     [0.5, 0.0, 0.0, 1.0], [3.0, -1.0, 0.0, -1.0], [5.0, 0.0, 3.0, 2.0], [4.0, 0.0, 0.0, 0.0],
                     [1.0, 1.0, 0.0, 1.0]]).T
    return (cx, cy, cyaw, ck, sp), np.ascontiguousarray(st)


def single_point_course():
    return tuple(np.float32([v]) for v in (2.0, -1.0, 0.7, 0.25, 1.5))


def update_cases(n: int = 4000, seed: int = 0x0DA7):
    """(state [4, n], a [n], delta [n]) for update: every |delta| range (clamped beyond MAX_STEER), |yaw| >= 120,
    negative and zero speeds, NaN and inf."""
    rng = np.random.default_rng(seed)
    st = np.stack([rng.uniform(-50, 50, n), rng.uniform(-50, 50, n), rng.uniform(-4, 4, n),
                   rng.uniform(-5, 8, n)]).astype(np.float32)
    st[2, ::9] = rng.uniform(-1e4, 1e4, st[2, ::9].size)
    st[2, 1::9] = np.float32([121.0, -120.0, 130.5, 1e6, -3e7, 119.99])[np.arange(st[2, 1::9].size) % 6]
    st[3, ::11] = 0.0
    a = rng.uniform(-3, 3, n).astype(np.float32)
    delta = rng.uniform(-1.5, 1.5, n).astype(np.float32)
    delta[::13] = np.float32(MAX_STEER)
    delta[1::13] = np.nextafter(np.float32(MAX_STEER), np.float32(1))
    delta[2::13] = -np.float32(MAX_STEER)
    delta[3::13] = np.float32(40.0)
    special = np.float32([NAN, INF, -INF])
    st[0, 5::101] = special[np.arange(st[0, 5::101].size) % 3]
    delta[7::103] = special[np.arange(delta[7::103].size) % 3]
    return np.ascontiguousarray(st), a, delta


def demo_start(nx: int):
    """The demo's course for a program and its start State(-0.0, -0.0, 0.0, 0.0)."""
    course = synth.lqr_course("demo" if nx == 4 else "demo_speed")
    return course, np.float32([-0.0, -0.0, 0.0, 0.0])
