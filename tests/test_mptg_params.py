"""Model-predictive trajectory generation away from the demo's start, speed and parameters (tests/mptg_cases.py
param_sets), at the limits of include/crb.h (limit_sets), and against a float64 model that shares no code with the
checker or the kernel.
CPU: the checker is bitwise the reference's own text on every parameter set (optimizer_traj, generate_trajectory and
generate_last_state at each base_l / ds); every limit case ends with the status it is built for, on the two sides of
its limit; the float64 model bounds the checker's trajectories, costs and converged end points.  H100: both kernels
are bitwise the checker on every set and limit case and on a 65536-problem mix; the float64 bounds hold on the
kernels' own outputs; mptg_yaw_p2p is C's exact fmod formula on all 2^32 floats and mptg_fmod_2pi is np.fmod on
1.2e7 doubles; slp_generate_path with non-default optimiser settings is bitwise the checker."""
import ctypes as C
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import mptg_cases as MC
from cpprobotics_b200 import _lib, synth
from oracle import mptg as OM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libref_mptg.so")
f32, f64 = np.float32, np.float64
EPS = 2.0 ** -24                 # float32 unit roundoff
PI, TWO_PI = np.pi, 2.0 * np.pi  # M_PI and 2 * M_PI as doubles
FILL = -7.25                     # sentinel: points beyond what is written must keep it
CAL = 2.0                        # rollout64's bounds times this hold the checker's errors with a margin of 5x
SETS = [s[0] for s in MC.param_sets()]
LIMITS = [s[0] for s in MC.limit_sets()]


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN (NaN payloads are not specified by either side)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(a.dtype.str.replace("f", "u")),
                                                     b[~nb].view(b.dtype.str.replace("f", "u")))


def lib_params(p):
    q = _lib.MptgParams()
    q.base_l, q.ds, q.max_iter, q.cost_th = p.base_l, p.ds, p.max_iter, p.cost_th
    for k in range(3):
        q.h_step[k] = p.h_step[k]
    return q


def with_max_iter(p, m):
    return OM.mptg_params(base_l=p.base_l, ds=p.ds, max_iter=m, cost_th=p.cost_th, h_step=tuple(p.h_step))


def param_set(name):
    return next(s for s in MC.param_sets() if s[0] == name)


def limit_set(name):
    return next(s for s in MC.limit_sets() if s[0] == name)


# ---- float64 model ---------------------------------------------------------------------------------------------
def wrap64(a):
    """YAW_P2P's formula in float64 (np.fmod is C's fmod: exact)."""
    with np.errstate(invalid="ignore"):
        return np.fmod(np.fmod(a + PI, TWO_PI) - TWO_PI, TWO_PI) + PI


def yaw_p2p64(y):
    """YAW_P2P of float32 y as the reference evaluates it: (float)(fmod(fmod((double)y + pi, 2pi) - 2pi, 2pi) + pi)."""
    with np.errstate(invalid="ignore"):
        return wrap64(np.asarray(y, f32).astype(f64)).astype(f32)


def rollout64(st, q, prm, steps):
    """MotionModel::update in float64 for `steps` [n] steps of each problem (the float32 loop's count), with the
    quadratic through (0, s0), (horizon / 2, s1), (horizon, s2) in closed form and t = k * dt.  Returns the points
    [K, 3, n] (yaw unwrapped) and, per step, bounds on how far a float32 evaluation of the same model can be from it:
    position [K, n] and yaw [K, n].  The bounds accumulate, per step, the roundings of the state update, of kp
    (coefficients, the float time's k-fold accumulated error) and their effect through tan(kp), and the position error
    that a heading error makes over v * dt."""
    x, y, yaw, v = (a.astype(f64).copy() for a in st)
    d, s0, s1, s2 = (a.astype(f64) for a in q)
    with np.errstate(all="ignore"):
        H = d / v
        dt = H / (d / f64(prm.ds))
        c2, c1, c0 = s0, (-3.0 * s0 + 4.0 * s1 - s2) / H, 2.0 * (s0 - 2.0 * s1 + s2) / (H * H)
        vl = v / f64(prm.base_l)
        S = np.abs(s0) + np.abs(s1) + np.abs(s2)
        K = int(steps.max()) if steps.size else 0
        pts = np.full((K, 3, x.size), np.nan)
        bp, by = np.zeros((K, x.size)), np.zeros((K, x.size))
        ep, ey = np.zeros(x.size), np.zeros(x.size)
        for k in range(K):
            live = k < steps
            t = k * dt
            kp = (c0 * t + c1) * t + c2
            dkp = EPS * (300.0 * S + 4.0 * (np.abs(c0) * t * t + np.abs(c1) * t + np.abs(c2))) \
                + np.abs(2.0 * c0 * t + c1) * (k + 3) * EPS * t
            tn = np.tan(kp)
            dyaw = vl * tn * dt
            ddyaw = 8.0 * EPS * np.abs(dyaw) + np.abs(vl) * dt * dkp / np.cos(kp) ** 2
            ep = ep + v * dt * ey + EPS * (4.0 * np.maximum(np.abs(x), np.abs(y)) + 8.0 * v * dt)
            ey = ey + ddyaw + 2.0 * EPS * (PI + np.abs(dyaw) + (np.abs(yaw) if k == 0 else 0.0))
            x = np.where(live, x + v * np.cos(yaw) * dt, x)
            y = np.where(live, y + v * np.sin(yaw) * dt, y)
            yaw = np.where(live, yaw + dyaw, yaw)
            pts[k] = (x, y, yaw)
            bp[k], by[k] = ep, ey
    return pts, CAL * bp, CAL * by


def cost64(pt, tg):
    """The cost of a float32 end point pt [3, n] against tg [3, n] in float64: the yaw difference is the float32
    subtraction the reference makes, wrapped exactly."""
    ex = tg[0].astype(f64) - pt[0].astype(f64)
    ey = tg[1].astype(f64) - pt[1].astype(f64)
    eyaw = wrap64((tg[2] - pt[2]).astype(f64))
    return np.sqrt(ex * ex + ey * ey + eyaw * eyaw), np.abs(ex) + np.abs(ey) + np.abs(eyaw)


def check_rollouts(st, q, prm, traj, steps, max_pts):
    """The float32 points traj [3*max_pts, n] of the roll-outs of q (steps [n] each) against the float64 model,
    within its bound, on every finite trajectory; and the step count against distance / ds.  A base_l, ds or v in the
    wrong place (v * base_l, ds / v, ...), a wrong sign or a step more or less moves points by far more than the
    bound.  Returns the largest error / bound seen and the number of trajectories checked."""
    m = min(int(steps.max()) if steps.size else 0, max_pts)
    if m == 0:
        return 0.0, 0
    pts, bp, by = rollout64(st, q, prm, np.minimum(steps, m))
    got = traj[:3 * m].reshape(m, 3, -1).astype(f64)
    k = np.arange(m)[:, None]
    shown = k < np.minimum(steps, m)[None, :]
    fin = np.isfinite(got).all(axis=1) | ~shown
    ok = fin.all(axis=0) & np.isfinite(bp).all(axis=0) & np.isfinite(by).all(axis=0) & (steps > 0)
    worst = 0.0
    if ok.any():
        with np.errstate(invalid="ignore"):
            e_pos = np.maximum(np.abs(got[:, 0] - pts[:, 0]), np.abs(got[:, 1] - pts[:, 1]))
            e_yaw = np.abs(wrap64(got[:, 2] - pts[:, 2]))
            r = np.maximum(e_pos / np.maximum(bp, 1e-300), e_yaw / np.maximum(by, 1e-300))
        r = np.where(shown & ok[None, :], r, 0.0)
        worst = float(r.max())
        assert worst <= 1.0, ("float64 bound", np.unravel_index(np.argmax(r), r.shape), worst)
    # the float loop `t += horizon / n` takes ceil(distance / ds) steps, give or take what the rounding of n, dt and
    # the accumulated t (k^2 eps steps after k steps) moves across an integer
    n = q[0].astype(f64) / f64(prm.ds)
    sel = ok & np.isfinite(n)
    s, n = steps[sel].astype(f64), n[sel]
    slack = 2.0 * (s + 6.0) * (s + 6.0) * EPS
    dev = np.abs(s - np.ceil(n))
    assert (dev <= np.floor(slack) + (np.abs(n - np.round(n)) <= slack)).all(), "step count"
    return worst, int(ok.sum())


def check_result(o, o_prev, st, tg, prm, max_pts):
    """For every problem that returns a trajectory: the returned cost is the float64 cost of the trajectory's last
    point, and the float64 roll-out of the parameter that trajectory belongs to (the returned one when CONVERGED, the
    one before the last update when MAX_ITER_REACHED, i.e. o_prev's, from max_iter - 1) stays within the float64 bound
    of the trajectory and its cost; a CONVERGED end point lies within cost_th plus that bound of the target."""
    st_ = o["status"]
    has = ((st_ == OM.CONVERGED) | (st_ == OM.MAX_ITER_REACHED)) & (o["traj_len"] > 0)
    q = np.where(st_ == OM.CONVERGED, o["param"], o_prev["param"])
    idx = np.flatnonzero(has)
    if not idx.size:
        return 0.0, 0
    cols = lambda a: np.ascontiguousarray(a[:, idx])   # noqa: E731
    steps = o["traj_len"][idx]
    worst, n_ok = check_rollouts(cols(st), cols(q), prm, cols(o["traj"]), steps, max_pts)
    pts, bp, by = rollout64(cols(st), cols(q), prm, steps)
    last = pts[steps - 1, :, np.arange(idx.size)].T
    ep, ey = bp[steps - 1, np.arange(idx.size)], by[steps - 1, np.arange(idx.size)]
    cost = o["cost"][idx].astype(f64)
    tgi = cols(tg)
    with np.errstate(invalid="ignore"):
        ex, eyy = tgi[0] - last[0], tgi[1] - last[1]
        eyaw = np.abs(wrap64(tgi[2].astype(f64) - last[2]))
        c_model = np.sqrt(ex * ex + eyy * eyy + eyaw * eyaw)
        tol_model = 2.0 * ep + ey + EPS * (np.abs(tgi[2].astype(f64)) + np.abs(last[2]) + 4.0 * c_model + 8.0)
    fin = np.isfinite(c_model) & np.isfinite(tol_model) & np.isfinite(cost)   # float64 does not overflow
    assert (np.abs(cost[fin] - c_model[fin]) <= tol_model[fin]).all(), "cost against the float64 roll-out"
    conv = fin & (st_[idx] == OM.CONVERGED)
    assert (c_model[conv] < f64(f32(prm.cost_th)) + tol_model[conv]).all(), "converged end point"
    # the returned cost against the returned trajectory's own last point, where it is stored
    inside = np.flatnonzero(steps <= max_pts)
    k = steps[inside] - 1
    tr = o["traj"][:, idx[inside]]
    lp = np.stack([tr[3 * k + j, np.arange(inside.size)] for j in range(3)])
    c64, scale = cost64(lp, tgi[:, inside])
    ci = cost[inside]
    fin = np.isfinite(c64)
    assert same(np.isnan(ci[~fin]), np.isnan(c64[~fin]))
    assert (np.abs(ci[fin] - c64[fin]) <= 2.0 * EPS * (scale[fin] + c64[fin]) + 1e-45).all(), "cost of last point"
    return worst, n_ok


# ---- CPU ------------------------------------------------------------------------------------------------------
def _ref_lib():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle -f mptg.mk)")
    import golden.make_mptg_golden as G
    return C.CDLL(REF), G


def test_sets_reach_what_they_are_for():
    got = {name: OM.optimize(st, tg, pa, prm) for name, st, tg, pa, prm in MC.param_sets()}
    st = param_set("start_yaw")[1]
    assert (np.abs(st[2]) > 3 * np.pi).mean() > 0.8 and f32(np.abs(st[2]).max()) == MC.BELOW_120
    assert (got["start_yaw"]["status"] == OM.CONVERGED).mean() > 0.9
    assert np.abs(param_set("far_start")[1][:2]).max() > 9000.0
    v = param_set("speed")[1][3]
    assert v.min() < 0.15 and v.max() > 15.0
    for name in ("base_l_0.3", "base_l_-1", "far_start", "speed"):
        assert (got[name]["status"] == OM.CONVERGED).mean() > 0.9, name
    assert (got["base_l_overflow"]["status"] == OM.MAX_ITER_REACHED).any()
    assert (got["ds_beyond_distance"]["traj_len"] == 1).all()
    assert (got["h_step_large"]["status"] == OM.OUT_OF_RANGE).any()
    assert (got["cost_th_negative"]["status"] == OM.MAX_ITER_REACHED).all()
    assert (got["cost_th_large"]["iters"] == 0).all()
    assert (got["fixed_point_1000"]["iters"] == OM.MAX_ITER).all()
    d = got["diverge_1000"]
    assert ((d["status"] == OM.MAX_ITER_REACHED) & (d["iters"] == OM.MAX_ITER)).any()
    assert len(set(d["status"].tolist())) >= 3 and d["iters"].max() > 100


@pytest.mark.parametrize("case", SETS)
def test_checker_is_bitwise_the_reference_text(case):
    L, G = _ref_lib()
    name, st, tg, pa, prm = param_set(case)
    o = OM.optimize(st, tg, pa, prm, max_pts=128)
    sel = np.flatnonzero(o["status"] <= OM.MAX_ITER_REACHED)   # the reference's UB / endless loops are not fed to it
    sub = [np.ascontiguousarray(a[:, sel]) for a in (st, tg, pa)]
    q, traj, tl, cost = G.reference(L, *sub, prm, 128)
    assert same(o["param"][:, sel], q) and same(o["traj"][:, sel], traj)
    assert np.array_equal(o["traj_len"][sel], tl) and same(o["cost"][sel], cost)
    assert len(sel) >= 2
    # generate_trajectory / generate_last_state at this base_l and ds: of the initial and the returned parameters
    for p in (pa, o["param"]):
        g = OM.generate(st, p, prm, max_pts=128)
        for i in np.flatnonzero(g["status"] == 0)[:24]:
            s, qi = (np.ascontiguousarray(a[:, i], f32) for a in (st, p))
            tr, last, k = np.full(3 * 128, np.nan, f32), np.zeros(3, f32), C.c_int(0)
            L.ref_mptg_generate(s.ctypes.data, qi.ctypes.data, C.c_float(prm.base_l), C.c_float(prm.ds),
                                tr.ctypes.data, 128, C.byref(k), last.ctypes.data)
            assert k.value == g["traj_len"][i] and same(tr, g["traj"][:, i]) and same(last, g["last"][:, i]), i


def check_limit(name, st, tg, pa, prm, want, opt, gen):
    """The limit case ends with its statuses, and its pairs are the two sides of one limit (opt / gen: the optimizer
    and generate_trajectory, either the checker's or the kernels')."""
    o = opt(st, tg, pa, prm)
    assert o["status"].tolist() == list(want), (name, o["status"])
    adjacent = lambda a, b: np.nextafter(f32(a), f32(np.inf) if b > a else f32(-np.inf)) == b   # noqa: E731
    one = lambda s, q: gen(np.ascontiguousarray(s, f32).reshape(4, 1),   # noqa: E731
                           np.ascontiguousarray(q, f32).reshape(4, 1), prm)
    h0 = f32(prm.h_step[0])
    if name == "cap_nominal":
        assert adjacent(pa[0, 0], pa[0, 1])
        g = gen(st, pa, prm)
        assert g["traj_len"].tolist() == [OM.MAX_STEPS, 0] and g["status"].tolist() == [0, OM.STEP_CAP]
    elif name == "cap_jacobian":       # both nominals complete; distance + h_step[0] crosses between them
        assert adjacent(pa[0, 0], pa[0, 1])
        assert gen(st, pa, prm)["status"].tolist() == [0, 0]
        up = pa.copy()
        up[0] += h0
        g = gen(st, up, prm)
        assert g["status"].tolist() == [0, OM.STEP_CAP] and g["traj_len"][0] == OM.MAX_STEPS
        assert o["iters"].tolist() == [1, 0]
    elif name == "cap_line_search":    # the same parameter (so the same Jacobian roll-outs), targets one ulp apart
        assert same(pa[:, 0], pa[:, 1]) and adjacent(tg[0, 0], tg[0, 1])
        dn, up = pa.copy(), pa.copy()
        dn[0] -= h0
        up[0] += h0
        assert gen(st, dn, prm)["status"].tolist() == [0, 0] and gen(st, up, prm)["status"].tolist() == [0, 0]
        assert o["iters"].tolist() == [1, 0]
    elif name == "steer_120":
        assert pa[1].tolist() == [MC.BELOW_120, 120.0, -MC.BELOW_120, -120.0]
        assert gen(st, pa, prm)["status"].tolist() == [0, OM.OUT_OF_RANGE, 0, OM.OUT_OF_RANGE]
    elif name == "start_yaw_120":
        assert st[2].tolist() == [MC.BELOW_120, 120.0, -MC.BELOW_120, -120.0]
        assert gen(st, pa, prm)["status"].tolist() == [0, OM.OUT_OF_RANGE, 0, OM.OUT_OF_RANGE]
    elif name == "cap_and_out_of_range":   # the six Jacobian roll-outs of the first iteration
        q = pa[:, 0]
        six = []
        for row, h in ((0, h0), (2, f32(prm.h_step[1])), (3, f32(prm.h_step[2]))):
            for sg in (1, -1):
                p = q.copy()
                p[row] = p[row] + h if sg > 0 else p[row] - h
                six.append(int(one(st[:, 0], p)["status"][0]))
        assert int(one(st[:, 0], q)["status"][0]) == 0
        assert six == [OM.STEP_CAP, 0, 0, 0, OM.OUT_OF_RANGE, 0], six
    return o


def _cpu_opt(st, tg, pa, prm, max_pts=0):
    return OM.optimize(st, tg, pa, prm, max_pts=max_pts, traj_fill=FILL)


def _cpu_gen(st, pa, prm, max_pts=0):
    return OM.generate(st, pa, prm, max_pts=max_pts, traj_fill=FILL)


@pytest.mark.parametrize("case", LIMITS)
def test_limit_cases_end_with_their_status(case):
    check_limit(*limit_set(case), _cpu_opt, _cpu_gen)


def test_float64_model_bounds_the_checker():
    """The float64 bound holds on every finite trajectory of every set with at least a 4x margin (its calibration),
    on generate_trajectory of the initial and returned parameters and on optimizer_traj's returned trajectory, cost
    and converged end point."""
    worst, n = 0.0, 0
    for name, st, tg, pa, prm, *_ in MC.param_sets() + MC.limit_sets():
        mp = 16400 if name.startswith("cap") else 6000
        o = OM.optimize(st, tg, pa, prm, max_pts=mp)
        prev = OM.optimize(st, tg, pa, with_max_iter(prm, max(prm.max_iter - 1, 0)), max_pts=mp)
        w, k = check_result(o, prev, st, tg, prm, mp)
        worst, n = max(worst, w), n + k
        for p in (pa, o["param"]) if not same(pa, o["param"]) else (pa,):
            g = OM.generate(st, p, prm, max_pts=mp)
            w, k = check_rollouts(st, p, prm, g["traj"], np.where(g["status"] == 0, g["traj_len"], 0), mp)
            worst, n = max(worst, w), n + k
    assert n > 2000 and 0.0 < worst <= 0.25, (n, worst)


def test_float64_model_catches_misplaced_parameters():
    """The bound is tight enough to see v * base_l for v / base_l, a flipped yaw increment, a ds 5% off and a step
    fewer than the float32 loop takes: each leaves the bound of the checker's trajectories.  (v itself cancels from
    the geometry: a step is v * dt = ds long and turns by v / base_l * tan(kp) * dt = ds / base_l * tan(kp).)"""
    name, st, tg, pa, prm = param_set("base_l_0.3")
    q = OM.optimize(st, tg, pa, prm)["param"]
    g = OM.generate(st, q, prm, max_pts=400)
    steps = np.where(g["status"] == 0, g["traj_len"], 0)
    assert check_rollouts(st, q, prm, g["traj"], steps, 400)[1] == st.shape[1]
    P = lambda **k: OM.mptg_params(**dict(dict(base_l=prm.base_l, ds=prm.ds), **k))   # noqa: E731
    for p, k in ((P(base_l=1.0 / prm.base_l), steps), (P(base_l=-prm.base_l), steps), (P(ds=prm.ds * 1.05), steps),
                 (prm, steps - 1)):
        with pytest.raises(AssertionError):
            check_rollouts(st, q, p, g["traj"], k, 400)


def test_yaw_p2p_formula_is_the_checkers_on_selected_floats():
    """The float64 YAW_P2P above is the checker's around every multiple of pi below 120 and at +-4 pi: one step of
    generate_last_state with zero steering leaves YAW_P2P(start yaw)."""
    ys = [f32(0.0), f32(-0.0), f32(4 * np.pi), f32(-4 * np.pi)]
    for k in range(-38, 39):
        c = f32(k * np.pi)
        ys += [np.nextafter(c, f32(-np.inf)), c, np.nextafter(c, f32(np.inf))]
    ys = np.float32([y for y in ys if abs(y) < 120.0])
    st = np.zeros((4, ys.size), f32)
    st[2], st[3] = ys, 1.0
    pa = np.zeros((4, ys.size), f32)
    pa[0] = 1.0
    g = OM.generate(st, pa, OM.mptg_params(ds=2.0, base_l=1.0), max_pts=1)
    assert (g["traj_len"] == 1).all() and same(g["last"][2], yaw_p2p64(ys))


# ---- H100 -----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, f32)).to("cuda:0")


def _gpu_opt(engine, st, tg, pa, prm, max_pts=0):
    import torch
    n = st.shape[1]
    sd, td, qd = _dev(st), _dev(tg), _dev(pa)
    traj = torch.full((3 * max_pts, n), FILL, dtype=torch.float32, device="cuda:0")
    i32 = [torch.empty(n, dtype=torch.int32, device="cuda:0") for _ in range(3)]
    cost = torch.empty(n, dtype=torch.float32, device="cuda:0")
    engine.mptg_optimize(sd, td, qd, lib_params(prm), traj=traj if max_pts else None, traj_len=i32[0], cost=cost,
                         status=i32[1], iters=i32[2])
    torch.cuda.synchronize()
    return dict(param=qd.cpu().numpy(), traj=traj.cpu().numpy(), traj_len=i32[0].cpu().numpy(),
                cost=cost.cpu().numpy(), status=i32[1].cpu().numpy(), iters=i32[2].cpu().numpy())


def _gpu_gen(engine, st, pa, prm, max_pts=0):
    import torch
    n = st.shape[1]
    traj = torch.full((3 * max_pts, n), FILL, dtype=torch.float32, device="cuda:0")
    tl, status = (torch.empty(n, dtype=torch.int32, device="cuda:0") for _ in range(2))
    last = torch.empty((3, n), dtype=torch.float32, device="cuda:0")
    engine.mptg_generate_trajectory(_dev(st), _dev(pa), lib_params(prm), traj=traj if max_pts else None,
                                    traj_len=tl, last=last, status=status)
    torch.cuda.synchronize()
    return dict(traj=traj.cpu().numpy(), traj_len=tl.cpu().numpy(), last=last.cpu().numpy(),
                status=status.cpu().numpy())


OPT_KEYS = ("param", "traj", "traj_len", "cost", "status", "iters")
GEN_KEYS = ("traj", "traj_len", "last", "status")


def _same_keys(r, o, keys):
    return [k for k in keys if not same(r[k], o[k])]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SETS + LIMITS)
def test_gpu_is_bitwise_the_checker(engine, case):
    is_limit = case in LIMITS
    s = limit_set(case) if is_limit else param_set(case)
    name, st, tg, pa, prm = s[:5]
    for mp in (0, 48):
        o, r = _cpu_opt(st, tg, pa, prm, mp), _gpu_opt(engine, st, tg, pa, prm, mp)
        assert not _same_keys(r, o, OPT_KEYS), (case, mp, _same_keys(r, o, OPT_KEYS))
        for p in (pa, o["param"]):
            g, rg = _cpu_gen(st, p, prm, mp), _gpu_gen(engine, st, p, prm, mp)
            assert not _same_keys(rg, g, GEN_KEYS), (case, mp, _same_keys(rg, g, GEN_KEYS))
    if is_limit:   # the kernels on the two sides of each limit
        check_limit(*s, lambda *a: _gpu_opt(engine, *a), lambda *a: _gpu_gen(engine, *a))


def mixed(n, seed=0x3A7):
    """n problems, each drawn (by index) from a random parameter set or from synth.mptg_inputs (which has every
    status's corner cases), all run with the demo's parameters."""
    pool = [s[1:4] for s in MC.param_sets()] + [synth.mptg_inputs(4096, seed=seed)]
    idx = np.arange(n, dtype=np.uint64)
    which = np.minimum((synth.u01(seed, 1, idx) * len(pool)).astype(np.int64), len(pool) - 1)
    u = synth.u01(seed, 2, idx)
    out = [np.empty((4, n), f32), np.empty((3, n), f32), np.empty((4, n), f32)]
    for j, (st, tg, pa) in enumerate(pool):
        sel = which == j
        col = np.minimum((u[sel] * st.shape[1]).astype(np.int64), st.shape[1] - 1)
        for o, a in zip(out, (st, tg, pa)):
            o[:, sel] = a[:, col]
    return tuple(out)


@pytest.mark.gpu
def test_gpu_mixed_sets_over_many_waves(engine):
    n, mp = 65536 + 77, 160
    st, tg, pa = mixed(n)
    prm = OM.mptg_params()
    o = _cpu_opt(st, tg, pa, prm, mp)
    assert (np.bincount(o["status"], minlength=5) > 0).all()
    assert (o["traj_len"] > mp).any() and ((o["traj_len"] > 1) & (o["traj_len"] < 40)).any()
    for m in (0, 1, 40, mp):
        r = _gpu_opt(engine, st, tg, pa, prm, m)
        want = dict(o, traj=np.ascontiguousarray(o["traj"][:3 * m]))
        assert not _same_keys(r, want, OPT_KEYS), (m, _same_keys(r, want, OPT_KEYS))
    g, rg = _cpu_gen(st, pa, prm, 40), _gpu_gen(engine, st, pa, prm, 40)
    assert not _same_keys(rg, g, GEN_KEYS)


@pytest.mark.gpu
def test_gpu_float64_model_bounds_the_kernels(engine):
    """The float64 bounds of test_float64_model_bounds_the_checker on the kernels' own outputs (the parameter before
    the last update from a second launch with max_iter - 1)."""
    n = 0
    for name, st, tg, pa, prm, *_ in MC.param_sets() + MC.limit_sets():
        mp = 16400 if name.startswith("cap") else 6000
        o = _gpu_opt(engine, st, tg, pa, prm, mp)
        prev = _gpu_opt(engine, st, tg, pa, with_max_iter(prm, max(prm.max_iter - 1, 0)), mp)
        n += check_result(o, prev, st, tg, prm, mp)[1]
        for p in (pa, o["param"]):
            g = _gpu_gen(engine, st, p, prm, mp)
            n += check_rollouts(st, p, prm, g["traj"], np.where(g["status"] == 0, g["traj_len"], 0), mp)[1]
    assert n > 2000


CENSUS_CU = r"""
// The shipped mptg_yaw_p2p and mptg_fmod_2pi of crb_mptg.cu (anonymous namespace: included, not copied) on the
// device; crb_mptg.cu's host helpers resolve against libcrb.
#include "crb_mptg.cu"

__global__ void yaw_p2p_bits(unsigned lo, unsigned long long count, float* out) {
  for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x)
    out[k] = mptg_yaw_p2p(__uint_as_float((unsigned)(lo + k)));
}
__global__ void fmod_2pi(const double* in, long long n, double* out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
    out[k] = mptg_fmod_2pi(in[k]);
}

extern "C" {
// mptg_yaw_p2p of the float with bit pattern lo + k into host[k], k < count: 0 or a CUDA error code
int census_yaw_p2p(unsigned lo, unsigned long long count, float* host) {
  float* d = nullptr;
  cudaError_t e = cudaMalloc(&d, count * sizeof(float));
  if (e == cudaSuccess) {
    yaw_p2p_bits<<<2048, 256>>>(lo, count, d);
    e = cudaMemcpy(host, d, count * sizeof(float), cudaMemcpyDeviceToHost);
  }
  cudaFree(d);
  return (int)e;
}
// mptg_fmod_2pi of in[k] into out[k], k < n
int census_fmod_2pi(const double* in, long long n, double* out) {
  double* d = nullptr;
  cudaError_t e = cudaMalloc(&d, 2 * n * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(d, in, n * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    fmod_2pi<<<2048, 256>>>(d, n, d + n);
    e = cudaMemcpy(out, d + n, n * sizeof(double), cudaMemcpyDeviceToHost);
  }
  cudaFree(d);
  return (int)e;
}
}
"""


@pytest.fixture(scope="module")
def census_lib(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    d = tmp_path_factory.mktemp("mptg_census")
    (d / "census.cu").write_text(CENSUS_CU)
    so = d / "libcensus.so"
    libdir = os.path.dirname(_lib.LIB_PATH)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                           "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "cpprobotics_b200", "csrc"),
                           str(d / "census.cu"), "-o", str(so), "-L", libdir, "-lcrb", "-Xlinker", f"-rpath,{libdir}"])
    L = C.CDLL(str(so))
    L.census_yaw_p2p.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
    L.census_fmod_2pi.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return L


def _yaw_mismatches(lo, got):
    """Patterns lo .. lo + len(got) - 1 where got differs from the float64 YAW_P2P (NaN equals NaN)."""
    y = np.arange(lo, lo + got.size, dtype=np.uint64).astype(np.uint32).view(f32)
    want = yaw_p2p64(y)
    bad = (got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))
    return int(bad.sum()), y[bad][:4].tolist()


@pytest.mark.gpu
def test_gpu_yaw_p2p_census_against_float64(census_lib):
    """mptg_yaw_p2p on every float32 bit pattern against the float64 formula with np.fmod (C's exact fmod): the
    general-fmod branch (|y + pi| >= 4 pi), the Sterbenz branch and the identity branch.  numpy's ufuncs release the
    GIL, so the host side runs on a thread pool."""
    chunk, sub = 1 << 26, 1 << 22
    bad, examples = 0, []
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        pending = []
        for lo in range(0, 1 << 32, chunk):
            got = np.empty(chunk, f32)
            assert census_lib.census_yaw_p2p(lo, chunk, got.ctypes.data) == 0
            done, pending = pending, [ex.submit(_yaw_mismatches, lo + j, got[j:j + sub]) for j in range(0, chunk, sub)]
            for f in done:
                b, e = f.result()
                bad, examples = bad + b, examples + e
        for f in pending:
            b, e = f.result()
            bad, examples = bad + b, examples + e
    assert bad == 0, (bad, examples[:8])


def fmod_inputs(n=12_000_000, seed=0xF0D):
    """Doubles for fmod(x, 2 pi): random bit patterns (every exponent, NaN and inf included), k * 2 pi +- a few ulps
    for k up to 2^40, 2 pi and 4 pi and their neighbours, and magnitudes log-uniform up to 1e308; both signs."""
    rng = np.random.default_rng(seed)
    q = n // 4
    bits = rng.integers(0, 2 ** 64, q, dtype=np.uint64, endpoint=False).view(f64)
    k = np.concatenate([rng.integers(1, 64, q // 2), rng.integers(1, 2 ** 40, q - q // 2)]).astype(f64)
    mult = k * TWO_PI
    near = (mult.view(np.int64) + rng.integers(-4, 5, q)).view(f64)
    mag = 10.0 ** rng.uniform(-300, 308, q) * rng.choice([-1.0, 1.0], q)
    edges = []
    for c in (TWO_PI, 2 * TWO_PI, 3 * TWO_PI, PI, 1e308, np.finfo(f64).max, np.finfo(f64).tiny, 5e-324):
        b = np.array(c, f64).view(np.int64)
        edges += list((b + np.arange(-8, 9)).view(f64))
    x = np.concatenate([bits, near, mag, np.float64(edges), [0.0, np.inf, np.nan]])
    return np.concatenate([x, -x])


@pytest.mark.gpu
def test_gpu_fmod_2pi_is_np_fmod(census_lib):
    x = fmod_inputs()
    got = np.empty_like(x)
    assert census_lib.census_fmod_2pi(x.ctypes.data, x.size, got.ctypes.data) == 0
    with np.errstate(invalid="ignore"):
        want = np.fmod(x, TWO_PI)
    bad = np.flatnonzero(~((got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))))
    assert bad.size == 0, (bad.size, x[bad[:4]].tolist(), got[bad[:4]].tolist(), want[bad[:4]].tolist())
    assert x.size > 10 ** 7 and (np.abs(x) >= 2 * TWO_PI).mean() > 0.4


@pytest.mark.gpu
def test_gpu_generate_path_with_changed_optimizer_parameters(engine):
    """slp_generate_path, the one consumer of the optimizer outside crb_mptg.cu, with every optimizer parameter and
    the start speed away from generate_path's own: bitwise oracle/slp.py's generate_path."""
    from oracle import slp as OS
    import slp_cases as SC
    tb = SC.table()
    prm = OM.mptg_params(base_l=1.7, ds=0.07, max_iter=60, cost_th=0.05, h_step=(0.4, 0.01, 0.03))
    for kind in (OS.UNIFORM, OS.BIASED, OS.LANE):
        fields, qp = synth.slp_inputs(200, kind, seed=0x5E + kind)
        t = OS.sample(SC.sampler_of(fields), qp)["target"]
        t = np.ascontiguousarray(t[:, np.isfinite(t).all(axis=0)][:, :2000])
        for v in (1.3, 7.5):
            o = OS.generate_path(t, tb, max_pts=96, params=prm, v=v)
            r = engine.slp_generate_path(_dev(t), _dev(tb), params=lib_params(prm), v=v, max_pts=96)
            r = {k: x.cpu().numpy() for k, x in r.items()}
            for k in ("param", "traj", "traj_len", "cost", "status", "iters", "row"):
                assert same(r[k], o[k]), (kind, v, k)
            assert (o["status"] == OM.CONVERGED).any()
