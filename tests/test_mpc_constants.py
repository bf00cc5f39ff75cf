"""The MPC path away from the reference's constants.

The reference's weights come in equal pairs and every other GPU test runs at its dt, wb and bounds, so a weight
meeting the wrong channel in the parameter fill, or a constant ignored by the plant step, would pass them.  Here:
- CPU: the oracle against the float64 statement and SciPy at three parameter sets (tests/mpc_cases.py) and with
  the lower speed bound active; the oracle's update() / calc_ref_trajectory() with constants; synth's lookup at
  the roundf edge; argument validation without a device.
- GPU: the solver bit for bit against the oracle at those sets on batches of at least three waves of problems for
  every horizon the resident-slot kernel's geometry depends on, at every horizon 2..32, at the loop limits, with
  problems that retire at refill, with each output alone and through the _host and hinted entries; update() and
  calc_ref_trajectory() bit for bit at those constants; a closed loop on the device in lockstep with the oracle's.
Every GPU output is pre-filled with a NaN / -7 sentinel, so a problem the scheduler skipped shows up."""
import ctypes as C

import numpy as np
import pytest

import mpc_cases as MC
import ref_mpc as M
from cpprobotics_b200 import _lib, mpc_default_params, synth
from oracle import oracle as O

OUTS = ("status", "iters", "u0", "cost", "sol")
SENTINEL = -7


def oparams(over=None, **kw):
    return O.mpc_params(**dict(over or {}, **kw))


def gparams(over=None, **kw):
    return MC.set_params(mpc_default_params(), dict(over or {}, **kw))


def dt_of(over):
    return O.plant_constant(oparams(over), "dt")


# ---- CPU: the oracle with constants -------------------------------------------------------------------------
def test_oracle_constant_entries_equal_the_macro_entries_at_the_defaults():
    """plant_update / calc_ref_trajectory with the default parameters go through the new entries that take the
    constants; they must give the bits of the entries with the macros compiled in."""
    rng = np.random.default_rng(5)
    prm = oparams()
    for _ in range(400):
        st = np.array([rng.uniform(-100, 100), rng.uniform(-100, 100), rng.uniform(-3, 3), rng.uniform(-6, 16)],
                      np.float32)
        a, d = np.float32(rng.uniform(-3, 3)), np.float32(rng.uniform(-1.2, 1.2))
        assert np.array_equal(O.plant_update(st, a, d), O.plant_update(st, a, d, params=prm))
    course = synth.mpc_course()
    stn, pind = synth.mpc_states(300, seed=3, course=course)
    for i in range(300):
        for dl in (0.5, 1.0):
            x0, t0 = O.calc_ref_trajectory(stn[:, i], *course, dl, 32, int(pind[i]))
            x1, t1 = O.calc_ref_trajectory(stn[:, i], *course, dl, 32, int(pind[i]), params=prm)
            assert t0 == t1 and np.array_equal(x0, x1)
    # the promotion rule: the macro rounded to float is the macro, anything else is the float's own value
    assert O.plant_constant(prm, "dt") == 0.2 and O.plant_constant(prm, "max_steer") == 45.0 / 180 * np.pi
    up = np.nextafter(np.float32(0.2), np.float32(1.0))
    assert O.plant_constant(oparams(dt=up), "dt") == float(up) != 0.2


@pytest.mark.parametrize("name", ["B", "S"])
def test_oracle_plant_update_matches_float64_at_constants(name):
    over = MC.SETS[name]
    prm = oparams(over)
    k = {f: O.plant_constant(prm, f) for f in ("max_steer", "dt", "wb", "max_speed", "min_speed")}
    rng = np.random.default_rng(1)
    for _ in range(300):
        st = np.array([rng.uniform(-100, 100), rng.uniform(-100, 100), rng.uniform(-3, 3), rng.uniform(-2, 6)],
                      np.float32)
        a, d = np.float32(rng.uniform(-4, 4)), np.float32(rng.uniform(-1.0, 1.0))
        got = O.plant_update(st, a, d, params=prm)
        dd = min(max(float(d), -k["max_steer"]), k["max_steer"])
        x, y, yaw, v = (float(s) for s in st)
        want = np.array([x + v * np.cos(yaw) * k["dt"], y + v * np.sin(yaw) * k["dt"],
                         yaw + v / k["wb"] * np.tan(dd) * k["dt"],
                         min(max(v + float(a) * k["dt"], k["min_speed"]), k["max_speed"])])
        assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("name", ["W", "B", "S", "REVERSE"])
def test_oracle_matches_float64_statement_at_constants(name):
    """The C oracle (float32, the GPU's specification) against the float64 box-DDP statement and, for a few
    problems, the reference NLP solved by SciPy.  REVERSE asks for -2 m/s with min_speed = -1: the lower speed
    bound binds at every stage."""
    T = 20
    over = dict(MC.REVERSE) if name == "REVERSE" else MC.SETS[name]
    if name == "REVERSE":
        st, xref = MC.reverse_case(16, T)
    else:
        st, xref = MC.case(48, T, dt=dt_of(over))
    n = st.shape[1]
    r = O.mpc_solve_batched(st, xref, T, oparams(over))
    assert (r["status"] == 0).all() and r["iters"].max() <= 30
    p64 = MC.f64_params(over)
    eu, ec = [], []
    for i in range(n):
        ref = M.box_ilqr(st[:, i].astype(float), xref[:, i].reshape(T, 4).T.astype(float), dict(p64, j_tol=0.0))
        eu.append(max(abs(ref["U"][1, 0] - r["u0"][0, i]), abs(ref["U"][0, 0] - r["u0"][1, i])))
        ec.append(abs(ref["cost"] - r["cost"][i]) / ref["cost"])
    eu, ec = np.array(eu), np.array(ec)
    assert np.median(eu) < 1e-5 and eu.max() < 1e-3 and ec.max() < 1e-5
    for i in range(2):
        ref = M.nlp_solve_scipy(st[:, i].astype(float), xref[:, i].reshape(T, 4).T.astype(float), p64)
        assert abs(ref["cost"] - r["cost"][i]) <= 2e-4 * ref["cost"]
        assert abs(ref["U"][1, 0] - r["u0"][0, i]) < 5e-3 and abs(ref["U"][0, 0] - r["u0"][1, i]) < 5e-3
    v = r["sol"][3 * T:4 * T]
    vmin, vmax = np.float32(over.get("min_speed", -20.0 / 3.6)), np.float32(over.get("max_speed", 55.0 / 3.6))
    inside = (st[3] >= vmin) & (st[3] <= vmax)        # agents that start inside the speed bounds stay inside
    assert (v[:, inside] >= vmin).all() and (v[:, inside] <= vmax).all()
    if name == "B":
        assert (~inside).sum() >= 5                   # starts above max_speed: the bound is active
    if name == "REVERSE":
        assert (v[-1] == vmin).all()          # the bound is active at the end of every horizon


def test_rounding_edge_of_the_lookup():
    """calc_ref_trajectory rounds travel / dl with roundf (:150).  At q = 0.49999997f, floorf(q + 0.5f) is 1 and
    roundf(q) is 0: synth's vectorised lookup (every MPC test's and bench.py's xref) must take roundf's side."""
    course = synth.mpc_course()
    found = 0
    for DT in (0.2, dt_of(MC.B), dt_of(MC.S)):
        for dl in (1.0, 0.5, 0.3):
            edges = MC.rounding_edge_speeds(dl, DT)
            found += len(edges)
            if not edges:
                continue
            st, pind = MC.edge_states([v for _, v in edges])
            xn, tn = synth.mpc_xref_numpy(st, pind, 32, course=course, dl=dl, dt=DT)
            prm = oparams(dt=np.float32(DT))
            for i in range(st.shape[1]):
                xo, to = O.calc_ref_trajectory(st[:, i], *course, dl, 32, int(pind[i]), params=prm)
                assert to == tn[i] and np.array_equal(xo.reshape(-1), xn[:, i]), (DT, dl, edges[i])
    assert found >= 60     # 84 stages with such a speed on this course


# ---- CPU: validation -----------------------------------------------------------------------------------------
def _invalid_params():
    bad = []
    for k in ("dt", "wb", "max_steer", "max_accel", "max_speed", "min_speed", "w_a", "w_delta", "w_da", "w_ddelta",
              "w_x", "w_y", "w_yaw", "w_v", "du_th", "j_tol"):
        for v in (np.nan, np.inf):
            bad.append({k: v})
    bad += [dict(dt=0.0), dict(dt=-0.1), dict(wb=0.0), dict(wb=-2.5), dict(max_steer=0.0), dict(max_steer=-0.5),
            dict(max_steer=np.float32(np.pi / 2)), dict(max_steer=2.0), dict(max_accel=-1.0),
            dict(min_speed=5.0, max_speed=4.0), dict(du_th=-1e-4), dict(j_tol=-1e-6), dict(max_iter=-1),
            dict(max_ls=-1)]
    bad += [{w: -0.01} for w in ("w_a", "w_delta", "w_da", "w_ddelta", "w_x", "w_y", "w_yaw", "w_v")]
    return bad


def test_validation_needs_no_device():
    """Parameters outside crb.h's limits are refused with CRB_ERR_INVALID_ARG before any device work, by the solve
    (all three entries), the plant step and, for dt, the lookup.  The context handle is an opaque buffer these
    paths never dereference.  Valid parameters with n = 0 are a no-op that needs no device either."""
    L = _lib.load_library()
    ctx = C.create_string_buffer(256)
    d = C.c_void_p(256)        # a device address: never dereferenced on these paths
    inv = -1

    def solve(fn, prm, n=1, T=20, **kw):
        args = [ctx, n, T, d, d, None, C.byref(prm), None, None, None, None, None]
        if fn is L.crb_mpc_solve_batched_hinted:
            args.append(kw.get("hint"))
        return fn(*args)

    def plant(prm, n=1):
        return L.crb_mpc_plant_update_batched(ctx, n, d, d, C.byref(prm))

    def lookup(prm, n=1):
        return L.crb_mpc_calc_ref_trajectory_batched(ctx, n, 20, d, d, d, d, d, 100, C.c_float(1.0), d, d,
                                                     C.byref(prm))
    entries = (L.crb_mpc_solve_batched, L.crb_mpc_solve_batched_host, L.crb_mpc_solve_batched_hinted)
    for over in _invalid_params():
        prm = gparams(over)
        for fn in entries:
            assert solve(fn, prm) == inv, over
            assert solve(fn, prm, n=0) == inv, over
        assert plant(prm) == inv and plant(prm, n=0) == inv, over
        if "dt" in over:
            assert lookup(prm) == inv and lookup(prm, n=0) == inv, over
        else:
            assert lookup(prm, n=0) == _lib.CRB_OK, over      # the lookup reads only dt
    assert b"invalid argument" in L.crb_last_error_string()
    # the defaults, bench.py's settings and the test sets are inside the limits
    for over in (dict(), dict(max_iter=50, du_th=1e-4, max_ls=4), MC.W, MC.B, MC.S, MC.REVERSE,
                 dict(max_iter=0, max_ls=0, j_tol=0.0, du_th=0.0, max_accel=0.0, min_speed=4.0, max_speed=4.0)):
        prm = gparams(over)
        for fn in entries:
            assert solve(fn, prm, n=0) == _lib.CRB_OK, over
        assert plant(prm, n=0) == _lib.CRB_OK and lookup(prm, n=0) == _lib.CRB_OK, over
    # other arguments
    prm = gparams()
    assert solve(L.crb_mpc_solve_batched, prm, T=1) == inv and solve(L.crb_mpc_solve_batched, prm, T=33) == inv
    assert solve(L.crb_mpc_solve_batched, prm, n=-1) == inv
    assert L.crb_mpc_solve_batched(ctx, 1, 20, None, d, None, C.byref(prm), None, None, None, None, None) == inv
    assert L.crb_mpc_solve_batched(ctx, 1, 20, d, d, None, None, None, None, None, None, None) == inv
    assert L.crb_mpc_solve_batched(None, 1, 20, d, d, None, C.byref(prm), None, None, None, None, None) == inv
    assert plant(prm, n=-1) == inv and L.crb_mpc_plant_update_batched(ctx, 1, None, d, C.byref(prm)) == inv
    assert L.crb_mpc_plant_update_batched(ctx, 1, d, d, None) == inv
    assert L.crb_mpc_plant_update_batched(None, 1, d, d, C.byref(prm)) == inv
    assert L.crb_mpc_calc_ref_trajectory_batched(ctx, 1, 20, d, d, d, d, d, 100, C.c_float(0.0), d, d,
                                                 C.byref(prm)) == inv
    assert L.crb_mpc_calc_ref_trajectory_batched(ctx, 1, 20, d, d, d, d, d, 0, C.c_float(1.0), d, d,
                                                 C.byref(prm)) == inv
    assert L.crb_mpc_calc_ref_trajectory_batched(ctx, 1, 20, d, d, d, d, d, 100, C.c_float(1.0), d, d,
                                                 None) == inv


# ---- GPU: the solver -----------------------------------------------------------------------------------------
def _multi_wave_n():
    """>= 3 waves of problems at every horizon: one CTA per SM holds at most MPC_TASK_SLOTS = 160 slots."""
    import torch
    return 3 * torch.cuda.get_device_properties(0).multi_processor_count * 160 + 77


def _gpu_out(n, T, outputs):
    import torch
    nsol = 4 * T + 2 * (T - 1)
    shape = dict(sol=(nsol, n), u0=(2, n), cost=(n,), status=(n,), iters=(n,))
    return {k: torch.full(shape[k], SENTINEL if k in ("status", "iters") else float("nan"),
                          dtype=torch.int32 if k in ("status", "iters") else torch.float32, device="cuda")
            for k in outputs}


def solve_gpu(engine, st, xref, T, prm, outputs=OUTS, entry="device", hint=None):
    import torch
    n = st.shape[1]
    if entry == "host":
        out = {k: v.cpu().numpy() for k, v in _gpu_out(n, T, outputs).items()}
        engine.mpc_solve_host(st, xref, T, prm, **out)
        return out
    std = torch.from_numpy(st).cuda()
    xrd = torch.from_numpy(np.ascontiguousarray(xref)).cuda()
    out = _gpu_out(n, T, outputs)
    if entry == "hinted":
        engine.mpc_solve_hinted(std, xrd, T, torch.from_numpy(np.ascontiguousarray(hint, np.int32)).cuda(), prm,
                                **out)
    else:
        engine.mpc_solve(std, xrd, T, prm, **out)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def same(got, want, keys=OUTS, cols=None):
    for k in keys:
        g, w = got[k], want[k]
        if cols is not None:
            g, w = g[..., cols], w[..., cols]
        assert np.array_equal(g, w), k


@pytest.mark.gpu
@pytest.mark.parametrize("T", [2, 3, 7, 20, 32])
@pytest.mark.parametrize("name", ["W", "B", "S"])
def test_solve_bit_exact_at_constants_multi_wave(engine, name, T):
    over = MC.SETS[name]
    n = _multi_wave_n()
    st, xref = MC.case(n, T, seed=0xC0FFEE + T, dt=dt_of(over))
    want = O.mpc_solve_batched(st, xref, T, oparams(over))
    got = solve_gpu(engine, st, xref, T, gparams(over))
    same(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("T", range(2, 33))
def test_solve_bit_exact_at_every_horizon(engine, T):
    over = MC.SETS["WBS"[T % 3]]
    st, xref = MC.case(97, T, seed=T, dt=dt_of(over))
    same(solve_gpu(engine, st, xref, T, gparams(over)), O.mpc_solve_batched(st, xref, T, oparams(over)))


@pytest.mark.gpu
@pytest.mark.parametrize("over", [dict(max_iter=0), dict(max_ls=0), dict(j_tol=0.0, du_th=1e-2)],
                         ids=["max_iter0", "max_ls0", "j_tol0"])
def test_solve_bit_exact_at_loop_limits_multi_wave(engine, over):
    """max_iter = 0: every slot goes refill -> refill and the backward / forward queues stay empty."""
    T = 20
    st, xref = MC.case(_multi_wave_n(), T, seed=31)
    want = O.mpc_solve_batched(st, xref, T, oparams(over))
    got = solve_gpu(engine, st, xref, T, gparams(over))
    same(got, want)
    if over.get("max_iter") == 0:
        assert (got["iters"] == 0).all() and (got["status"] == 1).all()


@pytest.mark.gpu
def test_solve_with_nonfinite_problems_interleaved_multi_wave(engine):
    """Every fifth problem has a NaN yaw and retires at refill, between problems that run for many iterations."""
    T = 20
    over = MC.W
    st, xref = MC.case(_multi_wave_n(), T, seed=41)
    st = st.copy()
    st[2, ::5] = np.nan
    want = O.mpc_solve_batched(st, xref, T, oparams(over))
    got = solve_gpu(engine, st, xref, T, gparams(over))
    bad = np.zeros(st.shape[1], bool)
    bad[::5] = True
    assert (want["status"][bad] == 3).all() and (want["status"][~bad] != 3).all()
    same(got, want, ("status", "iters", "u0"))     # u0 of a NaN-yaw problem is its (finite) cold start
    same(got, want, ("cost", "sol"), cols=~bad)


@pytest.mark.gpu
def test_each_output_alone_equals_the_full_run(engine):
    T = 20
    over = MC.W
    st, xref = MC.case(_multi_wave_n(), T, seed=51)
    prm = gparams(over)
    full = solve_gpu(engine, st, xref, T, prm)
    same(full, O.mpc_solve_batched(st, xref, T, oparams(over)))
    for k in OUTS:
        same(solve_gpu(engine, st, xref, T, prm, outputs=(k,)), full, (k,))


@pytest.mark.gpu
def test_host_and_hinted_entries_equal_the_device_entry_at_constants(engine):
    T = 20
    over = MC.B
    st, xref = MC.case(_multi_wave_n(), T, seed=61, dt=dt_of(over))
    prm = gparams(over)
    dev = solve_gpu(engine, st, xref, T, prm)
    same(dev, O.mpc_solve_batched(st, xref, T, oparams(over)))
    same(solve_gpu(engine, st, xref, T, prm, entry="host"), dev)
    rng = np.random.default_rng(7)
    for hint in (dev["iters"], rng.integers(0, 40, st.shape[1])):
        same(solve_gpu(engine, st, xref, T, prm, entry="hinted", hint=hint), dev)


# ---- GPU: update() and calc_ref_trajectory() ---------------------------------------------------------------------
def _few(n):
    """Agents allowed to differ from the oracle by an ulp: cos / sin of a float through a glibc build without FMA
    differ from crb_sincosf_libm on 2e-8 of the inputs (crb_common.cuh)."""
    return max(1, int(4e-6 * n))


def assert_plant_bits(got, want):
    diff = (got != want).any(axis=0)
    assert diff.sum() <= _few(got.shape[1]), f"{diff.sum()} of {got.shape[1]} agents differ"
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    return int(diff.sum())


def _plant_inputs(n, over, seed):
    st, _ = synth.mpc_states(n, seed=seed)
    rng = np.random.default_rng(seed)
    u0 = np.stack([rng.uniform(-4, 4, n), rng.uniform(-1.2, 1.2, n)]).astype(np.float32)
    vmax, vmin = np.float32(over.get("max_speed", 55 / 3.6)), np.float32(over.get("min_speed", -20 / 3.6))
    st[3, :64] = vmax                      # the speed clamps, from both sides
    st[3, 64:128] = vmin
    st[3, 128:192] = -st[3, 128:192]
    ms = np.float32(over.get("max_steer", 45.0 / 180 * np.pi))
    u0[1, 192:200] = [ms, -ms, np.nextafter(ms, np.float32(0)), np.nextafter(ms, np.float32(9)), 0.0, -0.0,
                      np.pi / 2, -np.pi / 2]   # the steering clamp's edges
    return st, u0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["B", "S"])
def test_plant_update_bit_exact_at_constants(engine, name):
    import torch
    over = MC.SETS[name]
    n = 20_000
    st, u0 = _plant_inputs(n, over, seed=9)
    s = torch.from_numpy(st.copy()).cuda()
    engine.mpc_plant_update(s, torch.from_numpy(u0).cuda(), gparams(over))
    torch.cuda.synchronize()
    prm = oparams(over)
    want = np.stack([O.plant_update(st[:, i], u0[0, i], u0[1, i], params=prm) for i in range(n)], axis=1)
    assert_plant_bits(s.cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 7, 32])
@pytest.mark.parametrize("dl", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("name", ["B", "S"])
def test_calc_ref_trajectory_bit_exact_at_constants(engine, name, dl, T):
    import torch
    over = MC.SETS[name]
    course = synth.mpc_course(length=1000.0, dl=dl)
    st, pind = synth.mpc_states(1500, seed=int(dl * 10) + T, course=course)
    est, epind = MC.edge_states([v for t, v in MC.rounding_edge_speeds(dl, dt_of(over), T)])
    st = np.ascontiguousarray(np.concatenate([st, est], axis=1))
    pind = np.concatenate([pind, epind]).astype(np.int32)
    pind[:40] = len(course[0]) - 1 - np.arange(40) % 12        # the window runs off the end of the course
    st[3, 40:80] = -st[3, 40:80]                                # |v|
    n = st.shape[1]
    tid = torch.from_numpy(pind.copy()).cuda()
    xr = torch.full((4 * T, n), float("nan"), dtype=torch.float32, device="cuda")
    engine.calc_ref_trajectory(torch.from_numpy(st).cuda(), *(torch.from_numpy(c).cuda() for c in course), dl,
                               tid, xr, T, gparams(over))
    torch.cuda.synchronize()
    got_x, got_t = xr.cpu().numpy(), tid.cpu().numpy()
    prm = oparams(over)
    for i in range(n):
        wx, wt = O.calc_ref_trajectory(st[:, i], *course, dl, T, int(pind[i]), params=prm)
        assert wt == got_t[i] and np.array_equal(wx.reshape(-1), got_x[:, i]), i


@pytest.mark.gpu
def test_promotion_rule_on_the_device(engine):
    """dt = float32(0.2) is the reference's DT = 0.2 (a double); the next float up is used as its own value."""
    import torch
    n = 4096
    st, u0 = _plant_inputs(n, {}, seed=13)
    course = synth.mpc_course()
    _, pind = synth.mpc_states(n, seed=13, course=course)
    k_up = np.array([45.0 / 180 * np.pi, float(np.nextafter(np.float32(0.2), np.float32(1))), 2.5, 55 / 3.6,
                     -20 / 3.6])
    L = O._mpc_lib()
    outs = {}
    for label, dt in (("macro", np.float32(0.2)), ("up", np.nextafter(np.float32(0.2), np.float32(1)))):
        prm = gparams(dt=dt)
        s = torch.from_numpy(st.copy()).cuda()
        engine.mpc_plant_update(s, torch.from_numpy(u0).cuda(), prm)
        tid = torch.from_numpy(pind.copy()).cuda()
        xr = torch.empty((4 * 32, n), dtype=torch.float32, device="cuda")
        engine.calc_ref_trajectory(torch.from_numpy(st).cuda(), *(torch.from_numpy(c).cuda() for c in course),
                                   1.0, tid, xr, 32, prm)
        torch.cuda.synchronize()
        outs[label] = (s.cpu().numpy(), xr.cpu().numpy(), tid.cpu().numpy())
    want_macro, want_up = [], []
    for i in range(n):
        want_macro.append(O.plant_update(st[:, i], u0[0, i], u0[1, i]))
        w = np.ascontiguousarray(st[:, i]).copy()
        L.crb_oracle_plant_update_k(w, float(u0[0, i]), float(u0[1, i]), k_up)
        want_up.append(w)
    assert_plant_bits(outs["macro"][0], np.stack(want_macro, axis=1))
    assert_plant_bits(outs["up"][0], np.stack(want_up, axis=1))
    assert not np.array_equal(outs["macro"][0], outs["up"][0])     # the two steps really differ
    for label, DT in (("macro", 0.2), ("up", k_up[1])):
        xn, tn = synth.mpc_xref_numpy(st, pind, 32, course=course, dt=DT)
        assert np.array_equal(outs[label][1], xn) and np.array_equal(outs[label][2], tn), label
    for i in range(0, n, 16):
        wx, wt = O.calc_ref_trajectory(st[:, i], *course, 1.0, 32, int(pind[i]))
        assert wt == outs["macro"][2][i] and np.array_equal(wx.reshape(-1), outs["macro"][1][:, i])


@pytest.mark.gpu
def test_closed_loop_lockstep_with_the_oracle_at_constants(engine):
    """mpc_simulation's loop body (:372-376) at set B, lookup -> solve -> update on the device for 15 steps, against
    the oracle running its own loop from the same start (never re-fed with the device's state).  Every agent must
    stay bit-identical at every step; an agent that diverges is counted, reported and dropped from later steps."""
    import torch
    n, T, steps = 4096, 20, 15
    over = MC.B
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, seed=21, course=course)
    prm_g, prm_o = gparams(over), oparams(over)
    cd = [torch.from_numpy(c).cuda() for c in course]
    state = torch.from_numpy(st.copy()).cuda()
    tind = torch.from_numpy(pind.copy()).cuda()
    xref = torch.empty((4 * T, n), dtype=torch.float32, device="cuda")
    u0 = torch.empty((2, n), dtype=torch.float32, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    s_o, t_o = st.copy(), pind.astype(np.int64).copy()
    live = np.ones(n, bool)
    for k in range(steps):
        engine.calc_ref_trajectory(state, *cd, 1.0, tind, xref, T, prm_g)
        engine.mpc_solve(state, xref, T, prm_g, u0=u0, status=status)
        engine.mpc_plant_update(state, u0, prm_g)
        torch.cuda.synchronize()
        xr_o = np.empty((4 * T, n), np.float32)
        for i in range(n):
            x, t_o[i] = O.calc_ref_trajectory(s_o[:, i], *course, 1.0, T, int(t_o[i]), params=prm_o)
            xr_o[:, i] = x.reshape(-1)
        ro = O.mpc_solve_batched(s_o, xr_o, T, prm_o)
        for i in range(n):
            s_o[:, i] = O.plant_update(s_o[:, i], ro["u0"][0, i], ro["u0"][1, i], params=prm_o)
        ok = ((xref.cpu().numpy() == xr_o).all(axis=0) & (tind.cpu().numpy() == t_o)
              & (u0.cpu().numpy() == ro["u0"]).all(axis=0) & (status.cpu().numpy() == ro["status"])
              & (state.cpu().numpy() == s_o).all(axis=0))
        live &= ok
    diverged = int((~live).sum())
    print(f"closed loop at set B: {diverged} of {n} agents diverged from the oracle within {steps} steps")
    assert diverged <= 4
    assert (t_o >= pind).all() and (t_o > pind).mean() > 0.5      # the fleet drives along the course
