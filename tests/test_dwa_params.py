"""Dynamic window approach away from the reference's default Config (tests/dwa_cases.py CONFIGS), and the rule that
keeps every accepted Config's sample grid within CRB_DWA_MAX_SPEED_SAMPLES x CRB_DWA_MAX_YAWRATE_SAMPLES.
CPU: the checker is bitwise the reference's own text at every configuration; the sample-count rule is sound for a
deterministic sweep of magnitudes and resolutions; the rollout length at 999, 1000 and 1001 steps.  H100: the kernel
is bitwise the checker (and the reference text where oracle/_ref exists) at every configuration, in a closed loop, in
the reference-style C++ program with a non-default Config, and with `traj` offsets past 2^31 elements."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dwa_cases as D
from cpprobotics_b200 import _lib, synth
from oracle import dwa as OD
from oracle._load import reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp", "dwa_ref_api.cpp")
VCAP, WCAP = _lib.CRB_DWA_MAX_SPEED_SAMPLES, _lib.CRB_DWA_MAX_YAWRATE_SAMPLES
f32 = np.float32
NAMES = list(D.CONFIGS)
# parameter sets the rule used to accept although the reference's float loop takes more samples than the cap (the
# first two) or never ends (the third: fl(v + v_reso) == v)
BEYOND_CAP = {
    "speed": dict(max_speed=1e5, min_speed=99999.4, max_accel=10.0, dt=0.1, v_reso=0.01, predict_time=0.3,
                  to_goal_cost_gain=0.0),
    "yaw": dict(max_yawrate=1e4, max_dyawrate=10.0, dt=0.02525, yawrate_reso=0.001),
    "stall": dict(max_speed=1e6, min_speed=1e6 - 0.6, max_accel=3.0, v_reso=0.01),
}


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def obstacle_set(k):
    return synth.DWA_DEMO_OBSTACLES if k == 10 else synth.dwa_obstacles(k)


def lib_params(p):
    return _lib.DwaParams(*[getattr(p, k) for k, _ in p._fields_])


def rollout_points(p):
    """crb_dwa_rollout_points: the point count, or None when the parameters are refused."""
    n = C.c_int(0)
    rc = _lib.load_library().crb_dwa_rollout_points(C.byref(lib_params(p)), C.byref(n))
    return n.value if rc == 0 else None


def axis_counts(s, half, lo, hi, reso, cap):
    """Samples the reference's loop takes on one axis (:52-60, :126-127) for states s (float32 arrays, broadcast):
    the window [max(s - half, lo), min(s + half, hi)] walked by float32 `v += reso`.  Counts stop at cap + 1."""
    s, half, lo, hi, reso = (np.asarray(a, f32) for a in (s, half, lo, hi, reso))
    a, b = s - half, s + half
    v = np.where(a < lo, lo, a)
    top = np.where(hi < b, hi, b)
    v, top, reso = np.broadcast_arrays(v, top, reso)
    v = v.copy()
    n = np.zeros(v.shape, np.int64)
    act = v <= top
    for _ in range(cap + 1):
        if not act.any():
            break
        n += act
        v = np.where(act, v + reso, v)
        act &= v <= top
    return n


def grid_counts(x, p):
    """(nv, nw) per robot of x [5, n] under the configuration p."""
    nv = axis_counts(x[3], f32(p.max_accel) * f32(p.dt), p.min_speed, p.max_speed, p.v_reso, VCAP)
    nw = axis_counts(x[4], f32(p.max_dyawrate) * f32(p.dt), -f32(p.max_yawrate), p.max_yawrate, p.yawrate_reso, WCAP)
    return nv, nw


def robots(name, n, ob, seed):
    """n robots for the configuration: seeded ones with the quirk robots at the end (all quirks when n < 9)."""
    p = D.config(name)
    qx, qu, qg = D.quirk_agents(ob, p)
    m = qx.shape[1]
    if n <= m:
        return tuple(np.ascontiguousarray(a[:, -n:]) for a in (qx, qu, qg))
    x, u, g = D.config_batch(name, n - m, ob, seed=seed)
    return tuple(np.ascontiguousarray(np.concatenate(a, axis=1)) for a in ((x, qx), (u, qu), (g, qg)))


def _ref_lib():
    L = reference("dwa")
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
    import golden.make_dwa_golden as G
    return L, G


def check_outcome(name, x, u, o, p):
    """What each configuration is there to reach, on the checker's (or the kernel's) result."""
    best = o["best"]
    if name in ("speed_gain_above_min_cost", "empty_speed_window", "empty_yaw_window"):
        assert (best == -1).all() and (o["cost"] == f32(10000.0)).all()
        assert (o["u"][0] == 0.0).all() and bits_equal(o["u"][1], u[1]) and np.isnan(o["traj"]).all()
    nv, nw = grid_counts(x, p)
    assert (nv <= VCAP).all() and (nw <= WCAP).all()
    assert (best < nv * nw).all()
    if name == "zero_steps":   # every sample ties: the last one in v-major order wins, or none is admissible
        ok = best >= 0
        assert ok.sum() > x.shape[1] // 2 and (best[ok] == (nv * nw)[ok] - 1).all()
        assert bits_equal(o["traj"][:, ok], x[:, ok])
    if name in ("speed_cap", "both_caps_2_steps", "both_caps_1_step"):
        assert nv.max() >= VCAP - 3
    if name in ("yaw_cap", "both_caps_2_steps", "both_caps_1_step"):
        assert nw.max() >= WCAP - 3
    if name == "gains_overflow":
        assert np.isinf(o["cost"]).any()
    if name == "yaw_past_120":
        tr = o["traj"][:, best >= 0].reshape(-1, 5, int((best >= 0).sum()))
        assert (np.abs(tr[-1, 2]) > 120.0).any() and (np.abs(tr[0, 2]) >= 2.0 ** 20).any()


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_configurations_are_accepted_and_reach_their_edges():
    for name in NAMES:
        p = D.config(name)
        assert rollout_points(p) == OD.dwa_rollout_points(p), name
    vals = [getattr(D.config("distinct"), k) for k, _ in OD.DwaParams._fields_]
    assert len(set(vals)) == 12
    assert [rollout_points(D.config(k)) for k in ("zero_steps", "one_step", "steps_999", "steps_1000")] == \
        [1, 2, 1000, 1001]
    # the cap configurations use the smallest resolution the rule accepts for their windows
    for name, field in (("speed_cap", "v_reso"), ("yaw_cap", "yawrate_reso"), ("both_caps_2_steps", "v_reso"),
                        ("both_caps_2_steps", "yawrate_reso")):
        p = D.config(name)
        setattr(p, field, float(np.nextafter(f32(getattr(p, field)), f32(0))))
        assert rollout_points(p) is None, (name, field)
    p = D.config("speed_cap_large")
    p.min_speed -= 1.0
    assert rollout_points(p) is None
    p = D.config("yaw_cap_large")
    p.max_dyawrate = float(np.nextafter(f32(p.max_dyawrate), f32(np.inf)))
    assert rollout_points(p) is None
    # limits of magnitude 0 (a single sample at 0) and subnormal resolutions on them
    assert rollout_points(OD.dwa_params(max_speed=0.0, min_speed=0.0, max_yawrate=0.0)) == 32
    assert rollout_points(OD.dwa_params(max_speed=0.0, min_speed=0.0, v_reso=1e-45, max_yawrate=0.0,
                                        yawrate_reso=1e-45)) == 32


@pytest.mark.parametrize("k", [0, 10, 256])
@pytest.mark.parametrize("name", NAMES)
def test_checker_is_bitwise_the_reference_text(name, k):
    L, G = _ref_lib()
    ob = obstacle_set(k)
    p = D.config(name)
    x, u, g = robots(name, 24 if D.heavy(name) else 96, ob, seed=0xD5A + k)
    ru, rc, rt, rm = G.reference(L, x, u, g, ob, p)
    o = OD.dwa_control(x, u, g, ob, p)
    assert bits_equal(o["u"], ru) and bits_equal(o["cost"], rc) and bits_equal(o["traj"], rt)
    assert np.array_equal(o["best"] < 0, rc == f32(10000.0))
    assert bits_equal(OD.dwa_motion(x, o["u"], p.dt), rm)
    check_outcome(name, x, u, o, p)


def three_four_five():
    """Robots 3-4-5 away from an integer obstacle (r == 5 exactly: collides), and just outside (r > 5)."""
    ob = np.float32([[3.0, 4.0], [-7.0, 11.0]])
    rows = [(0.0, 0.0), (-10.0, 7.0), (6.0, 8.0), (0.0, -0.001), (-10.001, 7.0)]
    x = np.zeros((5, len(rows)), np.float32)
    x[:2] = np.float32(rows).T
    x[2], x[3] = 0.3, 0.2
    u = np.ascontiguousarray(x[3:5])
    g = np.full((2, len(rows)), 20.0, np.float32)
    return x, u, g, ob


def test_obstacle_exactly_at_robot_radius_collides():
    L, G = _ref_lib()
    p = D.config("radius_five")
    x, u, g, ob = three_four_five()
    o = OD.dwa_control(x, u, g, ob, p)
    ru, rc, rt, _ = G.reference(L, x, u, g, ob, p)
    assert bits_equal(o["u"], ru) and bits_equal(o["cost"], rc) and bits_equal(o["traj"], rt)
    assert list(o["best"] >= 0) == [False, False, False, True, True]


def test_sample_count_rule_is_sound():
    """For magnitudes M from 1e-3 to 1e7, resolutions from 0.5 to 10^4 ulps of M and windows within one sample of
    the former rule's cap, every parameter set the library accepts keeps the reference's float32 sample loop within
    the cap, for states that put the window at the lower end of the limits, the upper end and 64 places between."""
    mags = np.float32(np.logspace(-3, 7, 41))
    ulps = np.array([0.5, 0.51, 0.6, 0.75, 1.0, 1.25, 1.5, 2.0, 2.5, 3.0, 4.5, 7.0, 10.0, 33.0, 100.0, 1e3, 1e4])
    deltas = (-1.0, -0.5, 0.0, 0.5, 1.0)
    pos = np.linspace(0.0, 1.0, 66)
    sets = []   # (axis, params, state low, state high)
    for m in mags:
        ulp = float(np.spacing(m))
        for r in ulps:
            reso = f32(r * ulp)
            for dl in deltas:
                for axis, cap in (("v", VCAP), ("w", WCAP)):
                    width = float(f32((cap - 2 + dl) * float(reso)))
                    if axis == "v":
                        fam = [dict(max_speed=m, min_speed=float(f32(m - width)), max_accel=float(m) * 4.0, dt=1.0),
                               dict(max_speed=float(f32(-m + width)), min_speed=-m, max_accel=float(m) * 4.0, dt=1.0),
                               dict(max_speed=m, min_speed=-m, max_accel=width / 2.0, dt=1.0)]
                        sets += [("v", dict(f, v_reso=float(reso), max_dyawrate=0.0)) for f in fam]
                    else:
                        sets += [("w", dict(max_yawrate=m, max_dyawrate=width / 2.0, dt=1.0, yawrate_reso=float(reso),
                                            max_accel=0.0)),
                                 ("w", dict(max_yawrate=float(f32(width / 2.0)), max_dyawrate=float(m) * 4.0, dt=1.0,
                                            yawrate_reso=float(reso), max_accel=0.0))]
    acc = {"v": [], "w": []}
    old_unsound = 0
    for axis, kw in sets:
        p = OD.dwa_params(**kw)
        if axis == "v":
            lo, hi, half, reso, cap = p.min_speed, p.max_speed, f32(p.max_accel) * f32(p.dt), p.v_reso, VCAP
            old = min(2.0 * p.max_accel * p.dt, p.max_speed - p.min_speed) / p.v_reso + 2.0 <= cap
        else:
            lo, hi, half, reso, cap = -p.max_yawrate, p.max_yawrate, f32(p.max_dyawrate) * f32(p.dt), p.yawrate_reso, WCAP
            old = min(2.0 * p.max_dyawrate * p.dt, 2.0 * p.max_yawrate) / p.yawrate_reso + 2.0 <= cap
        if rollout_points(p) is not None:
            acc[axis].append((lo, hi, half, reso))
        elif old:
            old_unsound += 1
    worst = {}
    for axis, cap in (("v", VCAP), ("w", WCAP)):
        lo, hi, half, reso = (np.float32(c)[:, None] for c in zip(*acc[axis]))
        s = np.float32(lo + half + (hi - half - (lo + half)) * pos[None, :].astype(np.float32))
        s[:, 0], s[:, -1] = (lo + half)[:, 0], (hi - half)[:, 0]
        n = axis_counts(s, half, lo, hi, reso, cap)
        worst[axis] = int(n.max())
        assert worst[axis] <= cap, (axis, worst[axis], np.argwhere(n > cap)[:3])
        assert len(acc[axis]) > 500
    # the sweep reaches near the caps, and it contains sets the former rule accepted that are refused now
    assert worst["v"] >= VCAP - 3 and worst["w"] >= WCAP - 3
    assert old_unsound > 100


def test_parameters_whose_grid_would_pass_its_cap_are_refused():
    """The reference's float loop takes 78 speed samples, 519 yaw-rate samples, or stalls (fl(v + 0.01) == v)."""
    for key, kw in BEYOND_CAP.items():
        assert rollout_points(OD.dwa_params(**kw)) is None, key
    p = OD.dwa_params(**BEYOND_CAP["speed"])
    assert axis_counts(f32(99999.7), f32(p.max_accel) * f32(p.dt), p.min_speed, p.max_speed, p.v_reso, 100) == 78
    p = OD.dwa_params(**BEYOND_CAP["yaw"])
    assert axis_counts(f32(1e4 - 0.2525), f32(p.max_dyawrate) * f32(p.dt), -f32(p.max_yawrate), p.max_yawrate,
                       p.yawrate_reso, 600) == 519
    p = OD.dwa_params(**BEYOND_CAP["stall"])
    v = f32(p.min_speed)
    assert v + f32(p.v_reso) == v


def test_rollout_points_are_the_reference_length_up_to_1000_steps():
    L, G = _ref_lib()
    for name in ("steps_999", "steps_1000"):
        p = D.config(name)
        x, u, g = robots(name, 1, np.zeros((0, 2), np.float32), 1)
        cfg = np.array([getattr(p, k) for k, _ in p._fields_], np.float32)
        t = np.zeros(5 * 1002, np.float32)
        k, c = C.c_int(0), C.c_float(0.0)
        uu = u[:, 0].copy()
        L.ref_dwa_control(*(np.ascontiguousarray(a).ctypes.data_as(C.c_void_p) for a in (x[:, 0], uu, g[:, 0])),
                          None, 0, cfg.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), C.byref(k), C.byref(c))
        assert k.value == rollout_points(p)
    assert rollout_points(OD.dwa_params(dt=0.0625, predict_time=62.5)) is None   # 1001 steps


# ---- H100 -----------------------------------------------------------------------------------------------------
def _gpu(engine, x, u, g, ob, p, outputs=True):
    import torch
    dev = torch.device("cuda:0")
    n = x.shape[1]
    xd, ud, gd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (x, u, g))
    obd = torch.from_numpy(np.ascontiguousarray(ob, np.float32).reshape(-1, 2)).to(dev)
    cost = best = traj = None
    if outputs:
        cost = torch.empty(n, dtype=torch.float32, device=dev)
        best = torch.empty(n, dtype=torch.int32, device=dev)
        traj = torch.empty((5 * OD.dwa_rollout_points(p), n), dtype=torch.float32, device=dev)
    engine.dwa_control(xd, ud, gd, obd, lib_params(p), cost=cost, best=best, traj=traj)
    torch.cuda.synchronize()
    r = dict(u=ud.cpu().numpy())
    if outputs:
        r.update(cost=cost.cpu().numpy(), best=best.cpu().numpy(), traj=traj.cpu().numpy())
    return r


def _same(r, o, cols=slice(None)):
    return (bits_equal(r["u"][:, cols], o["u"][:, cols]) and bits_equal(r["cost"][cols], o["cost"][cols])
            and np.array_equal(r["best"][cols], o["best"][cols]) and bits_equal(r["traj"][:, cols], o["traj"][:, cols]))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097])
@pytest.mark.parametrize("name", NAMES)
def test_gpu_is_bitwise_the_checker_and_the_reference(engine, name, n):
    if D.heavy(name) and n == 4097:
        n = 257
    k = {1: 0, 33: 10}.get(n, 256)
    ob = obstacle_set(k)
    p = D.config(name)
    x, u, g = robots(name, n, ob, seed=0xE00 + n)
    o = OD.dwa_control(x, u, g, ob, p)
    r = _gpu(engine, x, u, g, ob, p)
    assert _same(r, o)
    assert bits_equal(_gpu(engine, x, u, g, ob, p, outputs=False)["u"], o["u"])   # NULL outputs: the same u
    if n > 1:
        check_outcome(name, x, u, r, p)
    L = reference("dwa")
    if L is not None:
        import golden.make_dwa_golden as G
        cols = np.unique(np.r_[np.arange(0, n, max(1, n // 48)), np.arange(max(0, n - 8), n)])
        ru, rc, rt, _ = G.reference(L, *(np.ascontiguousarray(a[:, cols]) for a in (x, u, g)), ob, p)
        assert bits_equal(r["u"][:, cols], ru) and bits_equal(r["cost"][cols], rc)
        assert bits_equal(r["traj"][:, cols], rt)


@pytest.mark.gpu
def test_gpu_obstacle_exactly_at_robot_radius_collides(engine):
    p = D.config("radius_five")
    x, u, g, ob = three_four_five()
    o = OD.dwa_control(x, u, g, ob, p)
    assert _same(_gpu(engine, x, u, g, ob, p), o)
    assert list(o["best"] >= 0) == [False, False, False, True, True]


@pytest.mark.gpu
def test_gpu_refuses_traj_sized_for_another_rollout(engine):
    import torch
    p = D.config("distinct")
    assert OD.dwa_rollout_points(p) != OD.dwa_rollout_points()
    x, u, g = (torch.from_numpy(a).cuda() for a in D.config_batch("distinct", 8, synth.DWA_DEMO_OBSTACLES))
    ob = torch.from_numpy(synth.DWA_DEMO_OBSTACLES).cuda()
    u0 = u.clone()
    traj = torch.empty((5 * OD.dwa_rollout_points(), 8), dtype=torch.float32, device="cuda:0")
    with pytest.raises(ValueError):
        engine.dwa_control(x, u, g, ob, lib_params(p), traj=traj)
    torch.cuda.synchronize()
    assert torch.equal(u, u0)


@pytest.mark.gpu
def test_gpu_closed_loop_100_steps_at_a_non_default_config(engine):
    import torch
    p = D.config("distinct")
    ob = synth.DWA_DEMO_OBSTACLES
    n = 4096
    x, u, g = D.config_batch("distinct", n, ob, seed=2025)
    dev = torch.device("cuda:0")
    xd, ud, gd, obd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (x, u, g, ob))
    xo, uo = x.copy(), u.copy()
    for step in range(100):
        engine.dwa_control(xd, ud, gd, obd, lib_params(p))
        engine.dwa_motion(xd, ud, dt=p.dt)
        uo = OD.dwa_control(xo, uo, g, ob, p, traj=False)["u"]
        xo = OD.dwa_motion(xo, uo, p.dt)
        if step % 20 == 19:
            torch.cuda.synchronize()
            assert bits_equal(ud.cpu().numpy(), uo) and bits_equal(xd.cpu().numpy(), xo), step
    assert np.median(np.hypot(xo[0] - x[0], xo[1] - x[1])) > 1.0


@pytest.mark.gpu
def test_gpu_traj_offsets_past_2_31_elements(engine):
    """2^19 + 3 robots, 1000 rollout steps, a one-sample window and no obstacles: traj is 5005 x (2^19 + 3) floats
    (10.5 GB), and its element offsets pass 2^31 from row 4096 (step 819).  Each robot's result depends on its own
    column only, so the checker runs on the columns that are compared."""
    import torch
    if torch.cuda.mem_get_info()[0] < 12 * 2 ** 30:
        pytest.skip("needs 12 GiB of free device memory")
    p = OD.dwa_params(max_accel=0.0, max_dyawrate=0.0, dt=0.0625, predict_time=62.4375)
    n_pts = OD.dwa_rollout_points(p)
    assert n_pts == 1001 and rollout_points(p) == n_pts
    n = 2 ** 19 + 3
    x, u, g = synth.dwa_inputs(n, seed=31, max_speed=p.max_speed, min_speed=p.min_speed, max_yawrate=p.max_yawrate)
    ob = np.zeros((0, 2), np.float32)
    dev = torch.device("cuda:0")
    xd, ud, gd = (torch.from_numpy(a).to(dev) for a in (x, u, g))
    cost = torch.empty(n, dtype=torch.float32, device=dev)
    best = torch.empty(n, dtype=torch.int32, device=dev)
    traj = torch.empty((5 * n_pts, n), dtype=torch.float32, device=dev)
    try:
        engine.dwa_control(xd, ud, gd, torch.from_numpy(ob).to(dev), lib_params(p), cost=cost, best=best, traj=traj)
        row0 = (2 ** 31) // n                        # the row whose offsets cross 2^31
        assert row0 * n < 2 ** 31 < (row0 + 1) * n
        rows = np.r_[0, 1, row0 - 2:row0 + 3, 5 * n_pts - 5:5 * n_pts]
        c0 = 2 ** 31 - row0 * n                      # the first column past 2^31 in row row0
        cols = np.unique(np.r_[0:1000, c0 - 1000:c0 + 1000, n - 1000:n])
        got = traj.index_select(0, torch.from_numpy(rows).to(dev)).index_select(1, torch.from_numpy(cols).to(dev))
        got = got.cpu().numpy()
        r = dict(u=ud.cpu().numpy(), cost=cost.cpu().numpy(), best=best.cpu().numpy())
    finally:
        del traj
        torch.cuda.empty_cache()
    o = OD.dwa_control(x, u, g, ob, p, traj=False)
    assert bits_equal(r["u"], o["u"]) and bits_equal(r["cost"], o["cost"]) and np.array_equal(r["best"], o["best"])
    assert (o["best"] == 0).mean() > 0.9
    oc = OD.dwa_control(*(np.ascontiguousarray(a[:, cols]) for a in (x, u, g)), ob, p)
    assert bits_equal(got, np.ascontiguousarray(oc["traj"][rows]))


def _build_cpp(tmp_path):
    exe = str(tmp_path / "dwa_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), CPP,
                           "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


@pytest.mark.gpu
def test_gpu_reference_style_program_with_a_non_default_config(tmp_path):
    """dwa_ref_api's third argument sets its Config member by member, so crb::dwa_params_of maps each member by name;
    every member of this configuration differs from every other."""
    exe = _build_cpp(tmp_path)
    p = D.config("distinct")
    ob = synth.DWA_DEMO_OBSTACLES
    x, u, g = robots("distinct", 40, ob, seed=12)
    m = x.shape[1]
    blob = np.concatenate([np.float32([m, len(ob)]), np.concatenate([x, u, g], axis=0).T.reshape(-1),
                           ob.reshape(-1)]).astype(np.float32)
    blob.tofile(tmp_path / "in.bin")
    np.array([getattr(p, k) for k, _ in p._fields_], np.float32).tofile(tmp_path / "config.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(tmp_path / "config.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    o = OD.dwa_control(x, u, g, ob, p)
    nxt = OD.dwa_motion(x, o["u"], p.dt)
    n_pts = OD.dwa_rollout_points(p)
    q = 0
    for i in range(m):
        assert bits_equal(out[q:q + 2], o["u"][:, i]); q += 2
        k = int(out[q]); q += 1
        assert k == (n_pts if o["best"][i] >= 0 else 0)
        assert bits_equal(out[q:q + 5 * k], o["traj"][:5 * k, i]); q += 5 * k
        assert bits_equal(out[q:q + 5], nxt[:, i]); q += 5
    assert q == out.size
