"""Dynamic window approach (src/dynamic_window_approach.cpp): dwa_control and motion.
CPU: the oracle's acosf, dwa_control and motion are bitwise the host libm / the reference's own text / the golden
fixture; parameters, layouts and argument validation.  H100: crb_dwa_control_batched and crb_dwa_motion_batched are
bitwise the oracle (batch sizes, obstacle counts, quirk robots, shard invariance, a 200-step closed loop)."""
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
GOLDEN = os.path.join(ROOT, "tests", "golden", "dwa_golden.npz")
CPP = os.path.join(ROOT, "tests", "cpp", "dwa_ref_api.cpp")


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def obstacle_set(k):
    return synth.DWA_DEMO_OBSTACLES if k == 10 else synth.dwa_obstacles(k)


def lib_params(p):
    return _lib.DwaParams(*[getattr(p, k) for k, _ in p._fields_])


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_acosf_restatement_is_the_host_acosf_on_every_float_in_unit_interval():
    assert OD.libm_acosf_census(0, 0x3F800001) == 0          # [-1, 1], both signs, every bit pattern
    specials = np.array([0.0, -0.0, 1.0, -1.0, 1.0000001, -1.0000001, 2.0, -3.5, 1e30, np.inf, -np.inf, np.nan],
                        np.float32)
    libm = C.CDLL("libm.so.6")
    libm.acosf.restype, libm.acosf.argtypes = C.c_float, [C.c_float]
    for v in specials:
        a = np.float32(libm.acosf(float(v)))
        b = np.float32(OD.libm_acosf(float(v)))
        assert bits_equal(a, b) or (np.isnan(a) and np.isnan(b)), (v, a, b)


def _ref_lib():
    L = reference("dwa")
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
    import golden.make_dwa_golden as G
    return L, G


@pytest.mark.parametrize("k", [0, 10, 64])
def test_oracle_is_bitwise_the_reference_text(k):
    L, G = _ref_lib()
    ob = obstacle_set(k)
    p = OD.dwa_params()
    x, u, g = D.batch(2000, ob, seed=0xD5A + k)
    qx, qu, qg = D.quirk_agents(ob, p)
    x, u, g = (np.ascontiguousarray(np.concatenate(a, axis=1)) for a in ((x, qx), (u, qu), (g, qg)))
    ru, rc, rt, rm = G.reference(L, x, u, g, ob, p)
    o = OD.dwa_control(x, u, g, ob, p)
    assert bits_equal(o["u"], ru) and bits_equal(o["cost"], rc) and bits_equal(o["traj"], rt)
    assert np.array_equal(o["best"] < 0, rc == np.float32(10000.0))
    assert bits_equal(OD.dwa_motion(x, o["u"], p.dt), rm)
    m = qx.shape[1]
    if k:   # the robot standing on obstacle 0: every sample collides
        assert o["best"][-m] == -1 and o["cost"][-m] == 10000.0 and o["u"][0, -m] == 0.0
        assert o["u"][1, -m] == u[1, -m]
        m -= 1
    assert o["best"][-m] == -1 and o["cost"][-m] == 10000.0   # goal at the origin: every cost is NaN
    assert o["best"][-m + 4] == -1 and np.isnan(o["traj"][:, -m + 4]).all()   # empty window


def test_obstacle_free_cost_is_subnormal_and_quirk_goal_is_outside_acos_domain():
    p = OD.dwa_params()
    x = np.array(D.quirk_agents(np.zeros((0, 2)), p)[0][:, 1], np.float32)
    g = D.collinear_goal(x, p)
    assert abs(float(D._error(g, D._rollout_end(x, max(np.float32(x[3] - np.float32(p.max_accel * p.dt)),
                                                            np.float32(p.min_speed)),
                                                 max(np.float32(x[4] - np.float32(p.max_dyawrate * p.dt)),
                                                     np.float32(-p.max_yawrate)), p)))) > 1.0
    # with no obstacles the obstacle cost is (float)(1 / FLT_MAX), a subnormal; with both gains 0 it is the cost
    xs, us, gs = synth.dwa_inputs(64, seed=3)
    o = OD.dwa_control(xs, us, gs, np.zeros((0, 2), np.float32), OD.dwa_params(to_goal_cost_gain=0.0,
                                                                               speed_cost_gain=0.0))
    sub = np.float32(1.0 / np.finfo(np.float32).max)
    assert 0 < sub < np.finfo(np.float32).tiny
    assert (o["best"] >= 0).sum() > 32 and (o["cost"][o["best"] >= 0] == sub).all()


def test_oracle_reproduces_the_golden_fixture():
    d = np.load(GOLDEN)
    p = OD.dwa_params()
    for name in ("none", "demo", "random64"):
        ob = d[f"{name}_ob"]
        o = OD.dwa_control(d[f"{name}_x"], d[f"{name}_u_in"], d[f"{name}_goal"], ob, p)
        assert bits_equal(o["u"], d[f"{name}_u"]) and bits_equal(o["cost"], d[f"{name}_cost"]), name
        assert bits_equal(o["traj"], d[f"{name}_traj"]), name
        assert bits_equal(OD.dwa_motion(d[f"{name}_x"], o["u"], p.dt), d[f"{name}_motion"]), name


def test_defaults_are_the_reference_config_and_layout_matches(tmp_path):
    from cpprobotics_b200 import dwa_default_params
    lp, op = dwa_default_params(), OD.dwa_params()
    for k, _ in _lib.DwaParams._fields_:
        assert np.float32(getattr(lp, k)) == np.float32(getattr(op, k)), k
    assert np.float32(lp.max_yawrate) == np.float32(40.0 * 3.141592653 / 180.0) == np.float32(0.6981317)
    L = reference("dwa")
    if L is not None:
        cfg = np.zeros(12, np.float32)
        L.ref_dwa_default_config(cfg.ctypes.data_as(C.c_void_p))
        assert bits_equal(cfg, np.array([getattr(lp, k) for k, _ in _lib.DwaParams._fields_], np.float32))
    n = C.c_int(0)
    assert _lib.load_library().crb_dwa_rollout_points(C.byref(lp), C.byref(n)) == 0 and n.value == 32
    assert OD.dwa_rollout_points(op) == 32
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){printf("%zu %zu %zu '
                   '%d %d %d %d\\n",sizeof(crb_dwa_params),offsetof(crb_dwa_params,v_reso),'
                   'offsetof(crb_dwa_params,speed_cost_gain),CRB_DWA_MAX_OBSTACLES,CRB_DWA_MAX_SPEED_SAMPLES,'
                   'CRB_DWA_MAX_YAWRATE_SAMPLES,CRB_DWA_MAX_STEPS);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.DwaParams), _lib.DwaParams.v_reso.offset, _lib.DwaParams.speed_cost_gain.offset,
                   _lib.CRB_DWA_MAX_OBSTACLES, _lib.CRB_DWA_MAX_SPEED_SAMPLES, _lib.CRB_DWA_MAX_YAWRATE_SAMPLES,
                   _lib.CRB_DWA_MAX_STEPS]


def _invalid_params():
    cases = []
    for field, value in [("v_reso", 0.0), ("v_reso", -0.01), ("v_reso", np.nan), ("yawrate_reso", 0.0),
                         ("yawrate_reso", np.inf), ("dt", 0.0), ("dt", -0.1), ("dt", np.inf), ("dt", np.nan),
                         ("robot_radius", np.nan), ("max_speed", np.inf), ("predict_time", np.inf),
                         ("predict_time", 1.0e6), ("v_reso", 1.0e-5), ("yawrate_reso", 1.0e-6)]:
        p = OD.dwa_params()
        setattr(p, field, float(value))
        cases.append(lib_params(p))
    return cases


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE on a machine without
    a GPU.  The context handle is an opaque non-NULL buffer that these paths never dereference."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)           # a device address: never dereferenced on these paths
    good = lib_params(OD.dwa_params())
    ok_args = dict(ctx=ctx, n=1, x=d, u=d, goal=d, ob=d, n_ob=10, prm=C.byref(good))

    def ctl(**over):
        a = dict(ok_args, **over)
        return L.crb_dwa_control_batched(a["ctx"], a["n"], a["x"], a["u"], a["goal"], a["ob"], a["n_ob"], a["prm"],
                                         None, None, None)
    inv = -1
    for k in ("ctx", "x", "u", "goal", "prm"):
        assert ctl(**{k: None}) == inv, k
    assert ctl(n=-1) == inv and ctl(n_ob=-1) == inv and ctl(n_ob=_lib.CRB_DWA_MAX_OBSTACLES + 1) == inv
    assert ctl(ob=None) == inv
    for p in _invalid_params():
        assert ctl(prm=C.byref(p)) == inv
        k = C.c_int(0)
        assert L.crb_dwa_rollout_points(C.byref(p), C.byref(k)) == inv
    assert L.crb_dwa_rollout_points(None, C.byref(C.c_int())) == inv
    assert L.crb_dwa_rollout_points(C.byref(good), None) == inv
    assert L.crb_dwa_motion_batched(None, 1, d, d, C.c_float(0.1)) == inv
    assert L.crb_dwa_motion_batched(ctx, 1, None, d, C.c_float(0.1)) == inv
    assert L.crb_dwa_motion_batched(ctx, 1, d, None, C.c_float(0.1)) == inv
    assert L.crb_dwa_motion_batched(ctx, -1, d, d, C.c_float(0.1)) == inv
    for dt in (0.0, -0.1, np.inf, np.nan):
        assert L.crb_dwa_motion_batched(ctx, 1, d, d, C.c_float(dt)) == inv
    if not torch.cuda.is_available():
        assert ctl() == _lib.CRB_ERR_NO_DEVICE
        assert ctl(n=0, x=None, u=None, goal=None, ob=None, n_ob=0) == _lib.CRB_ERR_NO_DEVICE
        assert b"no CPU fallback" in L.crb_last_error_string()
        assert L.crb_dwa_motion_batched(ctx, 1, d, d, C.c_float(0.1)) == _lib.CRB_ERR_NO_DEVICE


def _build_cpp(tmp_path):
    exe = str(tmp_path / "dwa_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), CPP,
                           "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


def test_reference_style_program_compiles(tmp_path):
    _build_cpp(tmp_path)


# ---- H100 -----------------------------------------------------------------------------------------------------
def _gpu(engine, x, u, g, ob, p=None, outputs=True):
    import torch
    dev = torch.device("cuda:0")
    p = p or OD.dwa_params()
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


def _same(r, o):
    return (bits_equal(r["u"], o["u"]) and bits_equal(r["cost"], o["cost"]) and np.array_equal(r["best"], o["best"])
            and bits_equal(r["traj"], o["traj"]))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
@pytest.mark.parametrize("k", [0, 10, 64, _lib.CRB_DWA_MAX_OBSTACLES])
def test_gpu_is_bitwise_the_oracle(engine, n, k):
    ob = obstacle_set(k)
    x, u, g = D.batch(n, ob, seed=0xD00 + n)
    if n == 1:
        x, u, g = (np.ascontiguousarray(a[:, -1:]) for a in D.quirk_agents(ob))  # the obstacle-free corner robot
    o = OD.dwa_control(x, u, g, ob)
    r = _gpu(engine, x, u, g, ob)
    assert _same(r, o)
    if n == 4097:
        assert (o["best"] < 0).any() and (o["best"] >= 0).any()
        assert bits_equal(_gpu(engine, x, u, g, ob, outputs=False)["u"], o["u"])   # NULL outputs: same u


@pytest.mark.gpu
def test_gpu_n_zero_is_a_no_op(engine):
    import torch
    e = torch.empty((5, 0), dtype=torch.float32, device="cuda:0")
    engine.dwa_control(e, e[:2], e[:2], torch.empty((0, 2), dtype=torch.float32, device="cuda:0"))
    engine.dwa_motion(e, e[:2])
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_reproduces_the_golden_fixture(engine):
    d = np.load(GOLDEN)
    import torch
    for name in ("none", "demo", "random64"):
        r = _gpu(engine, d[f"{name}_x"], d[f"{name}_u_in"], d[f"{name}_goal"], d[f"{name}_ob"])
        assert bits_equal(r["u"], d[f"{name}_u"]) and bits_equal(r["cost"], d[f"{name}_cost"]), name
        assert bits_equal(r["traj"], d[f"{name}_traj"]), name
        xd = torch.from_numpy(d[f"{name}_x"]).cuda()
        engine.dwa_motion(xd, torch.from_numpy(r["u"]).cuda())
        torch.cuda.synchronize()
        assert bits_equal(xd.cpu().numpy(), d[f"{name}_motion"]), name


@pytest.mark.gpu
def test_gpu_shard_invariance(engine):
    ob = synth.DWA_DEMO_OBSTACLES
    x, u, g = D.batch(10000, ob, seed=77)
    full = _gpu(engine, x, u, g, ob)
    i0, i1 = 3001, 7203
    part = _gpu(engine, *(np.ascontiguousarray(a[:, i0:i1]) for a in (x, u, g)), ob)
    for k in ("u", "traj"):
        assert bits_equal(part[k], np.ascontiguousarray(full[k][:, i0:i1])), k
    for k in ("cost", "best"):
        assert np.array_equal(part[k].view(np.uint32), full[k][i0:i1].view(np.uint32)), k
    xs, us, gs = synth.dwa_inputs(i1 - i0, seed=77, i0=i0)
    xf, uf, gf = synth.dwa_inputs(10000, seed=77)
    assert bits_equal(xs, np.ascontiguousarray(xf[:, i0:i1])) and bits_equal(gs, np.ascontiguousarray(gf[:, i0:i1]))


@pytest.mark.gpu
def test_gpu_closed_loop_200_steps(engine):
    import torch
    ob = synth.DWA_DEMO_OBSTACLES
    n = 4096
    x, u, g = synth.dwa_inputs(n, seed=2024)
    x[:, 0], g[:, 0] = synth.DWA_DEMO_START, synth.DWA_DEMO_GOAL
    dev = torch.device("cuda:0")
    xd, ud, gd, obd = (torch.from_numpy(a).to(dev) for a in (x, u, g, ob))
    xo, uo = x.copy(), u.copy()
    for step in range(200):
        engine.dwa_control(xd, ud, gd, obd)
        engine.dwa_motion(xd, ud)
        o = OD.dwa_control(xo, uo, g, ob, traj=False)
        uo = o["u"]
        xo = OD.dwa_motion(xo, uo)
        assert np.abs(xo[2]).max() < 100.0
        if step % 20 == 19 or step == 199:
            torch.cuda.synchronize()
            assert bits_equal(ud.cpu().numpy(), uo) and bits_equal(xd.cpu().numpy(), xo), step
    moved = np.hypot(xo[0] - x[0], xo[1] - x[1])
    assert np.median(moved) > 1.0


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_oracle(tmp_path):
    exe = _build_cpp(tmp_path)
    d = np.load(GOLDEN)
    x, u, g, ob = d["demo_x"], d["demo_u_in"], d["demo_goal"], d["demo_ob"]
    m = x.shape[1]
    blob = np.concatenate([np.float32([m, len(ob)]), np.concatenate([x, u, g], axis=0).T.reshape(-1),
                           ob.reshape(-1)]).astype(np.float32)
    blob.tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    p = 0
    nxt = OD.dwa_motion(x, d["demo_u"])
    for i in range(m):
        assert bits_equal(out[p:p + 2], d["demo_u"][:, i]); p += 2
        k = int(out[p]); p += 1
        if np.isnan(d["demo_traj"][0, i]):
            assert k == 0
        else:
            assert bits_equal(out[p:p + 5 * k], d["demo_traj"][:, i]); p += 5 * k
        assert bits_equal(out[p:p + 5], nxt[:, i]); p += 5
    assert p == out.size
