"""Path tracking with a course per vehicle: crb_lqr_steering_control_many_batched (both LQR programs) and
crb_mpc_calc_ref_trajectory_many_batched.

Each vehicle's outputs must be bitwise those of the single-course entry point run on its own course, and so those of the
checker composed course by course (oracle/crb_oracle_lqrt.c, oracle/crb_oracle_mpc.c).
CPU: argument validation without a device, synth.pack_courses / fleet_courses, the compiler report and the C++ program.
H100 (-m gpu): the equivalence at n = 1, 33, 4097 and 65536 on 1-point, demo, 50 000-point and random courses with
vehicles in random order; NULL outputs, n = 0 and graph capture; bad course references; ind persisting per course,
BAD_INDEX and target_ind outside the course; a 300-tick closed loop against the checker."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from cpprobotics_b200 import _lib, lqr_track_default_params, synth
from oracle import lqrt as OL
from oracle import oracle as O
from test_lqr_track import ALL, _bits_equal, assert_same, nondefault_params
from toolchain import build_ref_program, ptxas_kernels

INV = -1
KP, STOP_SPEED = 1.0, 0.05


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is refused with CRB_ERR_INVALID_ARG before any device work."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)

    def lqr(nx=4, po=None, **over):
        p = lqr_track_default_params(nx)
        for k, v in (po or {}).items():
            if k in ("Q", "R"):
                getattr(p, k)[v[0]] = v[1]
            else:
                setattr(p, k, v)
        a = dict(dict(ctx=ctx, n=5, st=d, cx=d, ck=d, sp=d if nx == 5 else None, off=d, nc=3, npts=100, of=d,
                      prm=C.byref(p), ind=d, u=d), **over)
        return L.crb_lqr_steering_control_many_batched(a["ctx"], a["n"], nx, a["st"], a["cx"], d, d, a["ck"], a["sp"],
                                                       a["off"], a["nc"], a["npts"], a["of"], a["prm"], a["ind"], d, d,
                                                       a["u"], None, None, None)

    nan, inf = float("nan"), float("inf")
    for nx in (4, 5):
        for po in (dict(dt=nan), dict(wheelbase=inf), dict(max_steer=nan), dict(max_steer=120.0), dict(maxiter=-1),
                   dict(eps=nan), dict(Q=(3, nan)), dict(R=(0, inf))):
            assert lqr(nx, po) == INV, (nx, po)
        for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(nc=0), dict(nc=-2), dict(npts=0), dict(npts=-5),
                   dict(st=None), dict(cx=None), dict(ck=None), dict(off=None), dict(of=None), dict(ind=None),
                   dict(u=None)):
            assert lqr(nx, **kw) == INV, (nx, kw)
    assert lqr(4, sp=d) == INV and lqr(5, sp=None) == INV
    for nx in (0, 3, 6):
        assert lqr(nx, sp=d) == INV and lqr(nx) == INV

    def mpc(params=None, **over):
        p = params if params is not None else _lib.MpcParams()
        if params is None:
            L.crb_mpc_default_params(C.byref(p))
        a = dict(dict(ctx=ctx, n=5, T=20, st=d, cx=d, sp=d, off=d, nc=3, npts=100, of=d, dl=1.0, ti=d, xr=d,
                      prm=C.byref(p)), **over)
        return L.crb_mpc_calc_ref_trajectory_many_batched(a["ctx"], a["n"], a["T"], a["st"], a["cx"], d, d, a["sp"],
                                                          a["off"], a["nc"], a["npts"], a["of"], C.c_float(a["dl"]),
                                                          a["ti"], a["xr"], None, a["prm"])

    for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(T=0), dict(T=_lib.CRB_MPC_MAX_T + 1), dict(dl=0.0),
               dict(dl=-1.0), dict(dl=nan), dict(nc=0), dict(npts=0), dict(st=None), dict(cx=None), dict(sp=None),
               dict(off=None), dict(of=None), dict(ti=None), dict(xr=None)):
        assert mpc(**kw) == INV, kw
    for dt in (0.0, -0.2, nan, inf):
        p = _lib.MpcParams()
        L.crb_mpc_default_params(C.byref(p))
        p.dt = dt
        assert mpc(p) == INV and mpc(p, n=0) == INV, dt
    # n = 0 needs no arrays
    assert mpc(n=0, st=None, cx=None, sp=None, off=None, of=None, ti=None, xr=None) == _lib.CRB_OK
    if not torch.cuda.is_available():
        assert lqr(4) == _lib.CRB_ERR_NO_DEVICE and lqr(5, n=0, st=None, off=None, of=None) == _lib.CRB_ERR_NO_DEVICE


def test_pack_courses_round_trips():
    courses = synth.fleet_courses(50, seed=7)
    packed = synth.pack_courses(courses)
    off = packed[5]
    assert off.dtype == np.int64 and off.shape == (51,) and off[0] == 0 and off[-1] == packed[0].size
    for f in range(5):
        assert packed[f].dtype == np.float32 and packed[f].flags["C_CONTIGUOUS"]
    for c, course in enumerate(courses):
        for f in range(5):
            assert _bits_equal(packed[f][off[c]:off[c + 1]], course[f]), (c, f)


def test_fleet_courses_is_deterministic_and_varied():
    a, b = synth.fleet_courses(64, seed=11), synth.fleet_courses(64, seed=11)
    assert all(_bits_equal(x, y) for ca, cb in zip(a, b) for x, y in zip(ca, cb))
    c = synth.fleet_courses(64, seed=12)
    assert not all(len(x[0]) == len(y[0]) and _bits_equal(x[0], y[0]) for x, y in zip(a, c))
    lens = np.array([len(x[0]) for x in a])
    assert (lens == 1).sum() >= 4 and lens.max() > 300 and len(set(lens.tolist())) > 30
    starts = np.array([(x[0][0], x[1][0]) for x in a])
    assert np.ptp(starts[:, 0]) > 200 and np.ptp(starts[:, 1]) > 200          # translated
    for x in a:
        assert all(len(f) == len(x[0]) and f.dtype == np.float32 for f in x)


def test_new_kernels_do_not_spill():
    found = []
    for src, kernel in (("crb_lqr_track.cu", "crb_lqr_track_many_kernel"), ("crb_mpc.cu", "crb_mpc_lookup_many_kernel")):
        for name, f in ptxas_kernels(src).items():
            if kernel in name:
                found.append(kernel)
                assert (f.stack, f.spill_stores, f.spill_loads) == (0, 0, 0), f
    assert found.count("crb_lqr_track_many_kernel") == 2 and found.count("crb_mpc_lookup_many_kernel") == 1


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "track_many_ref_api.cpp")


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    return t.cpu().numpy()


def _eng_params(p):
    q = lqr_track_default_params(4)
    C.memmove(C.byref(q), C.byref(p), C.sizeof(q))
    return q


def course_sets():
    """(name, courses): fleet courses of random length (1-point ones among them), the demo course, a 50 000-point
    course and a 1-point course, shuffled together."""
    rng = np.random.default_rng(0xC0A5)
    long = tuple(a[:50_000] for a in synth.lqr_course("sine", ds=59.0 / 50_000))
    one = tuple(np.float32([v]) for v in (2.0, -1.0, 0.7, 0.25, 1.5))
    mixed = synth.fleet_courses(40, seed=3) + [synth.lqr_course("demo"), long, one, synth.lqr_course("demo_speed")]
    order = rng.permutation(len(mixed))
    return [("mixed", [mixed[k] for k in order]), ("demo_fleet", synth.fleet_courses(300, seed=5))]


def fleet_inputs(n, courses, seed):
    """Vehicles in random order over the courses: course_of [n] and each vehicle's state, ind, pe, pth_e drawn around
    its own course by synth.lqr_track_inputs."""
    rng = np.random.default_rng(seed)
    course_of = rng.integers(0, len(courses), n).astype(np.int32)
    state = np.zeros((4, n), np.float32)
    ind, pe, pth = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    for c in np.unique(course_of):
        sel = np.nonzero(course_of == c)[0]
        s, i, e, t = synth.lqr_track_inputs(sel.size, courses[c], seed=int(seed * 7919 + c))
        state[:, sel], ind[sel], pe[sel], pth[sel] = s, i, e, t
    return course_of, np.ascontiguousarray(state), ind, pe, pth


def gpu_many(engine, nx, packed, course_of, state, ind, pe, pth_e, p=None, with_k=True):
    import torch
    n = state.shape[1]
    nu = 1 if nx == 4 else 2
    dind, dpe, dpth = _dev(np.array(ind, np.int32)), _dev(np.array(pe, np.float32)), _dev(np.array(pth_e, np.float32))
    K = torch.full((nu * nx, n), 7.0, dtype=torch.float32, device="cuda:0") if with_k else None
    dc = [_dev(a) for a in packed]
    courses = dc[:4] + dc[5:] if nx == 4 else dc
    r = engine.lqr_steering_control_many(nx, _dev(state), courses, _dev(course_of), dind, dpe, dpth,
                                         _eng_params(p) if p is not None else None, K=K)
    torch.cuda.synchronize()
    out = dict(u=_host(r["u"]), ind=_host(dind), pe=_host(dpe), pth_e=_host(dpth), iters=_host(r["iters"]),
               status=_host(r["status"]))
    if with_k:
        out["K"] = _host(K)
    return out


def per_course(nx, courses, course_of, state, ind, pe, pth_e, run):
    """run(course, state, ind, pe, pth_e) -> dict, once per course on its own vehicles, scattered back."""
    n = state.shape[1]
    nu = 1 if nx == 4 else 2
    out = dict(u=np.zeros((nu, n), np.float32), K=np.zeros((nu * nx, n), np.float32), ind=np.array(ind, np.int32),
               pe=np.array(pe, np.float32), pth_e=np.array(pth_e, np.float32), iters=np.zeros(n, np.int32),
               status=np.zeros(n, np.int32))
    for c in np.unique(course_of):
        sel = np.nonzero(course_of == c)[0]
        r = run(courses[c], np.ascontiguousarray(state[:, sel]), ind[sel], pe[sel], pth_e[sel])
        for k in out:
            if k in r:
                out[k][..., sel] = r[k]
    return out


def single_gpu(engine, nx, p=None):
    from test_lqr_track import gpu_control

    def run(course, st, i, e, t):
        return gpu_control(engine, nx, st, course, i, e, t, p)
    return run


def checker(nx, p=None):
    def run(course, st, i, e, t):
        return OL.control(nx, st, course, i, e, t, p)
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_lqr_many_is_the_single_course_entry_per_course(engine, nx):
    for name, courses in course_sets():
        packed = synth.pack_courses(courses)
        for n in (1, 33, 4097, 65536):
            course_of, state, ind, pe, pth = fleet_inputs(n, courses, seed=n + len(courses))
            got = gpu_many(engine, nx, packed, course_of, state, ind, pe, pth)
            assert_same(got, per_course(nx, courses, course_of, state, ind, pe, pth, single_gpu(engine, nx)), ALL)
            assert_same(got, per_course(nx, courses, course_of, state, ind, pe, pth, checker(nx)), ALL)
            assert (got["status"] != _lib.CRB_LQR_TRACK_BAD_COURSE).all(), (name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_lqr_many_with_non_default_params(engine, nx):
    courses = course_sets()[0][1]
    packed = synth.pack_courses(courses)
    course_of, state, ind, pe, pth = fleet_inputs(4097, courses, seed=0xBEEF)
    for p in nondefault_params(nx):
        got = gpu_many(engine, nx, packed, course_of, state, ind, pe, pth, p)
        assert_same(got, per_course(nx, courses, course_of, state, ind, pe, pth, single_gpu(engine, nx, p)), ALL)
        assert_same(got, per_course(nx, courses, course_of, state, ind, pe, pth, checker(nx, p)), ALL)


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_lqr_many_launch_forms(engine, nx):
    """NULL optional outputs, n = 0 and a graph-captured launch give the same bits."""
    import torch
    courses = synth.fleet_courses(64, seed=21)
    packed = synth.pack_courses(courses)
    n = 5000
    course_of, state, ind, pe, pth = fleet_inputs(n, courses, seed=0xF0F0)
    want = per_course(nx, courses, course_of, state, ind, pe, pth, checker(nx))
    assert_same(gpu_many(engine, nx, packed, course_of, state, ind, pe, pth, with_k=False), want)
    dc = [_dev(a) for a in packed]
    prm = lqr_track_default_params(nx)
    sp = dc[4].data_ptr() if nx == 5 else None
    assert engine.lib.crb_lqr_steering_control_many_batched(
        engine.ctx, 0, nx, None, dc[0].data_ptr(), dc[1].data_ptr(), dc[2].data_ptr(), dc[3].data_ptr(), sp,
        dc[5].data_ptr(), len(courses), packed[0].size, None, C.byref(prm), None, None, None, None, None, None,
        None) == 0
    courses_d = dc[:4] + dc[5:] if nx == 4 else dc
    dst, dof, dind, dpe, dpth = _dev(state), _dev(course_of), _dev(ind), _dev(pe), _dev(pth)
    nu = 1 if nx == 4 else 2
    u = torch.empty((nu, n), dtype=torch.float32, device="cuda:0")
    it = torch.empty(n, dtype=torch.int32, device="cuda:0")
    stt = torch.empty(n, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        eng = type(engine)(0)
        try:
            with torch.cuda.graph(g, stream=s):
                eng.lqr_steering_control_many(nx, dst, courses_d, dof, dind, dpe, dpth, u=u, iters=it, status=stt)
            g.replay()
            torch.cuda.synchronize()
        finally:
            eng.close()
    got = dict(u=_host(u), ind=_host(dind), pe=_host(dpe), pth_e=_host(dpth), iters=_host(it), status=_host(stt))
    assert_same(got, want, ("u", "ind", "pe", "pth_e", "iters", "status"))


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_lqr_many_bad_course_references(engine, nx):
    import torch
    courses = synth.fleet_courses(32, seed=31)
    packed = synth.pack_courses(courses)
    off = packed[5].copy()
    npts = packed[0].size
    n = 4097
    course_of, state, ind, pe, pth = fleet_inputs(n, courses, seed=0xBAD)
    # three more courses in the store: 32 is empty, 33 decreasing, 34 ends past npts
    off_bad = np.concatenate([off, [off[-1], off[-1] - 3, off[-1] + 10 ** 6]])
    n_courses = len(off_bad) - 1
    rng = np.random.default_rng(5)
    bad = rng.random(n) < 0.2
    kinds = np.array([32, 33, 34, -1, n_courses, 2 ** 31 - 1, -(2 ** 31)], np.int64)
    cof = course_of.astype(np.int64)
    cof[bad] = kinds[rng.integers(0, kinds.size, int(bad.sum()))]
    cof = cof.astype(np.int32)
    nu = 1 if nx == 4 else 2
    dind, dpe, dpth = _dev(ind), _dev(pe), _dev(pth)
    K = torch.full((nu * nx, n), 7.0, dtype=torch.float32, device="cuda:0")
    dc = [_dev(a) for a in packed[:5]] + [_dev(off_bad)]
    r = engine.lqr_steering_control_many(nx, _dev(state), dc[:4] + dc[5:] if nx == 4 else dc, _dev(cof), dind, dpe,
                                         dpth, K=K)
    torch.cuda.synchronize()
    got = dict(u=_host(r["u"]), K=_host(K), ind=_host(dind), pe=_host(dpe), pth_e=_host(dpth), iters=_host(r["iters"]),
               status=_host(r["status"]))
    assert (got["status"][bad] == _lib.CRB_LQR_TRACK_BAD_COURSE).all()
    assert np.isnan(got["u"][:, bad]).all() and np.isnan(got["K"][:, bad]).all() and (got["iters"][bad] == 0).all()
    assert _bits_equal(got["ind"][bad], ind[bad]) and _bits_equal(got["pe"][bad], pe[bad])
    assert _bits_equal(got["pth_e"][bad], pth[bad])
    ok = ~bad
    want = per_course(nx, courses, course_of[ok], state[:, ok], ind[ok], pe[ok], pth[ok], checker(nx))
    assert_same({k: v[..., ok] for k, v in got.items()}, want, ALL)
    # a store whose last offset is past npts: only the vehicles on that course are refused
    off_past = off.copy()
    off_past[-1] = npts + 1
    r = engine.lqr_steering_control_many(nx, _dev(state), (dc[:4] if nx == 4 else dc[:5]) + [_dev(off_past)],
                                         _dev(course_of), _dev(ind), _dev(pe), _dev(pth))
    torch.cuda.synchronize()
    st = _host(r["status"])
    assert ((st == _lib.CRB_LQR_TRACK_BAD_COURSE) == (course_of == len(courses) - 1)).all()


@pytest.mark.gpu
def test_gpu_lqr_many_ind_persists_and_bad_index_per_course(engine):
    """4 states: ind carries over between calls on each vehicle's own course; a course whose distances are all NaN
    gives BAD_INDEX where the incoming ind is outside that course, and keeps ind where it is inside."""
    courses = synth.fleet_courses(24, seed=41)
    nan_course = tuple(np.full(9, np.nan, np.float32) if f < 2 else np.linspace(0, 1, 9).astype(np.float32)
                       for f in range(5))
    courses = courses[:10] + [nan_course] + courses[10:]
    packed = synth.pack_courses(courses)
    n = 4097
    course_of, state, ind, pe, pth = fleet_inputs(n, courses, seed=0x1D)
    on_nan = course_of == 10
    rng = np.random.default_rng(2)
    ind[on_nan] = rng.choice(np.int32([-1, 0, 4, 8, 9, 50, 2 ** 31 - 1]), int(on_nan.sum()))
    for _ in range(3):      # the outputs of one call are the inputs of the next
        got = gpu_many(engine, 4, packed, course_of, state, ind, pe, pth)
        want = per_course(4, courses, course_of, state, ind, pe, pth, checker(4))
        assert_same(got, want, ALL)
        bad = on_nan & ((ind < 0) | (ind >= 9))
        assert bad.any() and (got["status"][bad] == _lib.CRB_LQR_TRACK_BAD_INDEX).all()
        assert (got["status"][on_nan & ~bad] != _lib.CRB_LQR_TRACK_BAD_INDEX).all()
        assert (got["ind"][on_nan] == ind[on_nan]).all()
        ind, pe, pth = got["ind"], got["pe"], got["pth_e"]
        state = state.copy()
        state[:2] += np.float32(0.3)


def lqr_closed_loop_checker(nx, courses, course_of, state0, ticks):
    n = state0.shape[1]
    state = state0.copy()
    ind, pe, pth_e = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    lens = np.array([len(c[0]) for c in courses])
    hist = []
    for _ in range(ticks):
        r = per_course(nx, courses, course_of, state, ind, pe, pth_e, checker(nx))
        ind, pe, pth_e = r["ind"], r["pe"], r["pth_e"]
        if nx == 4:
            di = r["u"][0]
            spv = np.array([courses[c][4][min(max(j, 0), lens[c] - 1)] for c, j in zip(course_of, ind)], np.float32)
            ai = (np.float32(KP) * (spv - state[3])).astype(np.float32)
        else:
            ai, di = r["u"][0], r["u"][1]
        state = OL.update(state, ai, di)
        if nx == 4:
            ind = np.where(np.abs(state[3]) <= np.float32(STOP_SPEED), ind + 1, ind).astype(np.int32)
        hist.append((state.copy(), r["u"].copy(), ind.copy()))
    return hist


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_lqr_many_closed_loop_is_the_checker_at_every_tick(engine, nx):
    """4096 vehicles on 64 courses, 300 ticks of control and update driven by the test, every tick against the checker
    composed per course."""
    import torch
    courses = synth.fleet_courses(64, seed=0x64)
    packed = synth.pack_courses(courses)
    n, ticks = 4096, 300
    course_of, state0, _, _, _ = fleet_inputs(n, courses, seed=0xC10)
    state0[3] = np.abs(state0[3])
    hist = lqr_closed_loop_checker(nx, courses, course_of, state0, ticks)
    dc = [_dev(a) for a in packed]
    dcourses = dc[:4] + dc[5:] if nx == 4 else dc
    dsp, doff, dof = dc[4], dc[5], _dev(course_of)
    dst = _dev(state0)
    dind = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    dpe = torch.zeros(n, dtype=torch.float32, device="cuda:0")
    dpth = torch.zeros(n, dtype=torch.float32, device="cuda:0")
    nu = 1 if nx == 4 else 2
    u = torch.empty((nu, n), dtype=torch.float32, device="cuda:0")
    lens = doff[1:] - doff[:-1]
    start = doff[:-1][dof.long()]
    last = lens[dof.long()] - 1
    for tick in range(ticks):
        engine.lqr_steering_control_many(nx, dst, dcourses, dof, dind, dpe, dpth, u=u)
        if nx == 4:
            torch.cuda.synchronize()
            spv = dsp[start + torch.minimum(torch.clamp(dind.long(), min=0), last)]
            ai = (KP * (spv - dst[3])).contiguous()
            di = u[0].contiguous()
        else:
            ai, di = u[0].contiguous(), u[1].contiguous()
        torch.cuda.synchronize()
        engine.lqr_update(dst, ai, di)
        torch.cuda.synchronize()
        if nx == 4:
            dind = torch.where(dst[3].abs() <= STOP_SPEED, dind + 1, dind).to(torch.int32).contiguous()
        hs, hu, hind = hist[tick]
        assert _bits_equal(_host(u), hu), tick
        assert _bits_equal(_host(dst), hs), tick
        assert np.array_equal(_host(dind), hind), tick


# ---- H100: the MPC lookup -----------------------------------------------------------------------------------------------
def mpc_fleet(n, courses, seed):
    """course_of, state [4, n] and target_ind around each vehicle's own course (course-local), a few target_ind at and
    past the end of the course, and negative speeds."""
    rng = np.random.default_rng(seed)
    course_of = rng.integers(0, len(courses), n).astype(np.int32)
    lens = np.array([len(c[0]) for c in courses])
    state = np.zeros((4, n), np.float32)
    ti = np.zeros(n, np.int32)
    for c in np.unique(course_of):
        sel = np.nonzero(course_of == c)[0]
        s, i, _, _ = synth.lqr_track_inputs(sel.size, courses[c], seed=int(seed + 31 * c))
        state[:, sel] = s
        ti[sel] = np.maximum(i - rng.integers(0, 12, sel.size), 0)
    k = rng.random(n)
    ti = np.where(k < 0.05, lens[course_of] - 1 - rng.integers(0, 12, n), ti)
    ti = np.where((k >= 0.05) & (k < 0.08), lens[course_of] + rng.integers(0, 40, n), ti).astype(np.int32)
    ti = np.maximum(ti, np.int32(-9))
    return course_of, np.ascontiguousarray(state), ti


def gpu_lookup_many(engine, packed, course_of, state, ti, T, dl, prm=None, with_status=True):
    import torch
    n = state.shape[1]
    dti = _dev(ti)
    xr = torch.full((4 * T, n), 7.0, dtype=torch.float32, device="cuda:0")
    dc = [_dev(a) for a in packed]
    stt = torch.full((n,), 9, dtype=torch.int32, device="cuda:0") if with_status else None
    r = engine.calc_ref_trajectory_many(_dev(state), (dc[0], dc[1], dc[2], dc[4], dc[5]), _dev(course_of), dl, dti,
                                        xr, T, prm, status=stt)
    torch.cuda.synchronize()
    return _host(xr), _host(dti), _host(r)


def lookup_per_course(courses, course_of, state, ti, T, dl, run):
    n = state.shape[1]
    xr, to = np.zeros((4 * T, n), np.float32), np.array(ti, np.int32)
    for c in np.unique(course_of):
        sel = np.nonzero(course_of == c)[0]
        x, t = run(courses[c], np.ascontiguousarray(state[:, sel]), ti[sel])
        xr[:, sel], to[sel] = x, t
    return xr, to


def single_lookup(engine, T, dl, prm=None):
    import torch

    def run(course, st, ti):
        dti = _dev(ti)
        xr = torch.empty((4 * T, st.shape[1]), dtype=torch.float32, device="cuda:0")
        cx, cy, cyaw, _, sp = (_dev(a) for a in course)
        engine.calc_ref_trajectory(_dev(st), cx, cy, cyaw, sp, dl, dti, xr, T, prm)
        torch.cuda.synchronize()
        return _host(xr), _host(dti)
    return run


def checker_lookup(T, dl, prm=None):
    def run(course, st, ti):
        cx, cy, cyaw, _, sp = course
        xr = np.zeros((4 * T, st.shape[1]), np.float32)
        to = np.zeros(st.shape[1], np.int32)
        for i in range(st.shape[1]):
            x, to[i] = O.calc_ref_trajectory(st[:, i], cx, cy, cyaw, sp, dl, T, int(ti[i]), params=prm)
            xr[:, i] = x.reshape(-1)
        return xr, to
    return run


def checker_defined(courses, course_of, ti):
    """Agents whose target_ind the checker handles without reading outside the course: it reads cx[target_ind] when
    target_ind is past the end (as the reference does, :141-144), and its window of a target_ind below -9 runs over
    indices at or past 2^31.  The device entries never read there; past the end they are compared with the
    single-course entry only."""
    lens = np.array([len(c[0]) for c in courses])
    return (ti >= -9) & (ti < lens[course_of])


@pytest.mark.gpu
def test_gpu_lookup_many_is_the_single_course_entry_per_course(engine):
    for name, courses in course_sets():
        packed = synth.pack_courses(courses)
        for n in (1, 33, 4097, 65536):
            course_of, state, ti = mpc_fleet(n, courses, seed=n + 1)
            for T, dl in ((20, 1.0), (5, 0.1)):
                got_x, got_t, stt = gpu_lookup_many(engine, packed, course_of, state, ti, T, dl)
                assert (stt == _lib.CRB_MPC_REF_OK).all()
                wx, wt = lookup_per_course(courses, course_of, state, ti, T, dl, single_lookup(engine, T, dl))
                assert _bits_equal(got_x, wx) and np.array_equal(got_t, wt), (name, n, T)
                if n <= 4097:
                    d = checker_defined(courses, course_of, ti)
                    cx_, ct_ = lookup_per_course(courses, course_of[d], state[:, d], ti[d], T, dl,
                                                 checker_lookup(T, dl))
                    assert _bits_equal(got_x[:, d], cx_) and np.array_equal(got_t[d], ct_), (name, n, T)


@pytest.mark.gpu
def test_gpu_lookup_many_non_default_params_and_target_ind_outside(engine):
    """A non-default dt, T = CRB_MPC_MAX_T, and target_ind outside every course (below 0, at and far past the end,
    INT32_MAX): the single-course entry's behaviour per course; the checker where its index arithmetic is defined."""
    courses = course_sets()[0][1]
    packed = synth.pack_courses(courses)
    n = 4097
    course_of, state, ti = mpc_fleet(n, courses, seed=0xD7)
    rng = np.random.default_rng(9)
    lens = np.array([len(c[0]) for c in courses])
    out = rng.random(n) < 0.3
    extreme = np.int64([-1, -9, -10, -500, -(2 ** 31), 2 ** 30, 2 ** 31 - 1])
    far = rng.random(n) < 0.5
    pick = np.where(far, extreme[rng.integers(0, extreme.size, n)], lens[course_of] + rng.integers(0, 3, n))
    ti = np.where(out, pick, ti).astype(np.int32)
    prm = _lib.MpcParams()
    _lib.load_library().crb_mpc_default_params(C.byref(prm))
    prm.dt = 0.15
    T = _lib.CRB_MPC_MAX_T
    got_x, got_t, stt = gpu_lookup_many(engine, packed, course_of, state, ti, T, 0.5, prm)
    assert (stt == _lib.CRB_MPC_REF_OK).all()
    wx, wt = lookup_per_course(courses, course_of, state, ti, T, 0.5, single_lookup(engine, T, 0.5, prm))
    assert _bits_equal(got_x, wx) and np.array_equal(got_t, wt)
    defined = checker_defined(courses, course_of, ti)
    assert (~defined).sum() > 500
    cx_, ct_ = lookup_per_course(courses, course_of[defined], state[:, defined], ti[defined], T, 0.5,
                                 checker_lookup(T, 0.5, prm))
    assert _bits_equal(got_x[:, defined], cx_) and np.array_equal(got_t[defined], ct_)


@pytest.mark.gpu
def test_gpu_lookup_many_launch_forms_and_bad_courses(engine):
    """NULL status, n = 0, a graph-captured launch, and bad course references (NaN xref, target_ind untouched)."""
    import torch
    courses = synth.fleet_courses(64, seed=77)
    packed = synth.pack_courses(courses)
    n, T, dl = 5000, 12, 1.0
    course_of, state, ti = mpc_fleet(n, courses, seed=0x9A)
    ti = np.minimum(ti, np.array([len(c[0]) for c in courses])[course_of] - 1).astype(np.int32)
    want = lookup_per_course(courses, course_of, state, ti, T, dl, checker_lookup(T, dl))
    gx, gt, _ = gpu_lookup_many(engine, packed, course_of, state, ti, T, dl, with_status=False)
    assert _bits_equal(gx, want[0]) and np.array_equal(gt, want[1])
    dc = [_dev(a) for a in packed]
    prm = _lib.MpcParams()
    engine.lib.crb_mpc_default_params(C.byref(prm))
    assert engine.lib.crb_mpc_calc_ref_trajectory_many_batched(
        engine.ctx, 0, T, None, dc[0].data_ptr(), dc[1].data_ptr(), dc[2].data_ptr(), dc[4].data_ptr(),
        dc[5].data_ptr(), len(courses), packed[0].size, None, C.c_float(dl), None, None, None, C.byref(prm)) == 0
    # graph capture
    dst, dof, dti = _dev(state), _dev(course_of), _dev(ti)
    xr = torch.empty((4 * T, n), dtype=torch.float32, device="cuda:0")
    stt = torch.empty(n, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        eng = type(engine)(0)
        try:
            with torch.cuda.graph(g, stream=s):
                eng.calc_ref_trajectory_many(dst, (dc[0], dc[1], dc[2], dc[4], dc[5]), dof, dl, dti, xr, T, status=stt)
            g.replay()
            torch.cuda.synchronize()
        finally:
            eng.close()
    assert _bits_equal(_host(xr), want[0]) and np.array_equal(_host(dti), want[1])
    assert (_host(stt) == _lib.CRB_MPC_REF_OK).all()
    # bad references: an empty course, a decreasing pair, offsets past npts, course_of out of range
    off = packed[5]
    off_bad = np.concatenate([off, [off[-1], off[-1] - 3, off[-1] + 10 ** 6]])
    n_courses = len(off_bad) - 1
    rng = np.random.default_rng(3)
    bad = rng.random(n) < 0.2
    kinds = np.int64([64, 65, 66, -1, n_courses, 2 ** 31 - 1])
    cof = np.where(bad, kinds[rng.integers(0, kinds.size, n)], course_of).astype(np.int32)
    dti = _dev(ti)
    xr = torch.full((4 * T, n), 7.0, dtype=torch.float32, device="cuda:0")
    stt = engine.calc_ref_trajectory_many(_dev(state), (dc[0], dc[1], dc[2], dc[4], _dev(off_bad)), _dev(cof), dl,
                                          dti, xr, T)
    torch.cuda.synchronize()
    gx, gt, st = _host(xr), _host(dti), _host(stt)
    assert (st[bad] == _lib.CRB_MPC_REF_BAD_COURSE).all() and (st[~bad] == _lib.CRB_MPC_REF_OK).all()
    assert np.isnan(gx[:, bad]).all() and np.array_equal(gt[bad], ti[bad])
    assert _bits_equal(gx[:, ~bad], want[0][:, ~bad]) and np.array_equal(gt[~bad], want[1][~bad])


@pytest.mark.gpu
def test_gpu_reference_style_program_runs(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = subprocess.check_output([build_ref_program(tmp_path, "track_many_ref_api.cpp")], text=True)
    lines = out.strip().splitlines()
    assert len(lines) == 2 and lines[0].startswith("lqr_steer_control") and "nan" not in out
