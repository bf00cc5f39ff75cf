"""LQR path tracking: lqr_steering_control (with calc_nearest_index) and update of src/lqr_steer_control.cpp (4 states)
and src/lqr_speed_steer_control.cpp (5 states).

CPU: the checker (oracle/crb_oracle_lqrt.c) is bitwise the reference text compiled through oracle/shim (oracle/_ref) on
every course kind, corner cases and a test-driven closed loop; with non-default parameters it is checked against a
numpy composition of the reference-pinned dlqr restatement; plus the golden fixture, argument validation without a
device, the C++ program and the compiler report.
H100 (-m gpu): every output of crb_lqr_steering_control_batched and crb_lqr_update_batched is bitwise the checker, in a
closed loop too, and the feed-forward is the host's (float)atan2(0.5 * (double)k, 1.0) on every non-negative float."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import lqr_track_cases as LC
from cpprobotics_b200 import _lib, lqr_track_default_params, synth
from oracle import lqrt as OL
from oracle import oracle as O
from oracle._load import reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lqr_track_golden.npz")
CPP_API = os.path.join(ROOT, "tests", "cpp", "lqr_ref_api.cpp")
f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
KP, STOP_SPEED = 1.0, 0.05


def _bits_equal(a, b):
    """Bitwise equality with every NaN equal to every NaN (payloads aside)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))
    return bool(np.array_equal(a, b))


# ---- the reference text (oracle/_ref) --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    libs = {}
    for nx in (4, 5):
        L = reference(f"lqrt{nx}")
        if L is None:
            pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
        i32r = C.POINTER(C.c_int)
        fr = C.POINTER(C.c_float)
        getattr(L, f"ref_lqr_nearest{nx}").restype = C.c_float
        getattr(L, f"ref_lqr_nearest{nx}").argtypes = [f32p, f32p, f32p, f32p, C.c_int, i32r]
        getattr(L, f"ref_lqr_update{nx}").restype = None
        getattr(L, f"ref_lqr_update{nx}").argtypes = [f32p, C.c_float, C.c_float]
        if nx == 4:
            L.ref_lqr_control4.restype = C.c_float
            L.ref_lqr_control4.argtypes = [f32p, f32p, f32p, f32p, f32p, C.c_int, i32r, fr, fr]
        else:
            L.ref_lqr_control5.restype = None
            L.ref_lqr_control5.argtypes = [f32p, f32p, f32p, f32p, f32p, f32p, C.c_int, fr, fr, f32p]
        libs[nx] = L
    return libs


def ref_control(L, nx, state, course, ind, pe, pth_e):
    """The reference's lqr_steering_control per vehicle (and, for nx 5, its calc_nearest_index from 0 for ind)."""
    cx, cy, cyaw, ck = (np.ascontiguousarray(a, np.float32) for a in course[:4])
    nc = cx.size
    n = state.shape[1]
    nu = 1 if nx == 4 else 2
    u = np.zeros((nu, n), np.float32)
    ind, pe, pth_e = np.array(ind, np.int32), np.array(pe, np.float32), np.array(pth_e, np.float32)
    for i in range(n):
        st = np.ascontiguousarray(state[:, i])
        e, t = C.c_float(pe[i]), C.c_float(pth_e[i])
        if nx == 4:
            j = C.c_int(int(ind[i]))
            u[0, i] = L.ref_lqr_control4(st, cx, cy, cyaw, ck, nc, C.byref(j), C.byref(e), C.byref(t))
        else:
            out = np.zeros(2, np.float32)
            L.ref_lqr_control5(st, cx, cy, cyaw, ck, np.ascontiguousarray(course[4], np.float32), nc, C.byref(e),
                               C.byref(t), out)
            u[:, i] = out
            j = C.c_int(0)
            L.ref_lqr_nearest5(st, cx, cy, cyaw, nc, C.byref(j))
        ind[i], pe[i], pth_e[i] = j.value, e.value, t.value
    return dict(u=u, ind=ind, pe=pe, pth_e=pth_e)


def assert_same(got, want, keys=("u", "ind", "pe", "pth_e")):
    for k in keys:
        assert _bits_equal(got[k], want[k]), (k, np.nonzero(~((got[k] == want[k]) | (np.isnan(got[k]) & np.isnan(want[k])) if np.asarray(got[k]).dtype.kind == "f" else got[k] != want[k]))[0][:10])  # noqa: E501


@pytest.mark.parametrize("nx", [4, 5])
@pytest.mark.parametrize("kind", synth.LQR_KINDS)
def test_checker_is_the_reference_text_on_every_course(ref, nx, kind):
    course = synth.lqr_course(kind)
    state, ind, pe, pth_e = synth.lqr_track_inputs(10_000, course, seed=hash(kind) & 0xFFFF)
    got = OL.control(nx, state, course, ind, pe, pth_e)
    assert_same(got, ref_control(ref[nx], nx, state, course, ind, pe, pth_e))
    assert (got["status"] != OL.BAD_INDEX).all()
    # calc_nearest_index on its own: the signed squared distance and the index
    L = ref[nx]
    cx, cy, cyaw = course[:3]
    for i in range(0, 10_000, 97):
        st = np.ascontiguousarray(state[:, i])
        j = C.c_int(int(ind[i]))
        e = getattr(L, f"ref_lqr_nearest{nx}")(st, cx, cy, cyaw, cx.size, C.byref(j))
        assert _bits_equal(np.float32(e), np.float32(OL.nearest(st, course, int(ind[i]))[0]))
        assert j.value == OL.nearest(st, course, int(ind[i]))[1]


@pytest.mark.parametrize("nx", [4, 5])
def test_checker_is_the_reference_text_on_corner_cases(ref, nx):
    for course in (synth.lqr_course("demo"), synth.lqr_course("circle"), LC.duplicate_course()[0],
                   LC.single_point_course()):
        state, ind, pe, pth_e = LC.corner_states(course)
        got = OL.control(nx, state, course, ind, pe, pth_e)
        assert_same(got, ref_control(ref[nx], nx, state, course, ind, pe, pth_e))
    course, st = LC.duplicate_course()
    n = st.shape[1]
    z = np.zeros(n, np.float32)
    got = OL.control(nx, st, course, np.zeros(n, np.int32), z, z)
    assert_same(got, ref_control(ref[nx], nx, st, course, np.zeros(n, np.int32), z, z))
    assert got["ind"][0] == 1 and got["ind"][2] == 0      # the first of equal minima wins
    # v = 0: solve_DARE never converges and returns its last X
    course = synth.lqr_course("demo")
    state, ind, pe, pth_e = LC.corner_states(course)
    r = OL.control(nx, state, course, ind, pe, pth_e)
    v0 = state[3] == 0
    assert v0.any() and (r["status"][v0] == OL.DARE_MAXITER).all() and (r["iters"][v0] == 150).all()
    far = np.maximum(np.abs(state[0]), np.abs(state[1])) >= 1e20
    assert far.sum() >= 8 and (r["ind"][far] == (ind[far] if nx == 4 else 0)).all()


@pytest.mark.parametrize("nx", [4, 5])
def test_update_is_the_reference_text(ref, nx):
    st, a, delta = LC.update_cases()
    got = OL.update(st, a, delta)
    L = ref[nx]
    want = st.copy()
    for i in range(st.shape[1]):
        s = np.ascontiguousarray(want[:, i])
        getattr(L, f"ref_lqr_update{nx}")(s, float(a[i]), float(delta[i]))
        want[:, i] = s
    assert _bits_equal(got, want)


def closed_loop_checker(nx, course, state0, ticks, params=None):
    """The test-driven closed loop of closed_loop_prediction's body: nx 4 uses ai = KP * (sp[ind] - v) and advances ind
    when |v| <= stop_speed; nx 5 uses the controller's ai.  Returns the per-tick (state, u, ind) history."""
    n = state0.shape[1]
    state = state0.copy()
    ind, pe, pth_e = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    sp = course[4]
    hist = []
    for _ in range(ticks):
        r = OL.control(nx, state, course, ind, pe, pth_e, params)
        ind, pe, pth_e = r["ind"], r["pe"], r["pth_e"]
        if nx == 4:
            di = r["u"][0]
            ai = (np.float32(KP) * (sp[np.clip(ind, 0, len(sp) - 1)] - state[3])).astype(np.float32)
        else:
            ai, di = r["u"][0], r["u"][1]
        state = OL.update(state, ai, di, params)
        if nx == 4:
            ind = np.where(np.abs(state[3]) <= np.float32(STOP_SPEED), ind + 1, ind).astype(np.int32)
        hist.append((state.copy(), r["u"].copy(), ind.copy()))
    return hist


@pytest.mark.parametrize("nx", [4, 5])
def test_closed_loop_checker_is_the_reference_tick_by_tick(ref, nx):
    course, s0 = LC.demo_start(nx)
    hist = closed_loop_checker(nx, course, s0.reshape(4, 1), 600)
    L = ref[nx]
    cx, cy, cyaw, ck, sp = course
    st = s0.copy()
    j, e, t = C.c_int(0), C.c_float(0.0), C.c_float(0.0)
    for tick, (hs, hu, hind) in enumerate(hist):
        if nx == 4:
            di = L.ref_lqr_control4(st, cx, cy, cyaw, ck, cx.size, C.byref(j), C.byref(e), C.byref(t))
            ai = np.float32(KP * (sp[j.value] - st[3]))
            assert _bits_equal(np.float32([di]), hu[:, 0]), tick
        else:
            out = np.zeros(2, np.float32)
            L.ref_lqr_control5(st, cx, cy, cyaw, ck, sp, cx.size, C.byref(e), C.byref(t), out)
            ai, di = out
            assert _bits_equal(out, hu[:, 0]), tick
        L_upd = getattr(L, f"ref_lqr_update{nx}")
        L_upd(st, float(ai), float(di))
        if nx == 4 and abs(float(st[3])) <= STOP_SPEED:
            j.value += 1
        assert _bits_equal(st, hs[:, 0]), tick
        if nx == 4:
            assert j.value == hind[0]
    # the loop tracks: the vehicle ends near the course
    assert np.hypot(*(hist[-1][0][:2, 0] - np.array([cx[-1], cy[-1]]))) < 30


# ---- non-default parameters: a numpy composition of the reference-pinned dlqr ------------------------------------------
def _yaw_p2p(a):
    return np.float32(np.fmod(np.fmod(np.float64(np.float32(a)) + np.pi, 2 * np.pi) - 2 * np.pi, 2 * np.pi) + np.pi)


def composed_control(nx, state, course, ind, pe, pth_e, p):
    cx, cy, cyaw, ck = course[:4]
    nu = 1 if nx == 4 else 2
    n = state.shape[1]
    out = dict(u=np.zeros((nu, n), np.float32), ind=np.zeros(n, np.int32), pe=np.zeros(n, np.float32),
               pth_e=np.zeros(n, np.float32), K=np.zeros((nu * nx, n), np.float32), iters=np.zeros(n, np.int32))
    Q = np.array(p.Q, np.float32).reshape(5, 5).T[:nx, :nx].T.reshape(-1).copy()   # column-major top-left block
    R = np.array(p.R, np.float32).reshape(2, 2).T[:nu, :nu].T.reshape(-1).copy()
    with np.errstate(all="ignore"):
        for i in range(n):
            x, y, yaw, v = state[:, i]
            e, j = OL.nearest(state[:, i], course, int(ind[i]) if nx == 4 else 0)
            e = np.float32(e)
            th_e = _yaw_p2p(np.float32(yaw - cyaw[j]))
            A = np.zeros((nx, nx), np.float32)
            B = np.zeros((nx, nu), np.float32)
            A[0, 0], A[0, 1], A[1, 2], A[2, 2], A[2, 3] = 1, np.float32(p.dt), v, 1, np.float32(p.dt)
            B[3, 0] = np.float32(np.float64(v) / p.wheelbase)
            if nx == 5:
                A[4, 4], B[4, 1] = 1, np.float32(p.dt)
            r = O.dlqr_batched(A.T.reshape(-1, 1).copy(), B.T.reshape(-1, 1).copy(), Q, R, nx, nu, maxiter=p.maxiter,
                               eps=p.eps)
            K = r["K"][:, 0]
            xv = [e, np.float32(np.float64(np.float32(e - pe[i])) / p.dt), th_e,
                  np.float32(np.float64(np.float32(th_e - pth_e[i])) / p.dt)]
            if nx == 5:
                xv.append(np.float32(v - course[4][j]))
            us = []
            for rr in range(nu):
                s = np.float32(-K[rr] * xv[0])
                for c in range(1, nx):
                    s = np.float32(s + np.float32(-K[rr + nu * c] * xv[c]))
                us.append(s)
            ff = np.float32(math.atan2(p.wheelbase * float(ck[j]), 1.0))   # the host libm's atan2
            delta = np.float32(ff + _yaw_p2p(us[0]))
            out["u"][:, i] = [delta] if nx == 4 else [us[1], delta]
            out["ind"][i], out["pe"][i], out["pth_e"][i] = j, e, th_e
            out["K"][:, i], out["iters"][i] = K, r["iters"][0]
    return out


def nondefault_params(nx):
    ps = []
    for dt, L, maxiter, eps, q, r in ((0.05, 0.8, 150, 0.01, 1.0, 1.0), (0.2, 2.5, 60, 1e-3, 3.0, 0.5),
                                      (0.1, 0.5, 0, 0.01, 1.0, 1.0), (0.1, 0.5, 1, 0.01, 1.0, 1.0),
                                      (0.1, 0.5, 40, 0.0, 1.0, 1.0), (0.07, 1.3, 200, 0.05, 0.25, 4.0)):
        p = OL.default_params(nx)
        p.dt, p.wheelbase, p.maxiter, p.eps = dt, L, maxiter, float(np.float32(eps))
        for f in range(25):
            p.Q[f] = q * (1.0 + 0.1 * (f // 6)) if f % 6 == 0 else (0.05 if f in (1, 5) else 0.0)
        p.R[0], p.R[3] = r, (r * 2 if nx == 5 else 0.0)
        p.max_steer = 0.6
        ps.append(p)
    return ps


@pytest.mark.parametrize("nx", [4, 5])
def test_checker_with_non_default_params_is_the_composition(nx):
    course = synth.lqr_course("sine")
    state, ind, pe, pth_e = synth.lqr_track_inputs(120, course, seed=0x5EED)
    for p in nondefault_params(nx):
        got = OL.control(nx, state, course, ind, pe, pth_e, p)
        assert_same(got, composed_control(nx, state, course, ind, pe, pth_e, p), ("u", "ind", "pe", "pth_e", "K",
                                                                                    "iters"))
        if p.maxiter == 0:
            assert (got["status"] == OL.DARE_MAXITER).all() and (got["iters"] == 0).all()
        if p.eps == 0.0:
            assert (got["status"] == OL.DARE_MAXITER).all()


def test_golden_fixture():
    g = np.load(GOLDEN)
    for nx in (4, 5):
        course = tuple(g[f"course{nx}"])
        r = OL.control(nx, g["state"], course, g["ind"], g["pe"], g["pth_e"])
        for k in ("u", "ind", "pe", "pth_e"):
            assert _bits_equal(r[k], g[f"{k}{nx}"]), (nx, k)
    assert _bits_equal(OL.update(g["ustate"], g["ua"], g["udelta"]), g["unew"])


# ---- host-side checks ---------------------------------------------------------------------------------------------------
def test_default_params_are_the_reference_constants():
    for nx in (4, 5):
        p = lqr_track_default_params(nx)
        q = OL.default_params(nx)
        assert bytes(p) == bytes(q)
        assert p.max_steer == 45.0 / 180 * np.pi and p.dt == 0.1 and p.wheelbase == 0.5 and p.maxiter == 150


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE without a GPU."""
    import torch
    L = _lib.load_library()
    inv = -1
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)

    def ctl(nx=4, po=None, **over):
        p = lqr_track_default_params(nx)
        for k, v in (po or {}).items():
            if k in ("Q", "R"):
                getattr(p, k)[v[0]] = v[1]
            else:
                setattr(p, k, v)
        a = dict(dict(ctx=ctx, n=5, st=d, cx=d, sp=d if nx == 5 else None, nc=10, prm=C.byref(p), ind=d, u=d), **over)
        return L.crb_lqr_steering_control_batched(a["ctx"], a["n"], nx, a["st"], a["cx"], d, d, d, a["sp"], a["nc"],
                                                  a["prm"], a["ind"], d, d, a["u"], None, None, None)

    def upd(po=None, **over):
        p = lqr_track_default_params(4)
        for k, v in (po or {}).items():
            setattr(p, k, v)
        a = dict(dict(ctx=ctx, n=5, st=d, prm=C.byref(p)), **over)
        return L.crb_lqr_update_batched(a["ctx"], a["n"], a["st"], d, d, a["prm"])

    nan, inf = float("nan"), float("inf")
    for nx in (4, 5):
        for po in (dict(dt=nan), dict(wheelbase=inf), dict(max_steer=nan), dict(max_steer=120.0),
                   dict(max_steer=-200.0), dict(maxiter=-1), dict(eps=nan), dict(eps=inf), dict(Q=(3, nan)),
                   dict(R=(0, inf))):
            assert ctl(nx, po) == inv, (nx, po)
        for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(nc=0), dict(nc=-3), dict(st=None), dict(cx=None),
                   dict(ind=None), dict(u=None)):
            assert ctl(nx, **kw) == inv, (nx, kw)
    assert ctl(4, sp=d) == inv and ctl(5, sp=None) == inv
    for nx in (3, 6, 0):
        assert L.crb_lqr_steering_control_batched(ctx, 5, nx, d, d, d, d, d, d, 10,
                                                  C.byref(lqr_track_default_params(5)), d, d, d, d, None, None,
                                                  None) == inv
    for po in (dict(dt=inf), dict(wheelbase=nan), dict(max_steer=inf), dict(max_steer=-121.0)):
        assert upd(po) == inv, po
    for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(st=None)):
        assert upd(**kw) == inv, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert ctl(4) == nd and ctl(5) == nd and ctl(4, n=0, st=None) == nd and upd() == nd
        assert ctl(4, dict(maxiter=0, eps=0.0, dt=-1.0, wheelbase=0.0)) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def _build_api(tmp_path):
    exe = str(tmp_path / "lqr_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           CPP_API, "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


def test_reference_style_program_compiles(tmp_path):
    _build_api(tmp_path)


def test_new_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-c", os.path.join(ROOT, "cpprobotics_b200", "csrc", "crb_lqr_track.cu"),
                          "-o", str(tmp_path / "lqrt.o")], capture_output=True, text=True, check=True).stderr
    blocks = out.split("Compiling entry function")[1:]
    names = [b.splitlines()[0] for b in blocks]
    assert sum("crb_lqr_steering_control_kernel" in s for s in names) == 2
    assert sum("crb_lqr_update_kernel" in s for s in names) == 1
    for b in out.split("Function properties for")[1:]:   # the kernels and the out-of-line libm pieces
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b.splitlines()[1], b
    # the refactored dlqr kernel too
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-c", os.path.join(ROOT, "cpprobotics_b200", "csrc", "crb_lqr.cu"),
                          "-o", str(tmp_path / "lqr.o")], capture_output=True, text=True, check=True).stderr
    for b in out.split("Function properties for")[1:]:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b.splitlines()[1], b


# ---- H100 -----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    return t.cpu().numpy()


def _eng_params(p):
    q = lqr_track_default_params(4)
    C.memmove(C.byref(q), C.byref(p), C.sizeof(q))
    return q


def gpu_control(engine, nx, state, course, ind, pe, pth_e, p=None, with_k=True):
    import torch
    nu = 1 if nx == 4 else 2
    n = state.shape[1]
    dind, dpe, dpth = _dev(np.array(ind, np.int32)), _dev(np.array(pe, np.float32)), _dev(np.array(pth_e, np.float32))
    K = torch.full((nu * nx, n), 7.0, dtype=torch.float32, device="cuda:0") if with_k else None
    r = engine.lqr_steering_control(nx, _dev(state), [_dev(a) for a in course[: 4 if nx == 4 else 5]], dind, dpe, dpth,
                                    _eng_params(p) if p is not None else None, K=K)
    torch.cuda.synchronize()
    out = dict(u=_host(r["u"]), ind=_host(dind), pe=_host(dpe), pth_e=_host(dpth), iters=_host(r["iters"]),
               status=_host(r["status"]))
    if with_k:
        out["K"] = _host(K)
    return out


ALL = ("u", "ind", "pe", "pth_e", "K", "iters", "status")


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_control_is_the_checker(engine, nx):
    demo = synth.lqr_course("demo")
    long = tuple(a[:50_000] for a in synth.lqr_course("sine", ds=59.0 / 50_000))   # not a multiple of the tile
    assert len(long[0]) == 50_000
    for course, sizes in ((demo, (1, 33, 4097, 65536)), (long, (33, 4097, 65536)), (LC.single_point_course(), (33,))):
        for n in sizes:
            state, ind, pe, pth_e = synth.lqr_track_inputs(n, course, seed=n)
            assert_same(gpu_control(engine, nx, state, course, ind, pe, pth_e),
                        OL.control(nx, state, course, ind, pe, pth_e), ALL)
    for course in (demo, LC.duplicate_course()[0], LC.single_point_course()):
        state, ind, pe, pth_e = LC.corner_states(course)
        got = gpu_control(engine, nx, state, course, ind, pe, pth_e)
        assert_same(got, OL.control(nx, state, course, ind, pe, pth_e), ALL)
    # BAD_INDEX: no winner and an incoming ind outside the course (4 states only; the 5-state ind starts at 0)
    state, ind, pe, pth_e = LC.corner_states(demo)
    ind[np.maximum(np.abs(state[0]), np.abs(state[1])) >= 1e20] = len(demo[0]) + 3
    ind[np.isnan(state[0])] = -1
    got = gpu_control(engine, nx, state, demo, ind, pe, pth_e)
    want = OL.control(nx, state, demo, ind, pe, pth_e)
    assert_same(got, want, ALL)
    if nx == 4:
        bad = want["status"] == OL.BAD_INDEX
        assert bad.sum() >= 9 and np.isnan(got["u"][:, bad]).all() and (got["ind"][bad] == ind[bad]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_control_with_non_default_params(engine, nx):
    course = synth.lqr_course("scurve")
    state, ind, pe, pth_e = synth.lqr_track_inputs(4097, course, seed=0xBEEF)
    for p in nondefault_params(nx):
        assert_same(gpu_control(engine, nx, state, course, ind, pe, pth_e, p),
                    OL.control(nx, state, course, ind, pe, pth_e, p), ALL)


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_launch_forms(engine, nx):
    """NULL optional outputs, n = 0, a batch split in two, and a graph-captured launch give the same bits."""
    import torch
    course = synth.lqr_course("demo")
    n = 5000
    state, ind, pe, pth_e = synth.lqr_track_inputs(n, course, seed=0xF0F0)
    want = OL.control(nx, state, course, ind, pe, pth_e)
    got = gpu_control(engine, nx, state, course, ind, pe, pth_e, with_k=False)
    assert_same(got, want)
    L = engine.lib
    prm = lqr_track_default_params(nx)
    dc = [_dev(a) for a in course]
    sp = dc[4].data_ptr() if nx == 5 else None
    nu = 1 if nx == 4 else 2
    assert L.crb_lqr_steering_control_batched(engine.ctx, 0, nx, None, dc[0].data_ptr(), dc[1].data_ptr(),
                                              dc[2].data_ptr(), dc[3].data_ptr(), sp, len(course[0]), C.byref(prm),
                                              None, None, None, None, None, None, None) == 0
    # split: two launches on column ranges of separate arrays
    h = 1777
    parts = []
    for a, b in ((0, h), (h, n)):
        parts.append(gpu_control(engine, nx, np.ascontiguousarray(state[:, a:b]), course, ind[a:b], pe[a:b],
                                 pth_e[a:b]))
    cat = {k: np.concatenate([pp[k] for pp in parts], axis=-1) for k in ALL}
    assert_same(cat, want, ALL)
    # graph capture: the launch only enqueues
    dst, dind, dpe, dpth = _dev(state), _dev(ind), _dev(pe), _dev(pth_e)
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
                eng.lqr_steering_control(nx, dst, dc[: 4 if nx == 4 else 5], dind, dpe, dpth, u=u, iters=it, status=stt)
            g.replay()
            torch.cuda.synchronize()
        finally:
            eng.close()
    got = dict(u=_host(u), ind=_host(dind), pe=_host(dpe), pth_e=_host(dpth), iters=_host(it), status=_host(stt))
    assert_same(got, want, ("u", "ind", "pe", "pth_e", "iters", "status"))


@pytest.mark.gpu
def test_gpu_update_is_the_checker(engine):
    import torch
    st, a, delta = LC.update_cases(20_000)
    for p in (None, nondefault_params(4)[1]):
        d = _dev(st)
        engine.lqr_update(d, _dev(a), _dev(delta), _eng_params(p) if p is not None else None)
        torch.cuda.synchronize()
        assert _bits_equal(_host(d), OL.update(st, a, delta, p))


def gpu_closed_loop(engine, nx, course, state0, ticks, check_every=1):
    """The test-driven loop on the device (control and update chained on the engine's stream, the 4-state rule's ai
    and ind step in torch on the same stream) against closed_loop_checker's history at every tick."""
    import torch
    n = state0.shape[1]
    hist = closed_loop_checker(nx, course, state0, ticks)
    dst = _dev(state0)
    dind = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    dpe = torch.zeros(n, dtype=torch.float32, device="cuda:0")
    dpth = torch.zeros(n, dtype=torch.float32, device="cuda:0")
    dc = [_dev(a) for a in course]
    nu = 1 if nx == 4 else 2
    u = torch.empty((nu, n), dtype=torch.float32, device="cuda:0")
    for tick in range(ticks):
        engine.lqr_steering_control(nx, dst, dc[: 4 if nx == 4 else 5], dind, dpe, dpth, u=u)
        if nx == 4:
            torch.cuda.synchronize()
            sp = dc[4][dind.clamp(0, len(course[0]) - 1).long()]
            ai = (KP * (sp - dst[3])).contiguous()
            di = u[0].contiguous()
        else:
            ai, di = u[0].contiguous(), u[1].contiguous()
        torch.cuda.synchronize()
        engine.lqr_update(dst, ai, di)
        torch.cuda.synchronize()
        if nx == 4:
            dind = torch.where(dst[3].abs() <= STOP_SPEED, dind + 1, dind).to(torch.int32).contiguous()
        if tick % check_every == 0 or tick == ticks - 1:
            hs, hu, hind = hist[tick]
            assert _bits_equal(_host(u), hu), tick
            assert _bits_equal(_host(dst), hs), tick
            assert np.array_equal(_host(dind), hind), tick


@pytest.mark.gpu
@pytest.mark.parametrize("nx", [4, 5])
def test_gpu_closed_loop_is_the_checker_at_every_tick(engine, nx):
    course, s0 = LC.demo_start(nx)
    rng = np.random.default_rng(0xC10)
    n = 4096
    j = rng.integers(0, len(course[0]), n)
    state0 = np.stack([course[0][j] + rng.uniform(-1, 1, n), course[1][j] + rng.uniform(-1, 1, n),
                       course[2][j] + rng.uniform(-0.5, 0.5, n), rng.uniform(0.0, 3.0, n)]).astype(np.float32)
    state0[:, 0] = s0
    gpu_closed_loop(engine, nx, course, np.ascontiguousarray(state0), 600)


FF_CU = r"""
// The feed-forward crb_atan2_1_to_float(L * (double)k) on the device for every k with bit pattern in [lo, hi), in
// chunks, checked against the host's (float)atan2(L * (double)k, 1.0) by crb_oracle_lqrt_ff_check (argv[3] =
// liboracle_lqrt.so).  Prints the number of mismatches.
#include <dlfcn.h>

#include "crb_common.cuh"
__global__ void ff_k(unsigned lo, unsigned long long count, double L, float* out) {
  for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x)
    out[k] = crb_atan2_1_to_float(L * (double)__uint_as_float(lo + (unsigned)k));
}
int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const unsigned lo = (unsigned)strtoul(argv[1], 0, 0), hi = (unsigned)strtoul(argv[2], 0, 0);
  void* so = dlopen(argv[3], RTLD_NOW);
  if (!so) return 2;
  typedef long long (*check_fn)(double, unsigned, unsigned, const float*);
  check_fn check = (check_fn)dlsym(so, "crb_oracle_lqrt_ff_check");
  const unsigned chunk = 1u << 27;
  float *d, *h;
  if (!check || cudaMalloc(&d, chunk * 4ull) != cudaSuccess || cudaMallocHost(&h, chunk * 4ull) != cudaSuccess) return 3;
  long long bad = 0;
  for (unsigned a = lo; a < hi; a = (hi - a > chunk) ? a + chunk : hi) {
    const unsigned b = (hi - a > chunk) ? a + chunk : hi;
    ff_k<<<2048, 256>>>(a, b - a, 0.5, d);
    if (cudaMemcpy(h, d, (b - a) * 4ull, cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
    bad += check(0.5, a, b, h);
  }
  printf("%lld\n", bad);
  return 0;
}
"""


@pytest.mark.gpu
def test_gpu_feed_forward_census(tmp_path):
    """(float)atan2(0.5 * (double)k, 1.0): the device equals the host's glibc on all 2^31 non-negative floats (every
    finite one, the infinity and the NaNs), and on two 2^24 slices of negative ones (odd symmetry)."""
    src = tmp_path / "ff.cu"
    src.write_text(FF_CU)
    exe = tmp_path / "ff"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                           "-I", os.path.join(ROOT, "cpprobotics_b200", "csrc"), str(src), "-o", str(exe), "-ldl"])
    for lo, hi in (("0x0", "0x80000000"), ("0x80000000", "0x81000000"), ("0xbf000000", "0xc0000000")):
        assert int(subprocess.check_output([str(exe), lo, hi, OL.LIB_PATH], text=True).strip()) == 0, (lo, hi)


@pytest.mark.gpu
def test_gpu_dlqr_still_matches_the_restatement(engine):
    """crb_lqr_dlqr_batched after its iteration moved to crb_lqr_dare.cuh: bitwise the restatement."""
    import torch
    for nx, nu in ((4, 1), (5, 2)):
        A, B, Q, R = synth.lqr_inputs(3000, nx, seed=31)
        want = O.dlqr_batched(A, B, Q, R, nx, nu)
        X = torch.empty((nx * nx, 3000), dtype=torch.float32, device="cuda:0")
        it = torch.empty(3000, dtype=torch.int32, device="cuda:0")
        K = engine.dlqr(_dev(A), _dev(B), _dev(Q), _dev(R), nx, nu, X=X, iters=it)
        torch.cuda.synchronize()
        assert _bits_equal(_host(K), want["K"]) and _bits_equal(_host(X), want["X"])
        assert np.array_equal(_host(it), want["iters"])
