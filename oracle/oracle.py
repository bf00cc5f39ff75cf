"""ctypes wrapper of oracle/lib/liboracle.so — the CPU restatement of the reference hot paths.

TEST INFRASTRUCTURE ONLY.  May be imported by tests/, by __graft_entry__.smoke() and by bench.py's
cpu_baseline / --impl reference legs, never by the product package (cpprobotics_b200/).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from ._load import LIB_DIR, checker

LIB_PATH = os.path.join(LIB_DIR, "liboracle.so")

ORDER_SEQ = 0
ORDER_PAIRWISE = 1

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


class MpcParams(C.Structure):
    """Field-for-field the same as crb_mpc_params (include/crb.h)."""
    _fields_ = [("dt", C.c_float), ("wb", C.c_float), ("max_steer", C.c_float),
                ("max_accel", C.c_float), ("max_speed", C.c_float), ("min_speed", C.c_float),
                ("w_a", C.c_float), ("w_delta", C.c_float), ("w_da", C.c_float),
                ("w_ddelta", C.c_float), ("w_x", C.c_float), ("w_y", C.c_float),
                ("w_yaw", C.c_float), ("w_v", C.c_float), ("max_iter", C.c_int),
                ("du_th", C.c_float), ("max_ls", C.c_int), ("j_tol", C.c_float)]


PROTOTYPES = {
    "crb_oracle_num_threads": (C.c_int, []),
    "crb_oracle_motion_model": (None, [f32p, f32p, C.c_double, f32p]),
    "crb_oracle_jacobF": (None, [f32p, f32p, C.c_double, f32p]),
    "crb_oracle_ekf_estimation": (None, [f32p, f32p, f32p, f32p, f32p, f32p, C.c_double, C.c_int]),
    "crb_oracle_ekf_estimation_f64": (None, [f64p, f64p, f64p, f64p, f64p, f64p, C.c_double]),
    "crb_oracle_ekf_step_batched": (None, [C.c_int64, f32p, f32p, f32p, f32p, f32p, f32p, C.c_double, C.c_int,
                                           C.c_int, C.c_int]),
    "crb_oracle_gauss_likelihood": (C.c_float, [C.c_float, C.c_float, C.c_double]),
    "crb_oracle_pf_particle": (None, [f32p, f32p, f64p, f32p, f32p, f32p, C.c_int, C.c_float, C.c_double,
                                      C.c_double]),
    "crb_oracle_philox_normal2": (None, [C.c_uint64, C.c_uint64, f32p]),
    "crb_oracle_philox_uniform12": (C.c_double, [C.c_uint64, C.c_uint64]),
    "crb_oracle_pf_predict_weight_batched": (None, [C.c_int64, f32p, f32p, C.c_void_p, C.c_uint64, f32p, C.c_int,
                                                    f32p, f32p, C.c_float, C.c_double, C.c_double, C.c_int]),
    "crb_oracle_pf_estimate": (None, [C.c_int64, f32p, f32p, f32p, f32p, C.POINTER(C.c_double)]),
    "crb_oracle_pf_resample": (C.c_int, [C.c_int64, f32p, f32p, f64p, C.c_float, C.c_int, C.POINTER(C.c_float)]),
    "crb_oracle_dlqr_batched": (None, [C.c_int64, C.c_int, C.c_int, f32p, f32p, f32p, f32p, C.c_int, C.c_float,
                                       f32p, f32p, i32p, C.c_int]),
    "crb_oracle_sincosf": (None, [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "crb_oracle_mpc_solve_batched": (None, [C.c_int64, C.c_int, f32p, f32p, C.c_void_p, C.POINTER(MpcParams),
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "crb_oracle_plant_update": (None, [f32p, C.c_float, C.c_float]),
    "crb_oracle_plant_update_k": (None, [f32p, C.c_float, C.c_float, f64p]),
    "crb_oracle_calc_nearest_index": (C.c_int, [f32p, f32p, f32p, C.c_int, C.c_int]),
    "crb_oracle_calc_ref_trajectory": (None, [f32p, f32p, f32p, f32p, f32p, C.c_int, C.c_float, C.c_int,
                                              C.POINTER(C.c_int), f32p]),
    "crb_oracle_calc_ref_trajectory_dt": (None, [f32p, f32p, f32p, f32p, f32p, C.c_int, C.c_float, C.c_int,
                                                 C.POINTER(C.c_int), f32p, C.c_double]),
}


def use_library(which: str = "faithful") -> bool:
    """Selects the build the wrappers below call: "faithful" = liboracle.so (-O2 -ffp-contract=off, the
    parity oracle), "fast" = liboracle_fast.so (same sources, -O3 -march=x86-64-v3 -ffp-contract=fast:
    BASELINE.md's B2 "what the host can do" timing arm; NOT a parity reference), "O0" = liboracle_O0.so
    (BASELINE.md B0 "as shipped", the reference's CMakeLists.txt:5: a timing arm only).  Returns False (and
    selects the faithful build) when the build asked for is missing or, for "fast", the CPU lacks AVX2/FMA."""
    global LIB_PATH
    want = os.path.join(LIB_DIR, "liboracle.so")
    ok = True
    if which == "fast":
        flags = ""
        try:
            flags = open("/proc/cpuinfo").read()
        except OSError:
            pass
        fast = os.path.join(LIB_DIR, "liboracle_fast.so")
        if os.path.exists(fast) and " avx2" in flags and " fma" in flags:
            want = fast
        else:
            ok = False
    if which == "O0":
        p0 = os.path.join(LIB_DIR, "liboracle_O0.so")
        if os.path.exists(p0):
            want = p0
        else:
            ok = False
    LIB_PATH = want
    return ok


def lib() -> C.CDLL:
    return checker(LIB_PATH, PROTOTYPES)


def num_threads() -> int:
    return int(lib().crb_oracle_num_threads())


# ---- reference constants (the values main() of each reference program sets) ---------------------------
def ekf_constants():
    """DT :17, Q :142-146, R :149-151 of src/extended_kalman_filter.cpp (column-major, float32)."""
    Q = np.zeros(16, np.float32)
    Q[0] = np.float32(0.1 * 0.1)
    Q[5] = np.float32(0.1 * 0.1)
    Q[10] = np.float32((1.0 / 180 * np.pi) * (1.0 / 180 * np.pi))
    Q[15] = np.float32(0.1 * 0.1)
    R = np.array([1, 0, 0, 1], np.float32)
    return 0.1, Q, R


def pf_constants():
    """DT :18, PI :19, Q :217, Rsim :228-230, u :183 of src/particle_filter.cpp."""
    return dict(dt=0.1, pi=3.141592653, Q=np.float32(0.1 * 0.1),
                rsim_diag=np.array([1.0, (30.0 / 180 * np.pi) ** 2], np.float32),
                u=np.array([1.0, 0.1], np.float32))


# ---- EKF -------------------------------------------------------------------------------------------------
def ekf_estimation(xEst, PEst, z, u, Q=None, R=None, dt=None, order=ORDER_SEQ):
    """Single agent, in place on copies; P, Q are flat column-major 16-vectors.  Returns (x, P)."""
    d, Qd, Rd = ekf_constants()
    x = np.ascontiguousarray(xEst, np.float32).copy()
    P = np.ascontiguousarray(PEst, np.float32).copy()
    lib().crb_oracle_ekf_estimation(x, P, np.ascontiguousarray(z, np.float32),
                                    np.ascontiguousarray(u, np.float32),
                                    Qd if Q is None else np.ascontiguousarray(Q, np.float32),
                                    Rd if R is None else np.ascontiguousarray(R, np.float32),
                                    d if dt is None else dt, order)
    return x, P


def ekf_estimation_f64(xEst, PEst, z, u, Q=None, R=None, dt=None):
    d, Qd, Rd = ekf_constants()
    x = np.ascontiguousarray(xEst, np.float64).copy()
    P = np.ascontiguousarray(PEst, np.float64).copy()
    lib().crb_oracle_ekf_estimation_f64(
        x, P, np.ascontiguousarray(z, np.float64), np.ascontiguousarray(u, np.float64),
        np.ascontiguousarray(Qd if Q is None else Q, np.float64),
        np.ascontiguousarray(Rd if R is None else R, np.float64), d if dt is None else dt)
    return x, P


def ekf_step_batched(x, P, z, u, Q=None, R=None, dt=None, n_steps=1, order=ORDER_SEQ, nthreads=0,
                     inplace=False):
    """SoA batch with the libcrb layout; returns new (x, P) (copies unless inplace)."""
    d, Qd, Rd = ekf_constants()
    if not inplace:
        x = np.ascontiguousarray(x, np.float32).copy()
        P = np.ascontiguousarray(P, np.float32).copy()
    n = x.shape[1]
    lib().crb_oracle_ekf_step_batched(n, x, P, np.ascontiguousarray(z, np.float32),
                                      np.ascontiguousarray(u, np.float32),
                                      Qd if Q is None else np.ascontiguousarray(Q, np.float32),
                                      Rd if R is None else np.ascontiguousarray(R, np.float32),
                                      d if dt is None else dt, n_steps, order, nthreads)
    return x, P


# ---- PF --------------------------------------------------------------------------------------------------
def gauss_likelihood(x, sigma, pi=3.141592653):
    return float(lib().crb_oracle_gauss_likelihood(float(x), float(sigma), pi))


def philox_normal2(seed, index):
    g = np.zeros(2, np.float32)
    lib().crb_oracle_philox_normal2(int(seed), int(index), g)
    return g


def pf_predict_weight_batched(px, pw, noise, landmarks, seed=0, consts=None, nthreads=0,
                              inplace=False):
    c = consts or pf_constants()
    if not inplace:
        px = np.ascontiguousarray(px, np.float32).copy()
        pw = np.ascontiguousarray(pw, np.float32).copy()
    lm = np.ascontiguousarray(np.asarray(landmarks, np.float32).reshape(-1, 3))
    nptr = None
    if noise is not None:
        noise = np.ascontiguousarray(noise, np.float32)
        nptr = noise.ctypes.data
    lib().crb_oracle_pf_predict_weight_batched(
        px.shape[1], px, pw, nptr, int(seed), lm, lm.shape[0],
        np.ascontiguousarray(c["u"], np.float32), np.ascontiguousarray(c["rsim_diag"], np.float32),
        float(c["Q"]), c["dt"], c["pi"], nthreads)
    return px, pw


def pf_resample(px, pw, uniforms, nth=None, reference_mode=False):
    """resampling() :120-148.  uniforms [n] in [1,2).  Returns (px, pw, did_resample, neff)."""
    L = lib()
    px = np.ascontiguousarray(px, np.float32).copy()
    pw = np.ascontiguousarray(pw, np.float32).copy()
    n = px.shape[1]
    neff = C.c_float(0.0)
    did = L.crb_oracle_pf_resample(n, px, pw, np.ascontiguousarray(uniforms, np.float64),
                                   float(n // 2 if nth is None else nth), int(reference_mode), C.byref(neff))
    return px, pw, bool(did), neff.value


def philox_uniform12(seed, index):
    return lib().crb_oracle_philox_uniform12(int(seed), int(index))


def dlqr_batched(A, B, Q, R, nx, nu, maxiter=150, eps=0.01, nthreads=0):
    """A [nx*nx, n], B [nx*nu, n] column-major per agent; Q [nx*nx], R [nu*nu] shared.
    Returns dict(K [nu*nx, n], X [nx*nx, n], iters [n])."""
    L = lib()
    A = np.ascontiguousarray(A, np.float32); B = np.ascontiguousarray(B, np.float32)
    n = A.shape[1]
    K = np.zeros((nu * nx, n), np.float32); X = np.zeros((nx * nx, n), np.float32); it = np.zeros(n, np.int32)
    L.crb_oracle_dlqr_batched(n, nx, nu, A, B, np.ascontiguousarray(Q, np.float32).reshape(-1),
                              np.ascontiguousarray(R, np.float32).reshape(-1), maxiter, eps, K, X, it, nthreads)
    return dict(K=K, X=X, iters=it)


def pf_estimate(px, pw):
    px = np.ascontiguousarray(px, np.float32)
    pw = np.ascontiguousarray(pw, np.float32).copy()
    xe = np.zeros(4, np.float32)
    pe = np.zeros(16, np.float32)
    sw = C.c_double(0.0)
    lib().crb_oracle_pf_estimate(px.shape[1], px, pw, xe, pe, C.byref(sw))
    return pw, xe, pe.reshape(4, 4).T.copy(), sw.value


# ---- MPC -------------------------------------------------------------------------------------------------
def mpc_params(**over) -> MpcParams:
    """Reference constants (src/model_predictive_control.cpp:26-39, :202-210, :247-250, :326)."""
    d = dict(dt=0.2, wb=2.5, max_steer=np.float32(45.0 / 180 * np.pi), max_accel=1.0,
             max_speed=np.float32(55.0 / 3.6), min_speed=np.float32(-20.0 / 3.6), w_a=0.01,
             w_delta=0.01, w_da=0.01, w_ddelta=1.0, w_x=1.0, w_y=1.0, w_yaw=0.5, w_v=0.5,
             max_iter=50, du_th=1e-4, max_ls=4, j_tol=1e-6)
    d.update(over)
    p = MpcParams()
    for k, v in d.items():
        setattr(p, k, v)
    return p


def _mpc_lib():
    return lib()


def sincosf(x):
    s, c = C.c_float(), C.c_float()
    _mpc_lib().crb_oracle_sincosf(float(x), C.byref(s), C.byref(c))
    return s.value, c.value


def mpc_solve_batched(x0, xref, T, params=None, u_init=None, nthreads=0):
    """libcrb layout: x0 [4,n], xref [4T,n] (field 4t+k), u_init [2(T-1),n] or None.
    Returns dict(sol [4T+2(T-1),n], u0 [2,n]=(a0,delta0), cost [n], status [n], iters [n])."""
    p = params or mpc_params()
    x0 = np.ascontiguousarray(x0, np.float32)
    xref = np.ascontiguousarray(xref, np.float32)
    n = x0.shape[1]
    sol = np.zeros((4 * T + 2 * (T - 1), n), np.float32)
    u0 = np.zeros((2, n), np.float32)
    cost = np.zeros(n, np.float32)
    status = np.zeros(n, np.int32)
    iters = np.zeros(n, np.int32)
    ui = None
    if u_init is not None:
        u_init = np.ascontiguousarray(u_init, np.float32)
        ui = u_init.ctypes.data
    _mpc_lib().crb_oracle_mpc_solve_batched(n, T, x0, xref, ui, C.byref(p), sol.ctypes.data,
                                            u0.ctypes.data, cost.ctypes.data, status.ctypes.data,
                                            iters.ctypes.data, nthreads)
    return dict(sol=sol, u0=u0, cost=cost, status=status, iters=iters)


# update()'s double macros (src/model_predictive_control.cpp:26-38) in crb_mpc_params' field names
PLANT_MACROS = dict(max_steer=45.0 / 180 * np.pi, dt=0.2, wb=2.5, max_speed=55.0 / 3.6, min_speed=-20.0 / 3.6)


def plant_constant(params, name):
    """libcrb's promotion rule (include/crb.h): a float parameter equal to the reference's macro rounded to
    float stands for the macro's double value; any other value is promoted from float."""
    v = np.float32(getattr(params, name))
    ref = PLANT_MACROS[name]
    return ref if v == np.float32(ref) else float(v)


def plant_update(state, a, delta, params=None):
    """update() :69-81 on one state [4]; params (MpcParams) gives max_steer, dt, wb, max_speed and min_speed,
    None = the reference's macros."""
    st = np.ascontiguousarray(state, np.float32).copy()
    if params is None:
        _mpc_lib().crb_oracle_plant_update(st, float(a), float(delta))
    else:
        k = np.array([plant_constant(params, f) for f in ("max_steer", "dt", "wb", "max_speed", "min_speed")])
        _mpc_lib().crb_oracle_plant_update_k(st, float(a), float(delta), k)
    return st


def calc_nearest_index(state, cx, cy, pind):
    return int(_mpc_lib().crb_oracle_calc_nearest_index(
        np.ascontiguousarray(state, np.float32), np.ascontiguousarray(cx, np.float32),
        np.ascontiguousarray(cy, np.float32), len(cx), int(pind)))


def calc_ref_trajectory(state, cx, cy, cyaw, sp, dl, T, target_ind, params=None):
    """Returns (xref [T,4], new target_ind).  params (MpcParams) gives dt, None = the reference's DT."""
    ti = C.c_int(int(target_ind))
    xref = np.zeros((T, 4), np.float32)
    args = (np.ascontiguousarray(state, np.float32), np.ascontiguousarray(cx, np.float32),
            np.ascontiguousarray(cy, np.float32), np.ascontiguousarray(cyaw, np.float32),
            np.ascontiguousarray(sp, np.float32), len(cx), float(dl), int(T), C.byref(ti), xref)
    if params is None:
        _mpc_lib().crb_oracle_calc_ref_trajectory(*args)
    else:
        _mpc_lib().crb_oracle_calc_ref_trajectory_dt(*args, plant_constant(params, "dt"))
    return xref, ti.value
