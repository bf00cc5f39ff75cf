"""ctypes wrapper of oracle/lib/liboracle_lqrt.so — the CPU restatement of calc_nearest_index, lqr_steering_control and
update of src/lqr_steer_control.cpp (nx 4) and src/lqr_speed_steer_control.cpp (nx 5).  Built by
`make -C oracle -f lqrt.mk` (python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liboracle_lqrt.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_lib = None

# include/crb.h
OK, DARE_MAXITER, BAD_INDEX = 0, 1, 2


class Params(C.Structure):  # include/crb.h crb_lqr_track_params
    _fields_ = [("dt", C.c_double), ("wheelbase", C.c_double), ("max_steer", C.c_double), ("Q", C.c_float * 25),
                ("R", C.c_float * 4), ("maxiter", C.c_int32), ("eps", C.c_float)]


def default_params(nx: int) -> Params:
    """The reference's constants (src/lqr_steer_control.cpp:20-23, :77-78, :114-115 and the 5-state program's)."""
    p = Params()
    p.dt, p.wheelbase, p.max_steer = 0.1, 0.5, 45.0 / 180 * np.pi
    for f in range(25):
        p.Q[f] = 1.0 if f % 6 == 0 else 0.0
    p.R[0] = 1.0
    p.R[3] = 1.0 if nx == 5 else 0.0
    p.maxiter, p.eps = 150, float(np.float32(0.01))
    return p


def params_from(prm) -> Params:
    """A Params with the fields of any structure of the same layout (cpprobotics_b200.LqrTrackParams)."""
    p = Params()
    C.memmove(C.byref(p), C.byref(prm), C.sizeof(Params))
    return p


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run `make -C oracle -f lqrt.mk` (or python __graft_entry__.py)")
        L = C.CDLL(LIB_PATH)
        L.crb_oracle_lqrt_nearest.restype = C.c_float
        L.crb_oracle_lqrt_nearest.argtypes = [f32p, f32p, f32p, f32p, C.c_int32, C.POINTER(C.c_int32)]
        L.crb_oracle_lqrt_control_batched.restype = None
        L.crb_oracle_lqrt_control_batched.argtypes = [C.c_int64, C.c_int, f32p, f32p, f32p, f32p, f32p, C.c_void_p,
                                                      C.c_int32, C.POINTER(Params), i32p, f32p, f32p, f32p, C.c_void_p,
                                                      i32p, i32p, C.c_int]
        L.crb_oracle_lqrt_update_batched.restype = None
        L.crb_oracle_lqrt_update_batched.argtypes = [C.c_int64, f32p, f32p, f32p, C.POINTER(Params), C.c_int]
        L.crb_oracle_lqrt_ff_check.restype = C.c_int64
        L.crb_oracle_lqrt_ff_check.argtypes = [C.c_double, C.c_uint32, C.c_uint32, f32p]
        _lib = L
    return _lib


def num_threads() -> int:
    return len(os.sched_getaffinity(0))


def _f(a):
    return np.ascontiguousarray(a, np.float32)


def nearest(st, course, ind: int = 0):
    """calc_nearest_index for one state (x, y, yaw, v): (signed squared distance, ind)."""
    cx, cy, cyaw = (_f(a) for a in course[:3])
    i = C.c_int32(ind)
    e = lib().crb_oracle_lqrt_nearest(_f(st), cx, cy, cyaw, cx.size, C.byref(i))
    return float(np.float32(e)), int(i.value)


def control(nx: int, state, course, ind, pe, pth_e, params: Params | None = None, nthreads: int = 0):
    """crb_lqr_steering_control_batched on the host.  state [4, n]; course (cx, cy, cyaw, ck[, sp]); ind, pe, pth_e
    [n] (copied, not modified).  Returns dict(u [nu, n], ind, pe, pth_e, K [nu*nx, n], iters, status)."""
    st = _f(state)
    n = st.shape[1]
    nu = 1 if nx == 4 else 2
    cx, cy, cyaw, ck = (_f(a) for a in course[:4])
    sp = _f(course[4]) if nx == 5 else None
    p = params if params is not None else default_params(nx)
    ind = np.array(ind, np.int32).reshape(n)
    pe = np.array(pe, np.float32).reshape(n)
    pth_e = np.array(pth_e, np.float32).reshape(n)
    u = np.zeros((nu, n), np.float32)
    K = np.zeros((nu * nx, n), np.float32)
    it, stt = np.zeros(n, np.int32), np.zeros(n, np.int32)
    lib().crb_oracle_lqrt_control_batched(n, nx, st, cx, cy, cyaw, ck, sp.ctypes.data if sp is not None else None,
                                          cx.size, C.byref(p), ind, pe, pth_e, u, K.ctypes.data, it, stt, int(nthreads))
    return dict(u=u, ind=ind, pe=pe, pth_e=pth_e, K=K, iters=it, status=stt)


def update(state, a, delta, params: Params | None = None, nthreads: int = 0):
    """crb_lqr_update_batched on the host; returns the new state [4, n]."""
    st = np.array(state, np.float32)
    n = st.shape[1]
    p = params if params is not None else default_params(4)
    lib().crb_oracle_lqrt_update_batched(n, st, _f(a).reshape(n), _f(delta).reshape(n), C.byref(p), int(nthreads))
    return st


def ff_check(lo_bits: int, hi_bits: int, got, L: float = 0.5) -> int:
    """Bit patterns k in [lo_bits, hi_bits) where got differs from (float)atan2(L * (double)k, 1.0) of the host."""
    return int(lib().crb_oracle_lqrt_ff_check(float(L), lo_bits, hi_bits, _f(got)))
