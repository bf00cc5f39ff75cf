"""ctypes wrapper of oracle/lib/liboracle_mptg.so — the CPU restatement of include/trajectory_optimizer.h
(optimizer_traj) and include/motion_model.h (MotionModel, glibc's tanf).  Built by `make -C oracle -f mptg.mk`
(python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liboracle_mptg.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_lib = None

# include/crb.h
CONVERGED, MAX_ITER_REACHED, EMPTY_TRAJ, STEP_CAP, OUT_OF_RANGE = 0, 1, 2, 3, 4
MAX_ITER, MAX_STEPS = 1000, 16384
# crb_oracle_mptg.h: bits of the quirks output
Q_CONVERGED_AT_0, Q_LS_TIE, Q_LS_NAN, Q_SINGULAR_J, Q_STEPS_OFF_CEIL, Q_STEER_BEYOND_PIO4 = 1, 2, 4, 8, 16, 32


class MptgParams(C.Structure):
    """Field-for-field the same as crb_mptg_params (include/crb.h)."""
    _fields_ = [("base_l", C.c_float), ("ds", C.c_float), ("max_iter", C.c_int32), ("cost_th", C.c_float),
                ("h_step", C.c_float * 3)]


def mptg_params(**over) -> MptgParams:
    """The demo's values (src/model_predictive_trajectory_generator.cpp:19-33), narrowed to float."""
    d = dict(base_l=1.0, ds=0.1, max_iter=100, cost_th=0.1, h_step=(0.2, 0.005, 0.005))
    d.update(over)
    p = MptgParams()
    p.base_l, p.ds, p.cost_th = (float(np.float32(d[k])) for k in ("base_l", "ds", "cost_th"))
    p.max_iter = int(d["max_iter"])
    for k in range(3):
        p.h_step[k] = float(np.float32(d["h_step"][k]))
    return p


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run `make -C oracle -f mptg.mk` (or python __graft_entry__.py)")
        L = C.CDLL(LIB_PATH)
        L.crb_oracle_num_threads.restype = C.c_int
        L.crb_oracle_libm_tanf.restype = C.c_float
        L.crb_oracle_libm_tanf.argtypes = [C.c_float]
        L.crb_oracle_libm_tanf_census.restype = C.c_int64
        L.crb_oracle_libm_tanf_census.argtypes = [C.c_uint32, C.c_uint32]
        L.crb_oracle_mptg_optimize.argtypes = [C.c_int64, f32p, f32p, f32p, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.crb_oracle_mptg_generate.argtypes = [C.c_int64, f32p, f32p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_int]
        _lib = L
    return _lib


def num_threads() -> int:
    return int(lib().crb_oracle_num_threads())


def libm_tanf(x) -> float:
    return float(lib().crb_oracle_libm_tanf(float(x)))


def libm_tanf_census(lo_bits: int, hi_bits: int) -> int:
    """Number of bit patterns in [lo_bits, hi_bits), both signs, where the restatement differs from the host tanf."""
    return int(lib().crb_oracle_libm_tanf_census(int(lo_bits), int(hi_bits)))


def _ptr(a):
    return None if a is None else a.ctypes.data


def optimize(state, target, param, params=None, max_pts=0, traj_fill=np.nan, nthreads=0):
    """optimizer_traj :53-128 in the libcrb layout.  state [4,n], target [3,n], param [4,n] (copied).  Returns dict
    (param, traj [3*max_pts,n] pre-filled with traj_fill, traj_len, cost, status, iters, quirks)."""
    p = params or mptg_params()
    st = np.ascontiguousarray(state, np.float32)
    n = st.shape[1]
    q = np.ascontiguousarray(param, np.float32).copy()
    traj = np.full((3 * max_pts, n), traj_fill, np.float32)
    out = {k: np.zeros(n, np.int32) for k in ("traj_len", "status", "iters", "quirks")}
    cost = np.zeros(n, np.float32)
    lib().crb_oracle_mptg_optimize(n, st, np.ascontiguousarray(target, np.float32), q, C.byref(p), int(max_pts),
                                   _ptr(traj), _ptr(out["traj_len"]), _ptr(cost), _ptr(out["status"]),
                                   _ptr(out["iters"]), _ptr(out["quirks"]), nthreads)
    return dict(param=q, traj=traj, cost=cost, **out)


def generate(state, param, params=None, max_pts=0, traj_fill=np.nan, nthreads=0):
    """generate_trajectory / generate_last_state :110-150.  Returns dict(traj, traj_len, last [3,n], status)."""
    p = params or mptg_params()
    st = np.ascontiguousarray(state, np.float32)
    n = st.shape[1]
    traj = np.full((3 * max_pts, n), traj_fill, np.float32)
    tl, status = np.zeros(n, np.int32), np.zeros(n, np.int32)
    last = np.zeros((3, n), np.float32)
    lib().crb_oracle_mptg_generate(n, st, np.ascontiguousarray(param, np.float32), C.byref(p), int(max_pts),
                                   _ptr(traj), _ptr(tl), _ptr(last), _ptr(status), nthreads)
    return dict(traj=traj, traj_len=tl, last=last, status=status)
