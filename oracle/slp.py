"""ctypes wrapper of oracle/lib/liboracle_slp.so — the CPU restatement of src/state_lattice_planner.cpp's samplers
(sample_states, calc_uniform_polar_states, calc_biased_polar_states, calc_lane_states) and its lookup-table search.
generate_path is that search followed by the optimizer of liboracle_mptg.so (oracle/mptg.py).  Built by
`make -C oracle` (python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from ._load import LIB_DIR, checker

from . import mptg as OM

LIB_PATH = os.path.join(LIB_DIR, "liboracle_slp.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")

# include/crb.h
UNIFORM, BIASED, LANE = 0, 1, 2
OK, OUT_OF_RANGE = 0, 1
MAX_NXY, MAX_NH, MAX_NS, MAX_STATES = 4096, 1024, 1 << 20, 65536
N_FIELDS = {UNIFORM: 4, BIASED: 5, LANE: 5}


class Sampler(C.Structure):
    """Field-for-field the same as crb_slp_sampler (include/crb.h)."""
    _fields_ = [("kind", C.c_int32), ("nxy", C.c_int32), ("nh", C.c_int32), ("ns", C.c_int32), ("d", C.c_int32)]


def sampler(kind, nxy, nh=1, ns=0, d=0) -> Sampler:
    return Sampler(int(kind), int(nxy), int(nh), int(ns), int(d))


def states_per_query(s: Sampler) -> int:
    """S of crb.h (the sampler must be within the limits)."""
    if s.kind == UNIFORM:
        return s.nxy * s.nh
    if s.kind == BIASED:
        return max(s.nxy - 1, 0) * s.nh
    return s.nxy


def slp_params():
    """generate_path's optimizer settings (:22-24, :146-148), narrowed to float, and CONST_V."""
    return OM.mptg_params(base_l=1.0, ds=0.1, max_iter=100, cost_th=0.1, h_step=(0.5, 0.02, 0.02)), float(np.float32(3.0))


PROTOTYPES = {
    "crb_oracle_slp_sample": (None, [C.c_int64, C.POINTER(Sampler), C.c_int, f32p, f32p, i32p, C.c_void_p, C.c_int]),
    "crb_oracle_slp_search": (None, [C.c_int64, f32p, f32p, C.c_int, C.c_void_p, f32p, C.c_void_p, C.c_int]),
}


def lib() -> C.CDLL:
    return checker(LIB_PATH, PROTOTYPES)


def sample(s: Sampler, qp, nthreads=0):
    """The samplers in the libcrb layout: qp [F, n_q].  Returns dict(target [3, n_q*S], n_states, status)."""
    q = np.ascontiguousarray(qp, np.float32)
    n = q.shape[1]
    S = states_per_query(s)
    target = np.empty((3, n * S), np.float32)
    ns, st = np.zeros(n, np.int32), np.zeros(n, np.int32)
    lib().crb_oracle_slp_sample(n, C.byref(s), S, q, target, ns, st.ctypes.data, nthreads)
    return dict(target=target, n_states=ns, status=st)


def search(target, table, k0=None, nthreads=0):
    """search_nearest_one_from_lookuptable: target [3, n], table [rows, 6].  Returns dict(param [4, n], row)."""
    t = np.ascontiguousarray(target, np.float32)
    tb = np.ascontiguousarray(table, np.float32)
    n = t.shape[1]
    k = None if k0 is None else np.ascontiguousarray(k0, np.float32)
    param = np.empty((4, n), np.float32)
    row = np.zeros(n, np.int32)
    lib().crb_oracle_slp_search(n, t, tb, tb.shape[0], None if k is None else k.ctypes.data, param, row.ctypes.data,
                                nthreads)
    return dict(param=param, row=row)


def generate_path(target, table, k0=None, max_pts=0, traj_fill=np.nan, params=None, v=None, nthreads=0):
    """generate_path :137-155: search, start (0, 0, 0, v), optimizer_traj.  Returns the optimizer's dict (param after
    optimisation, traj, traj_len, cost, status, iters, quirks) with the search's row."""
    p0, v0 = slp_params()
    sr = search(target, table, k0, nthreads)
    n = sr["param"].shape[1]
    st = np.zeros((4, n), np.float32)
    st[3] = np.float32(v0 if v is None else v)
    o = OM.optimize(st, target, sr["param"], params or p0, max_pts=max_pts, traj_fill=traj_fill, nthreads=nthreads)
    o["row"] = sr["row"]
    return o
