"""ctypes wrapper of oracle/lib/liboracle_rrt.so — the CPU restatement of RRT::planning (include/rrt.h) with
std::mt19937, its two distributions and glibc's atan2f written out.  Built by `make -C oracle -f rrt.mk`
(python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liboracle_rrt.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_lib = None

# include/crb.h
FOUND, MAX_ITER, BAD_INPUT = 0, 1, 2
MAX_ITER_LIMIT = 16384


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run `make -C oracle -f rrt.mk` (or python __graft_entry__.py)")
        L = C.CDLL(LIB_PATH)
        L.crb_oracle_rrt_mt_run.restype = None
        L.crb_oracle_rrt_mt_run.argtypes = [C.c_uint32, C.c_int64, u32p]
        L.crb_oracle_rrt_dist_run.restype = C.c_int64
        L.crb_oracle_rrt_dist_run.argtypes = [C.c_int, C.c_float, C.c_float, C.c_int64, u32p, u32p, i32p]
        L.crb_oracle_rrt_atanf.restype = C.c_float
        L.crb_oracle_rrt_atanf.argtypes = [C.c_float]
        L.crb_oracle_rrt_atan2f.restype = C.c_float
        L.crb_oracle_rrt_atan2f.argtypes = [C.c_float, C.c_float]
        L.crb_oracle_rrt_atanf_census.restype = C.c_int64
        L.crb_oracle_rrt_atanf_census.argtypes = [C.c_uint32, C.c_uint32]
        L.crb_oracle_rrt_atan2f_pairs.restype = C.c_int64
        L.crb_oracle_rrt_atan2f_pairs.argtypes = [C.c_int64, f32p, f32p]
        L.crb_oracle_rrt_plan.restype = None
        L.crb_oracle_rrt_plan.argtypes = [C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int32, f32p, C.c_int32,
                                          C.c_int64, f32p, u32p, C.c_int32, C.c_void_p, i32p, C.c_int32, C.c_void_p,
                                          C.c_void_p, i32p, i32p, i32p, i64p, i32p, C.c_int]
        _lib = L
    return _lib


def num_threads() -> int:
    return len(os.sched_getaffinity(0))


def mt_run(seed: int, n: int) -> np.ndarray:
    """The first n outputs of std::mt19937(seed)."""
    out = np.zeros(n, np.uint32)
    lib().crb_oracle_rrt_mt_run(seed, n, out)
    return out


def dist_run(kind: int, u, a: float = 0.0, b: float = 1.0):
    """The distributions on a fixed list of generator outputs: kind 0 uniform_int_distribution<int>(0, 100), kind 1
    uniform_real_distribution<float>(a, b).  Returns (results uint32 (float bits for kind 1), values used per draw)."""
    v = np.ascontiguousarray(u, np.uint32)
    out, used = np.zeros(v.size, np.uint32), np.zeros(v.size, np.int32)
    k = lib().crb_oracle_rrt_dist_run(kind, a, b, v.size, v, out, used)
    return out[:k], used[:k]


def atan2f(y, x) -> float:
    return float(lib().crb_oracle_rrt_atan2f(float(y), float(x)))


def atanf_census(lo_bits: int, hi_bits: int) -> int:
    """Bit patterns in [lo_bits, hi_bits) where the restated atanf differs from the host atanf."""
    return int(lib().crb_oracle_rrt_atanf_census(lo_bits, hi_bits))


def atan2f_pairs(y, x) -> int:
    """Pairs where the restated atan2f differs from the host atan2f."""
    y, x = np.ascontiguousarray(y, np.float32), np.ascontiguousarray(x, np.float32)
    return int(lib().crb_oracle_rrt_atan2f_pairs(y.size, y, x))


def plan(prm, ob, se, seed, max_pts=0, max_nodes=0, fill=np.nan, nthreads=0):
    """crb_rrt_plan_batched on the host.  prm: dict(rand_min, rand_max, expand_dis, goal_sample_rate, max_iter); ob
    [n_ob, 3] (x, y, r); se [4, n] (sx, sy, gx, gy); seed [n] uint32.  Returns dict(path [2*max_pts, n], path_len, tree
    [2*max_nodes, n], parent [max_nodes, n], n_nodes, n_iter, status, draws, branches (bit 0 a uniform_int redraw, bit 1
    a canonical 1.0 mapped below 1)), crb_rrt_plan_batched's layout; path and
    tree are `fill` (parent -1) past what is written."""
    o = np.ascontiguousarray(ob, np.float32).reshape(-1, 3)
    s = np.ascontiguousarray(se, np.float32)
    sd = np.ascontiguousarray(seed, np.uint32)
    n = s.shape[1]
    path = np.full((2 * max_pts, n), fill, np.float32)
    tree = np.full((2 * max_nodes, n), fill, np.float32)
    parent = np.full((max_nodes, n), -1, np.int32)
    pl, nn, it, st = (np.zeros(n, np.int32) for _ in range(4))
    draws = np.zeros(n, np.int64)
    br = np.zeros(n, np.int32)
    lib().crb_oracle_rrt_plan(prm["rand_min"], prm["rand_max"], prm["expand_dis"], int(prm["goal_sample_rate"]),
                              int(prm["max_iter"]), o.reshape(-1) if o.size else np.zeros(1, np.float32), o.shape[0], n,
                              s, sd, int(max_pts), path.ctypes.data if max_pts > 0 else None, pl, int(max_nodes),
                              tree.ctypes.data if max_nodes > 0 else None, parent.ctypes.data if max_nodes > 0 else None,
                              nn, it, st, draws, br, int(nthreads))
    return dict(path=path, path_len=pl, tree=tree, parent=parent, n_nodes=nn, n_iter=it, status=st, draws=draws,
                branches=br)
