"""ctypes wrapper of oracle/lib/liboracle_grid.so — the CPU restatement of src/a_star.cpp and src/dijkstra.cpp: the
obstacle cells and box, calc_obstacle_map, the two searches with calc_final_path, the expansion trace, and the
restated libstdc++ heap on its own.  Built by `make -C oracle -f grid.mk` (python __graft_entry__.py).

TEST INFRASTRUCTURE ONLY, like oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liboracle_grid.so")

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_lib = None

# include/crb.h
ASTAR, DIJKSTRA = 0, 1
FOUND, NO_PATH, START_OUTSIDE, BAD_POINT = 0, 1, 2, 3
MAX_SIDE, MAX_CELLS = 32768, 1 << 24


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} missing: run `make -C oracle -f grid.mk` (or python __graft_entry__.py)")
        L = C.CDLL(LIB_PATH)
        L.crb_oracle_grid_box.restype = C.c_int
        L.crb_oracle_grid_box.argtypes = [C.c_int64, f32p, f32p, C.c_float, i32p]
        L.crb_oracle_grid_map.restype = None
        L.crb_oracle_grid_map.argtypes = [C.c_int64, f32p, f32p, C.c_float, C.c_float, i32p, u8p]
        L.crb_oracle_grid_plan.restype = None
        L.crb_oracle_grid_plan.argtypes = [C.c_int, i32p, u8p, C.c_float, C.c_int64, f32p, C.c_int, C.c_void_p,
                                           i32p, f32p, i32p, i32p, C.c_int]
        L.crb_oracle_grid_trace.restype = C.c_int64
        L.crb_oracle_grid_trace.argtypes = [C.c_int, i32p, u8p, C.c_float, C.c_float, C.c_float, C.c_float,
                                            C.c_float, i32p, C.c_int64]
        L.crb_oracle_grid_heap_run.restype = C.c_int64
        L.crb_oracle_grid_heap_run.argtypes = [C.c_int64, u8p, f32p, i32p]
        _lib = L
    return _lib


def num_threads() -> int:
    return len(os.sched_getaffinity(0))


def box_of_obstacles(ox, oy, reso):
    """(min_x, min_y, max_x, max_y) as int32[4], or None where crb_grid_box_of_obstacles refuses the input."""
    x, y = np.ascontiguousarray(ox, np.float32), np.ascontiguousarray(oy, np.float32)
    b = np.zeros(4, np.int32)
    return b if lib().crb_oracle_grid_box(x.size, x, y, np.float32(reso), b) == 0 else None


def dims(box):
    return int(box[2]) - int(box[0]), int(box[3]) - int(box[1])


def obstacle_map(ox, oy, reso, rr, box):
    """calc_obstacle_map: uint8 [W, H], 1 = blocked."""
    x, y = np.ascontiguousarray(ox, np.float32), np.ascontiguousarray(oy, np.float32)
    b = np.ascontiguousarray(box, np.int32)
    W, H = dims(b)
    m = np.zeros((W, H), np.uint8)
    lib().crb_oracle_grid_map(x.size, x, y, np.float32(reso), np.float32(rr), b, m)
    return m


def plan(algo, box, grid_map, reso, sg, max_pts=0, path_fill=np.nan, nthreads=0):
    """The planners for sg [4, n] (sx, sy, gx, gy) on one map: dict(path [2*max_pts, n] (path_fill past path_len),
    path_len, cost, n_visited, status), crb_grid_plan_batched's layout."""
    s = np.ascontiguousarray(sg, np.float32)
    n = s.shape[1]
    b = np.ascontiguousarray(box, np.int32)
    m = np.ascontiguousarray(grid_map, np.uint8)
    path = np.full((2 * max_pts, n), path_fill, np.float32)
    ln, nv, st = (np.zeros(n, np.int32) for _ in range(3))
    cost = np.zeros(n, np.float32)
    lib().crb_oracle_grid_plan(int(algo), b, m, np.float32(reso), n, s, int(max_pts),
                               path.ctypes.data if max_pts > 0 else None, ln, cost, nv, st, int(nthreads))
    return dict(path=path, path_len=ln, cost=cost, n_visited=nv, status=st)


def trace(algo, box, grid_map, reso, sx, sy, gx, gy):
    """One query's expansion trace: int32 [k, 2] absolute cells in the order the reference draws them, or None for a
    query the search does not run (START_OUTSIDE, BAD_POINT)."""
    b = np.ascontiguousarray(box, np.int32)
    m = np.ascontiguousarray(grid_map, np.uint8)
    f = np.float32
    args = (int(algo), b, m, f(reso), f(sx), f(sy), f(gx), f(gy))
    cap = 1 << 16
    while True:
        t = np.zeros(2 * cap, np.int32)
        k = lib().crb_oracle_grid_trace(*args, t, cap)
        if k < 0:
            return None
        if k <= cap:
            return t[:2 * k].reshape(k, 2)
        cap = int(k)


def heap_run(op, keys):
    """The restated heap: op[i] 1 pushes keys[i] with id i, 0 pops.  Returns the popped ids in order."""
    o = np.ascontiguousarray(op, np.uint8)
    k = np.ascontiguousarray(keys, np.float32)
    out = np.zeros(max(1, int((o == 0).sum())), np.int32)
    n = lib().crb_oracle_grid_heap_run(o.size, o, k, out)
    if n < 0:
        raise ValueError("pop of an empty heap")
    return out[:n]
