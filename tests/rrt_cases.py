"""Inputs and reference calls for tests/test_rrt.py and tests/golden/make_rrt_golden.py: the demo, scattered maps,
corner cases, and the reference's own RRT::planning (oracle/_ref/libref_rrt.so) with a seeded goal_gen."""
import ctypes as C
import os

import numpy as np

from cpprobotics_b200 import synth
from oracle import rrt as OR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libref_rrt.so")


def ref_lib():
    return C.CDLL(REF) if os.path.exists(REF) else None


def demo_prm(max_iter=4096):
    """The demo's planner (src/rrt.cpp: rand_area {-2, 15}, expand_dis 0.5) with a cap the demo never reaches."""
    d = synth.RRT_DEMO
    return dict(rand_min=d["rand_min"], rand_max=d["rand_max"], expand_dis=d["expand_dis"], goal_sample_rate=5,
                max_iter=max_iter)


def ref_run(L, prm, ob, sx, sy, gx, gy, seed, cap):
    """The reference on one query.  Returns dict(tree [k, 2], parent [k], path [m, 2] (end ... start), draws), or None
    when it accepts more than cap nodes."""
    o = np.ascontiguousarray(ob, np.float32).reshape(-1, 3)
    tree = np.zeros(2 * cap, np.float32)
    parent = np.zeros(cap, np.int32)
    path = np.zeros(2 * (cap + 1), np.float32)
    pl, dr = C.c_int(0), C.c_longlong(0)
    F = C.c_float
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    k = L.ref_rrt_run(F(sx), F(sy), F(gx), F(gy), o.shape[0], p(o), F(prm["rand_min"]), F(prm["rand_max"]),
                      F(prm["expand_dis"]), int(prm["goal_sample_rate"]), C.c_uint32(seed), cap, p(tree), p(parent),
                      p(path), C.byref(pl), C.byref(dr))
    if k < 0:
        return None
    return dict(tree=tree[:2 * k].reshape(k, 2), parent=parent[:k], path=path[:2 * pl.value].reshape(pl.value, 2),
                draws=dr.value)


def checker_one(prm, ob, sx, sy, gx, gy, seed):
    """The checker on one query with room for every node and point: dict as ref_run's plus status and n_iter."""
    cap = int(prm["max_iter"]) + 1
    r = OR.plan(prm, ob, np.float32([[sx], [sy], [gx], [gy]]), np.uint32([seed]), max_pts=cap + 1, max_nodes=cap)
    k, m = int(r["n_nodes"][0]), int(r["path_len"][0])
    return dict(tree=r["tree"][:2 * k, 0].reshape(k, 2), parent=r["parent"][:k, 0],
                path=r["path"][:2 * m, 0].reshape(m, 2), draws=int(r["draws"][0]), status=int(r["status"][0]),
                n_iter=int(r["n_iter"][0]))


def scattered_maps(count, seed):
    """count seeded scenarios: 4..40 obstacles of radius 0.2..1.5 over a square area of side 8..40, expand_dis 0.3..2,
    goal_sample_rate 0..30, and a start / goal pair drawn outside the obstacles.  Yields (prm, ob, sx, sy, gx, gy,
    seed)."""
    rng = np.random.default_rng(seed)
    for _ in range(count):
        side = float(rng.uniform(8, 40))
        lo = float(rng.uniform(-10, 5))
        k = int(rng.integers(4, 41))
        ob = np.stack([rng.uniform(lo, lo + side, k), rng.uniform(lo, lo + side, k),
                       rng.uniform(0.2, 1.5, k)], axis=1).astype(np.float32)
        prm = dict(rand_min=np.float32(lo), rand_max=np.float32(lo + side),
                   expand_dis=np.float32(rng.uniform(0.3, 2.0)), goal_sample_rate=int(rng.integers(0, 31)),
                   max_iter=8192)
        pts = []
        while len(pts) < 2:
            p = rng.uniform(lo, lo + side, 2).astype(np.float32)
            if (np.hypot(ob[:, 0] - p[0], ob[:, 1] - p[1]) > ob[:, 2] + 0.05).all():
                pts.append(p)
        yield prm, ob, float(pts[0][0]), float(pts[0][1]), float(pts[1][0]), float(pts[1][1]), int(rng.integers(1 << 32))


# demo seeds whose run takes a rare branch, found by scanning seeds 0..2^20 with the checker (its `branches` output)
REDRAW_SEEDS = [116411, 348681, 376035, 487627]      # a uniform_int_distribution redraw (low word below 68)
CANONICAL_ONE_SEEDS = [209138, 492364, 508205, 523231]  # generate_canonical rounds to 1.0 (u >= 2^32 - 128)
