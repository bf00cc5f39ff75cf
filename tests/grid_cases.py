"""Inputs and reference calls for tests/test_grid.py and tests/golden/make_grid_golden.py: the demo, seeded scenarios
inside the reference's defined domain, corner cases, and the reference's own planners (oracle/_ref/libref_astar.so,
libref_dijkstra.so) with what they compute recovered from their cv::rectangle calls."""
import ctypes as C
import os

import numpy as np

from cpprobotics_b200 import synth
from oracle import grid as OG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = {OG.ASTAR: os.path.join(ROOT, "oracle", "_ref", "libref_astar.so"),
       OG.DIJKSTRA: os.path.join(ROOT, "oracle", "_ref", "libref_dijkstra.so")}
ALGOS = ((OG.ASTAR, "astar"), (OG.DIJKSTRA, "dijkstra"))
IMG_RESO = 5   # the planners' img_reso: a cell x is drawn from x * 5 + 1


def ref_lib(algo):
    p = REF[algo]
    return C.CDLL(p) if os.path.exists(p) else None


def ref_run(L, sx, sy, gx, gy, ox, oy, reso, rr):
    """The reference planner on one query.  Returns dict(map_cells [k, 2] box-relative blocked cells in drawing order,
    trace [k, 2] absolute cells, path [k, 2] absolute cells (goal first)).  Only for defined inputs."""
    x, y = np.ascontiguousarray(ox, np.float32), np.ascontiguousarray(oy, np.float32)
    F = C.c_float
    cap = 1 << 16
    while True:
        out = np.zeros(8 * cap, np.int32)
        k = L.ref_grid_run(F(sx), F(sy), F(gx), F(gy), x.size, x.ctypes.data_as(C.c_void_p),
                           y.ctypes.data_as(C.c_void_p), F(reso), F(rr), out.ctypes.data_as(C.c_void_p), cap)
        if k <= cap:
            break
        cap = k
    rec = out[:8 * k].reshape(k, 8)
    cell = (rec[:, :2] - 1) // IMG_RESO
    assert ((rec[:, :2] - 1) % IMG_RESO == 0).all()
    color = [tuple(c) for c in rec[:, 4:7]]
    black = np.array([c == (0, 0, 0) for c in color])
    green = np.array([c == (0, 255, 0) for c in color])
    blue = np.array([c == (255, 0, 0) for c in color])
    assert blue[0] and color[1] == (0, 0, 255)   # the start and goal markers
    # the trailing run of filled blue rectangles is calc_final_path's
    j = k
    while j > 2 and blue[j - 1] and rec[j - 1, 7] == -1:
        j -= 1
    return dict(map_cells=cell[black], trace=cell[green], path=cell[j:])


def check_ref_domain(algo, box, status):
    """The reference is defined on a square box (for A* also min = 0), a start inside and a reachable goal."""
    W, H = OG.dims(box)
    return W == H and (algo != OG.ASTAR or (box[0] == 0 and box[1] == 0)) and status == OG.FOUND


def demo():
    """(ox, oy, reso, rr, sg [4, 1])"""
    ox, oy = synth.grid_demo_obstacles()
    d = synth.GRID_DEMO
    return ox, oy, d["reso"], d["rr"], np.float32([[d["sx"]], [d["sy"]], [d["gx"]], [d["gy"]]])


def seeded_scenarios(algo, count, seed):
    """count random scenarios inside the reference's domain: a square box of side 4..64 cells (min = 0 for A*, any
    min for Dijkstra), reso in {0.5, 1, 2}, rr / reso in [-0.3, 2.2], 2 + up to side^2 / 12 scattered obstacles (two
    of them pin the box's corners), and one start / goal pair on free cells (maps without one are skipped).  Yields
    (ox, oy, reso, rr, sx, sy, gx, gy)."""
    rng = np.random.default_rng(seed)
    made = 0
    while made < count:
        side = int(rng.integers(4, 65))
        reso = float(rng.choice([0.5, 1.0, 2.0]))
        rr = float(np.float32(rng.uniform(-0.3, 2.2) * reso))
        mn = (0, 0) if algo == OG.ASTAR else tuple(int(v) for v in rng.integers(-40, 40, 2))
        k = int(rng.integers(0, side * side // 12 + 1))
        cx = np.concatenate([[mn[0], mn[0] + side], rng.integers(mn[0], mn[0] + side + 1, k)])
        cy = np.concatenate([[mn[1], mn[1] + side], rng.integers(mn[1], mn[1] + side + 1, k)])
        # metres with a jitter the double rounding removes
        ox = ((cx + rng.uniform(-0.4, 0.4, cx.size)) * reso).astype(np.float32)
        oy = ((cy + rng.uniform(-0.4, 0.4, cy.size)) * reso).astype(np.float32)
        box = OG.box_of_obstacles(ox, oy, reso)
        m = OG.obstacle_map(ox, oy, reso, rr, box)
        if m.all():
            continue
        made += 1
        sg = synth.grid_inputs(1, box, m, reso, seed=int(rng.integers(1 << 30)), i0=int(rng.integers(1, 64)) * 64 + 7)
        yield ox, oy, reso, rr, float(sg[0, 0]), float(sg[1, 0]), float(sg[2, 0]), float(sg[3, 0])


def corner_cases():
    """(name, ox, oy, reso, rr, sx, sy, gx, gy), each inside the reference's domain for both planners."""
    ox, oy = synth.grid_demo_obstacles()
    out = [("start_is_goal", ox, oy, 1.0, 1.0, 10.0, 10.0, 10.0, 10.0),
           ("goal_adjacent", ox, oy, 1.0, 1.0, 10.0, 10.0, 11.0, 11.0),
           ("start_on_obstacle", ox, oy, 1.0, 1.0, 21.0, 5.0, 30.0, 5.0)]
    # an empty open box: only the two corner obstacles, rr below every distance
    e = np.float32([0.0, 24.0]), np.float32([0.0, 24.0])
    out += [("open_box", e[0], e[1], 1.0, -1.0, 3.0, 4.0, 20.0, 17.0),
            ("open_box_far_corner", e[0], e[1], 1.0, -1.0, 0.0, 0.0, 23.0, 23.0)]
    # .5 in start, goal and obstacles: roundf / round take them away from zero
    h = np.float32([0.0, 12.5, 5.5, 6.5, 7.5, 16.0]), np.float32([0.0, 12.5, 2.5, 8.5, 3.5, 16.0])
    out += [("half_rounding", h[0], h[1], 1.0, 0.9, 2.5, 1.5, 10.5, 11.5),
            ("half_rounding_reso2", h[0] * 2, h[1] * 2, 2.0, 1.5, 5.0, 3.0, 21.0, 23.0)]
    return out
