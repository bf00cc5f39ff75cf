"""Inputs and reference calls for tests/test_grid.py, tests/test_grid_boxes.py and tests/golden/make_grid_golden.py:
the demo, seeded scenarios inside the reference's defined domain, corner cases, the reference's own planners
(oracle/_ref/libref_astar.so, libref_dijkstra.so) with what they compute recovered from their cv::rectangle calls, and
the boxes away from the demo (rectangular, offset, at the ends of the int range, degenerate, a maze, maximum size),
each with a one-line reason."""
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


def same(a, b):
    """The rule every GPU output is held to against the checker: bitwise equal, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


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


# ---- boxes away from the demo (tests/test_grid_boxes.py) --------------------------------------------------------
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


def random_map(W, H, density, seed):
    """uint8 [W, H], each cell blocked with probability density"""
    return (np.random.default_rng(seed).random((W, H)) < density).astype(np.uint8)


# name -> (reason, (min_x, min_y), (W, H), density, reso); the maps are random_map(W, H, density, seed of the name)
BOXES = {
    "tall_17x61": ("W != H and min = (-7, 5): a swapped W and H, or a dropped offset, leaves the box",
                   (-7, 5), (17, 61), 0.25, 0.3),
    "wide_61x17": ("the transpose of tall_17x61, at min = (5, -7)", (5, -7), (61, 17), 0.25, 0.7),
    "corridor_1x53": ("W = 1: every move but two leaves the box; reso 2.5", (-7, 5), (1, 53), 0.0, 2.5),
    "corridor_53x1": ("H = 1: the parent step is the move's x times H = 1; reso 1e3", (5, -7), (53, 1), 0.0, 1e3),
    "winding_45x70": ("density 0.42: long, winding paths and many unreachable goals", (-300, 812), (45, 70), 0.42, 1.0),
    "winding_70x45": ("density 0.45 at reso 1e-3, min far from zero", (911, -1000), (70, 45), 0.45, 1e-3),
    "sparse_89x23": ("density 0.05 at reso 2.5: near-straight paths, Dijkstra ties everywhere", (1000, -1000),
                     (89, 23), 0.05, 2.5),
    "mid_37x29": ("density 0.15 at the non-dyadic reso 0.7, negative min on both axes", (-512, -77), (37, 29), 0.15,
                  0.7),
}


def box_case(name):
    """(box int32[4], map uint8 [W, H], reso) of BOXES[name]"""
    _, (x0, y0), (W, H), density, reso = BOXES[name]
    seed = sum(name.encode()) * 7919 + W * 131 + H
    return np.int32([x0, y0, x0 + W, y0 + H]), random_map(W, H, density, seed), reso


def scatter_case(reso=0.7, rr=0.9):
    """A map from crb_grid_obstacle_map's rule on a rectangular, offset box: 700 obstacles scattered over 64 x 40
    cells at min = (-37, 101), two of them pinning the box's corners.  (ox, oy, reso, rr)."""
    rng = np.random.default_rng(0x5CA7)
    cx = np.concatenate([[-37, -37 + 64], rng.integers(-37, -37 + 64, 700)])
    cy = np.concatenate([[101, 101 + 40], rng.integers(101, 101 + 40, 700)])
    ox = ((cx + rng.uniform(-0.4, 0.4, cx.size)) * reso).astype(np.float32)
    oy = ((cy + rng.uniform(-0.4, 0.4, cy.size)) * reso).astype(np.float32)
    return ox, oy, reso, float(np.float32(rr * reso))


def int_end_cases():
    """Boxes at the ends of the int range, reso 1: name -> (reason, box, map, sg [4, n]).  Near 2^31 a float holds
    only multiples of 128, so start and goal lie on such cells and every path crosses cells whose coordinates round
    when converted to float; the map is random at density 0.1 with those cells kept free."""
    out = {}
    # min_x = -2^31: cells x in [-2^31, -2^31 + 300); x = -2^31 + 128 k for k = 0, 1, 2 are floats
    box = np.int32([I32_MIN, -20, I32_MIN + 300, 20])
    m = random_map(300, 40, 0.1, 0xE1)
    xs = [I32_MIN, I32_MIN + 128, I32_MIN + 256]
    ys = [-20, -7, 0, 6, 19]
    for x in xs:
        m[x - I32_MIN, [y + 20 for y in ys]] = 0
    sg = [(xs[0], -20, xs[2], 19), (xs[2], 19, xs[0], -20), (xs[1], 0, xs[2], 6), (xs[0], 6, xs[1], -7),
          (xs[1], -7, xs[1], -7), (xs[2], 0, xs[0], 0)]
    # past max_x (-2^31 + 384, a float): a goal there is NO_PATH, a start START_OUTSIDE
    sg += [(xs[0], 0, I32_MIN + 384, 0), (I32_MIN + 384, 0, xs[0], 0)]
    # the next float below -2^31 (-2^31 - 256) and -2^32 round to no int: BAD_POINT
    sg += [(xs[0], 0, -2147483904.0, 0), (-4294967296.0, 0, xs[1], 0)]
    # a goal past max_y: NO_PATH after visiting the start's component
    sg += [(xs[1], 6, xs[1], 20)]
    out["min_x_int_min"] = ("min_x = -2^31: offsets and point conversions at the bottom of the int range", box, m,
                            np.float32(sg).T.copy())
    # max_y = 2^31 - 1: cells y in [2^31 - 301, 2^31 - 1); y = 2^31 - 128, 2^31 - 256 are floats
    box = np.int32([-17, I32_MAX - 300, 23, I32_MAX])
    m = random_map(40, 300, 0.1, 0xE2)
    ys = [I32_MAX + 1 - 128, I32_MAX + 1 - 256]
    xs = [-17, -3, 0, 22]
    for y in ys:
        m[[x + 17 for x in xs], y - (I32_MAX - 300)] = 0
    sg = [(-17, ys[0], 22, ys[1]), (22, ys[1], -17, ys[0]), (0, ys[0], -3, ys[1]), (-3, ys[1], -3, ys[1]),
          (0, ys[1], 22, ys[1])]
    # 2^31 rounds to no int: BAD_POINT, as a goal and as a start
    sg += [(0, ys[0], 0, 2147483648.0), (0, 2147483648.0, 0, ys[0])]
    # a goal below the box's y range, a start right of it
    sg += [(0, ys[0], 0, I32_MAX + 1 - 512), (23, ys[0], 0, ys[0])]
    out["max_y_int_max"] = ("max_y = 2^31 - 1: the top of the int range, where 2^31 itself is a float and no int", box,
                            m, np.float32(sg).T.copy())
    return out


def maze(W=257, H=129):
    """A serpentine corridor: walls on every odd column with one gap, alternately at the top and the bottom, so the
    only way from column 0 to column W - 1 walks every free column end to end (more than 10^4 points)."""
    m = np.zeros((W, H), np.uint8)
    for k, x in enumerate(range(1, W, 2)):
        m[x, :] = 1
        m[x, H - 1 if k % 2 == 0 else 0] = 0
    return m


# Maximum-size boxes: name -> (reason, (W, H)); W * H = CRB_GRID_MAX_CELLS, random maps at density 0.2
MAX_BOXES = {
    "max_4096x4096": ("the square at CRB_GRID_MAX_CELLS: the largest heap and state per slot", (4096, 4096)),
    "max_32768x512": ("W at CRB_GRID_MAX_SIDE: cell indices up to 2^24 - 1 with a short column", (32768, 512)),
    "max_512x32768": ("H at CRB_GRID_MAX_SIDE: x * H is the large term of every index", (512, 32768)),
}


def max_case(name, min_xy=(-1234, 567)):
    """(box, map, reso, sg [4, n]) for MAX_BOXES[name], reso 0.5.  Every search stays bounded: start / goal pairs at
    most 96 cells apart on free cells of one component within a 256-cell window, and one NO_PATH query whose start
    lies in an 8 x 8 pocket walled off by a ring of blocked cells (64 cells visited).  n = 7: each of the 3 slots
    takes more than one query."""
    _, (W, H) = MAX_BOXES[name]
    rng = np.random.default_rng(W * 7 + H)
    m = (rng.random((W, H), dtype=np.float32) < 0.2).astype(np.uint8)
    x0, y0 = min_xy
    box = np.int32([x0, y0, x0 + W, y0 + H])
    reso = 0.5
    sg = []
    anchors = [(0, 0), (W - 1, H - 1), (W // 2, H // 2), (W - 1, 0), (0, H - 1), (W // 3, 2 * H // 3)]
    for k, (ax, ay) in enumerate(anchors):
        # a window of 256 x 256 cells (clipped) holding the pair; both cells freed, then a connecting check
        wx0, wy0 = min(max(ax - 128, 0), max(W - 256, 0)), min(max(ay - 128, 0), max(H - 256, 0))
        sx, sy = ax, ay
        while True:
            d = rng.integers(-96, 97, 2)
            gx, gy = min(max(sx + int(d[0]), 0), W - 1), min(max(sy + int(d[1]), 0), H - 1)
            if (gx, gy) != (sx, sy):
                break
        m[sx, sy] = m[gx, gy] = 0
        win = m[wx0:wx0 + 256, wy0:wy0 + 256]
        if not _connected(win, (sx - wx0, sy - wy0), (gx - wx0, gy - wy0)):
            # carve an L-shaped free corridor between them
            m[min(sx, gx):max(sx, gx) + 1, sy] = 0
            m[gx, min(sy, gy):max(sy, gy) + 1] = 0
        sg.append((sx + x0, sy + y0, gx + x0, gy + y0))
    # the pocket: interior [px, px + 8) x [py, py + 8) free, the ring around it blocked
    px, py = W // 4 + 1, min(H // 4 + 1, H - 10)
    m[px - 1:px + 9, py - 1:py + 9] = 1
    m[px:px + 8, py:py + 8] = 0
    gx, gy = px + 20 if px + 20 < W else px - 20, py + 4
    m[gx, gy] = 0
    sg.append((px + 3 + x0, py + 3 + y0, gx + x0, gy + y0))
    sg = np.float32(sg).T * np.float32(reso)
    return box, m, reso, np.ascontiguousarray(sg, np.float32)


def _connected(m, a, b):
    """a and b joined by 8-neighbour moves into free cells of m (a itself may be anything)"""
    from scipy import ndimage
    lab, _ = ndimage.label(m == 0, structure=np.ones((3, 3), int))
    return lab[a] != 0 and lab[a] == lab[b]


MAP_BYTES = (1, 2, 0x7F, 0x80, 0x88, 0xFF)   # nonzero = blocked; 0x80 and 0x88 are the kernel's own state bits


def square_cases():
    """(name, ox, oy, reso, rr, sx, sy, gx, gy) inside the reference's domain for both planners (a square box at
    min = 0, a reachable goal): the resolutions of the box tests, start and goal at exact halves and at 0.49999997 of
    a cell, obstacles at .5, and rr at reso * (float)sqrt(2), its float predecessor, 0 and below 0, which put the
    diagonal neighbour of an obstacle on both sides of the map test."""
    f = np.float32
    out = []
    side, goal, start = 23, (17, 15), (3, 4)
    for j, reso in enumerate((0.3, 0.7, 2.5, 1e-3, 1e3)):
        rng = np.random.default_rng(0x5A + j)
        c = rng.integers(0, side, (2, 60))   # below side: + .5 keeps the box square
        away = [np.maximum(abs(c[0] - e[0]), abs(c[1] - e[1])) > 3 for e in (goal, start)]
        c = c[:, away[0] & away[1]][:, :18]
        cx = np.concatenate([[0, side], c[0]]).astype(np.float64)
        cy = np.concatenate([[0, side], c[1]]).astype(np.float64)
        cx[2:8] += 0.5   # obstacles at .5: away from zero
        ox, oy = f(cx) * f(reso), f(cy) * f(reso)
        diag = f(reso) * f(1.41421354)
        for rname, rr in (("diag", diag), ("below_diag", np.nextafter(diag, f(0))), ("zero", f(0)), ("neg", -f(reso))):
            out.append((f"reso{reso:g}_{rname}", ox, oy, reso, float(rr), float(f(2.5) * f(reso)),
                        float(f(3.49999997) * f(reso)), float(f(goal[0] - 0.5) * f(reso)),
                        float(f(goal[1] + 0.49999997) * f(reso))))
    # the 1 x 1 box: obstacles at (0, 0) and (1, 1), rr < 0 so that the one cell is free
    o = np.float32([0, 1])
    out.append(("box_1x1", o, o, 1.0, -1.0, 0.0, 0.0, 0.4, -0.4))
    return out
