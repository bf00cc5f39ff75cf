"""Grid A* and Dijkstra away from the demo: rectangular and offset boxes, the ends of the int range, degenerate boxes,
a maze, maximum-size boxes, workspace reuse, any nonzero map byte, the rounding of start and goal, and the obstacle
map on such boxes (case sets in tests/grid_cases.py).

Two references for every case.  The checker (oracle/grid.py), which the GPU must equal bit for bit.  And a float64
oracle, here, that shares no code with the checker: cells are copysign(floor(|q| + 0.5), q) of the float32 quotient
q = p / reso, which decide BAD_POINT, START_OUTSIDE and whether the goal is in the box; the map blocks a cell when
float32(sqrt(dx^2 + dy^2)) <= float32(rr) / float32(reso) for an obstacle rounded in float64; and d64 is the float64
shortest distance of scipy.sparse.csgraph.dijkstra on the graph verify_node defines (steps 1 and sqrt 2, a move
allowed into any free cell of the box).  With d64: NO_PATH exactly when the goal cannot be reached, n_visited then the
reachable count; a found path is an 8-neighbour walk inside the box from the goal to the start over free cells, each
point float32(cell) * float32(reso) and never -0; Dijkstra's cost and path length are d64 within
(path_len + 1) * 2^-23 relative, and its n_visited lies between the counts of cells nearer and not farther than the
goal; A*'s path is no shorter than d64.

CPU: the checker against the float64 oracle on every small and medium case, and against the reference text on the
square cases inside its domain.  H100: both kernels against the checker, bitwise, and against the float64 oracle."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

import grid_cases as GC
from grid_cases import same
from cpprobotics_b200 import _lib, synth
from oracle import grid as OG

F = np.float32
EPS = 2.0 ** -23
MOVES = ((1, 0), (0, 1), (-1, 0), (0, -1), (-1, -1), (-1, 1), (1, -1), (1, 1))
ALGO_IDS = [a for a, _ in GC.ALGOS]
KEYS = ("path", "path_len", "cost", "n_visited", "status")
NS = (1, 33, 4097)


# ---- the float64 oracle -----------------------------------------------------------------------------------------
def cells64(p, reso):
    """(cell int64, ok): copysign(floor(|q| + 0.5), q) of the float32 quotient q = p / reso, evaluated in float64; ok
    is false where that is not finite or leaves the int range."""
    with np.errstate(all="ignore"):
        q = (np.asarray(p, F) / F(reso)).astype(np.float64)
        r = np.copysign(np.floor(np.abs(q) + 0.5), q)
        ok = np.isfinite(r) & (r >= -2.0 ** 31) & (r < 2.0 ** 31)
    return np.where(ok, r, 0).astype(np.int64), ok


def map64(ox, oy, reso, rr, box):
    """bool [W, H]: blocked when float32(sqrt(dx^2 + dy^2)) <= float32(rr) / float32(reso) for some obstacle, whose
    cell is its float64 quotient rounded half away from zero (none where that leaves the int range)."""
    W, H = OG.dims(box)
    thr = F(rr) / F(reso)
    with np.errstate(all="ignore"):
        qx, qy = (np.asarray(o, F).astype(np.float64) / float(F(reso)) for o in (ox, oy))
        cx, cy = (np.copysign(np.floor(np.abs(q) + 0.5), q) for q in (qx, qy))
    ok = np.isfinite(cx) & np.isfinite(cy) & (np.abs(cx + 0.5) <= 2.0 ** 31) & (np.abs(cy + 0.5) <= 2.0 ** 31)
    R = int(np.ceil(max(float(thr), 0.0))) + 1   # no cell farther than R on an axis can pass the test
    m = np.zeros((W, H), bool)
    for x, y in zip(cx[ok].astype(np.int64), cy[ok].astype(np.int64)):
        x0, x1 = max(x - R, int(box[0])), min(x + R + 1, int(box[2]))
        y0, y1 = max(y - R, int(box[1])), min(y + R + 1, int(box[3]))
        if x0 >= x1 or y0 >= y1:
            continue
        dx = np.arange(x0, x1, dtype=np.float64) - x
        dy = np.arange(y0, y1, dtype=np.float64) - y
        d = np.sqrt(dx[:, None] ** 2 + dy[None, :] ** 2).astype(F)
        m[x0 - box[0]:x1 - box[0], y0 - box[1]:y1 - box[1]] |= d <= thr
    return m


def graph64(m):
    """verify_node's graph: an edge from every cell of the box to every free 8-neighbour in it, weight 1 or sqrt 2"""
    W, H = m.shape
    idx = np.arange(W * H).reshape(W, H)
    free = np.asarray(m) == 0
    src, dst, w = [], [], []
    for dx, dy in MOVES:
        sx, sy = slice(max(0, -dx), W - max(0, dx)), slice(max(0, -dy), H - max(0, dy))
        tx, ty = slice(max(0, dx), W - max(0, -dx)), slice(max(0, dy), H - max(0, -dy))
        f = free[tx, ty]
        src.append(idx[sx, sy][f])
        dst.append(idx[tx, ty][f])
        w.append(np.full(int(f.sum()), np.sqrt(2.0) if dx and dy else 1.0))
    return csr_matrix((np.concatenate(w), (np.concatenate(src), np.concatenate(dst))), shape=(W * H, W * H))


def _decode(pts, reso):
    """the cells whose points (float32(cell) * reso) are pts [k, 2], when rint(p / reso) gives them; None otherwise"""
    c = np.rint(pts.astype(np.float64) / float(F(reso)))
    if not np.isfinite(c).all():
        return None
    c = c.astype(np.int64)
    if not same(c.astype(F) * F(reso), pts):
        return None
    return c


def walk64(pts, reso, box, m, first, last):
    """(lo, hi): the least and greatest float64 length of a cell walk whose points are pts [k, 2] (goal first), that
    begins at cell `first`, takes 8-neighbour steps inside the box, passes only free cells except the final one when
    `last` is given, and ends at `last` (anywhere when None).  None when no walk fits.  Near 2^31 several cells share
    a point, so the walks are followed as sets of cells."""
    W, H = OG.dims(box)
    k = len(pts)
    free = np.asarray(m) == 0
    need_free = np.ones(k, bool)
    if last is not None:
        need_free[-1] = False
    c = _decode(pts, reso)
    if c is not None:
        r = c - np.int64(box[:2])
        step = np.abs(np.diff(c, axis=0))
        inside = ((r >= 0) & (r < [W, H])).all()
        if (inside and tuple(c[0]) == tuple(first) and (step.max(axis=1, initial=1) == 1).all()
                and (last is None or tuple(c[-1]) == tuple(last)) and free[r[need_free, 0], r[need_free, 1]].all()):
            L = float(np.where(step.sum(axis=1) == 2, np.sqrt(2.0), 1.0).sum())
            return L, L
    px = np.arange(box[0], box[2], dtype=np.int64).astype(F) * F(reso)
    py = np.arange(box[1], box[3], dtype=np.int64).astype(F) * F(reso)
    lo, hi = np.full((W, H), np.inf), np.full((W, H), -np.inf)
    f0 = (int(first[0]) - int(box[0]), int(first[1]) - int(box[1]))
    if not (0 <= f0[0] < W and 0 <= f0[1] < H and px[f0[0]] == pts[0, 0] and py[f0[1]] == pts[0, 1]):
        return None
    if need_free[0] and not free[f0]:
        return None
    lo[f0] = hi[f0] = 0.0
    for j in range(1, k):
        match = (px[:, None] == pts[j, 0]) & (py[None, :] == pts[j, 1])
        if need_free[j]:
            match &= free
        nlo, nhi = np.full((W, H), np.inf), np.full((W, H), -np.inf)
        for dx, dy in MOVES:
            s = np.sqrt(2.0) if dx and dy else 1.0
            sx, sy = slice(max(0, -dx), W - max(0, dx)), slice(max(0, -dy), H - max(0, dy))
            tx, ty = slice(max(0, dx), W - max(0, -dx)), slice(max(0, dy), H - max(0, -dy))
            nlo[tx, ty] = np.minimum(nlo[tx, ty], lo[sx, sy] + s)
            nhi[tx, ty] = np.maximum(nhi[tx, ty], hi[sx, sy] + s)
        lo, hi = np.where(match, nlo, np.inf), np.where(match, nhi, -np.inf)
        if np.isinf(lo).all():
            return None
    if last is not None:
        e = (int(last[0]) - int(box[0]), int(last[1]) - int(box[1]))
        return (lo[e], hi[e]) if np.isfinite(lo[e]) else None
    return float(lo[np.isfinite(lo)].min()), float(hi[np.isfinite(hi)].max())


def pre_status64(box, sg, reso):
    """(status, cells): BAD_POINT or START_OUTSIDE where the rule decides before any search, -1 elsewhere"""
    c = [cells64(sg[i], reso) for i in range(4)]
    ok = c[0][1] & c[1][1] & c[2][1] & c[3][1]
    sx, sy, gx, gy = (v[0] for v in c)
    s_in = (sx >= box[0]) & (sx < box[2]) & (sy >= box[1]) & (sy < box[3])
    return np.where(~ok, OG.BAD_POINT, np.where(~s_in, OG.START_OUTSIDE, -1)), (sx, sy, gx, gy)


def check_plan(algo, box, m, reso, sg, r, max_pts, d64=True):
    """Hold one batch's outputs r (dict of numpy arrays) to the float64 oracle.  d64=False (boxes too large for a
    float64 graph) keeps the cell, status and walk rules and drops those that need distances.  Returns the counts of
    each status."""
    W, H = OG.dims(box)
    n = sg.shape[1]
    free = np.asarray(m) == 0
    pre, (sx, sy, gx, gy) = pre_status64(box, sg, reso)
    st, plen, cost, nvis = r["status"], r["path_len"], r["cost"], r["n_visited"]
    path = r["path"] if max_pts > 0 else None
    if path is not None:
        z = path[~np.isnan(path)]
        assert not (np.signbit(z) & (z == 0)).any(), "a path point is -0"
    rs = (sx - box[0]) * H + (sy - box[1])
    g_in = (gx >= box[0]) & (gx < box[2]) & (gy >= box[1]) & (gy < box[3])
    rg = np.where(g_in, (gx - box[0]) * H + (gy - box[1]), -1)
    search = np.flatnonzero(pre < 0)
    rows = {}
    if d64 and search.size:
        G = graph64(m)
        starts = np.unique(rs[search])
        for i in range(0, starts.size, 256):
            D = dijkstra(G, directed=True, indices=starts[i:i + 256])
            rows.update(zip(starts[i:i + 256].tolist(), D))
    for q in range(n):
        where = (q, [float(v) for v in sg[:, q]])
        if pre[q] >= 0:
            assert st[q] == pre[q] and plen[q] == 0 and nvis[q] == 0 and np.isnan(cost[q]), where
            continue
        assert st[q] in (OG.FOUND, OG.NO_PATH), where
        goal_ok = g_in[q] and (free.reshape(-1)[rg[q]] or rg[q] == rs[q])   # a blocked start is its own goal
        if d64:
            row = rows[int(rs[q])]
            reach = int(np.isfinite(row).sum())
            dg = row[rg[q]] if goal_ok else np.inf
            if np.isinf(dg):
                assert st[q] == OG.NO_PATH and nvis[q] == reach and plen[q] == 0 and np.isnan(cost[q]), where
                continue
            assert st[q] == OG.FOUND, where
        elif not goal_ok:
            assert st[q] == OG.NO_PATH, where
            continue
        if st[q] == OG.NO_PATH:   # d64=False: the goal may be unreachable
            continue
        L = int(plen[q])
        tol = (L + 1) * EPS
        if rg[q] == rs[q]:
            assert L == 1 and cost[q] == 0 and nvis[q] == 1, where
        if d64:
            if algo == OG.DIJKSTRA:
                assert abs(float(cost[q]) - dg) <= tol * dg, (where, cost[q], dg)
                lo_n = int((row < dg * (1 - tol)).sum())
                hi_n = int((row <= dg * (1 + tol)).sum())
                assert lo_n <= nvis[q] <= hi_n, (where, lo_n, int(nvis[q]), hi_n)
            else:
                assert 1 <= nvis[q] <= reach, where
        if path is None:
            continue
        k = min(L, max_pts)
        pts = path[:2 * k, q].reshape(k, 2)
        assert np.isnan(path[2 * k:, q]).all(), where
        w = walk64(pts, reso, box, m, (gx[q], gy[q]), (sx[q], sy[q]) if k == L else None)
        assert w is not None, ("not a walk from the goal to the start", where)
        if d64 and k == L:
            if algo == OG.DIJKSTRA:
                assert w[0] <= dg * (1 + tol) and w[1] >= dg * (1 - tol), (where, w, dg)
            else:
                assert w[1] >= dg * (1 - tol), (where, w, dg)
    return np.bincount(st, minlength=4)


# ---- helpers ------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _box(b):
    return _lib.GridBox(*[int(v) for v in b])


def _gpu_plan(engine, algo, box, m, reso, sg, max_pts):
    r = engine.grid_plan(algo, _box(box), _dev(m), reso, _dev(sg), max_pts=max_pts)
    return {k: (None if v is None else v.cpu().numpy()) for k, v in r.items()}


def _gpu_map(engine, ox, oy, reso, rr, box):
    return engine.grid_obstacle_map(_dev(np.asarray(ox, F)), _dev(np.asarray(oy, F)), reso, rr, _box(box)).cpu().numpy()


def _bitwise(r, o):
    for k in KEYS:
        if o[k].size or r[k] is not None:
            assert same(r[k], o[k]), k


def _box_plan_case(name, n):
    """(box, map, reso, sg) for a BOXES entry or the scatter map, n queries of synth.grid_inputs"""
    if name == "scatter_64x40":
        ox, oy, reso, rr = GC.scatter_case()
        box = OG.box_of_obstacles(ox, oy, reso)
        m = OG.obstacle_map(ox, oy, reso, rr, box)
    else:
        box, m, reso = GC.box_case(name)
    return box, m, reso, synth.grid_inputs(n, box, m, reso, seed=0xB0C5 + n)


BOX_NAMES = list(GC.BOXES) + ["scatter_64x40"]
MAX_PTS = 96


def _points(reso):
    """start / goal coordinates for the rounding rules: exact and near halves, -0, 0.49999997 of a cell, the ends of
    the int range times reso, and plain metres (which overflow the quotient when reso is tiny)"""
    r = F(reso)
    with np.errstate(over="ignore"):   # at reso 3e38 most of them overflow to inf: BAD_POINT
        v = [F(s * (k + 0.5)) * r for k in (0, 1, 2, 5) for s in (1, -1)]
        v += [F(-0.0), F(0.49999997) * r, F(-0.49999997) * r, F(1.0), F(-3.0)]
        top = F(2.0 ** 31) * r
        v += [np.nextafter(top, F(0)), top, -top]
    return np.array(v, F)


def point_batch(box, reso, anchor, axis):
    """queries that put each of _points(reso) on one axis, as the goal and as the start, the other end and the other
    coordinate at the anchor cell; the map is open"""
    a = F(anchor[0]) * F(reso), F(anchor[1]) * F(reso)
    cols = []
    for p in _points(reso):
        pt = (p, a[1]) if axis == 0 else (a[0], p)
        cols += [(a[0], a[1], pt[0], pt[1]), (pt[0], pt[1], a[0], a[1])]
    return np.array(cols, F).T.copy()


POINT_CASES = [  # (name, box, reso, anchor cell, axis): an open map
    *[(f"tall_reso{r:g}_{'xy'[ax]}", np.int32([-7, -5, 10, 40]), r, (0, 0), ax)
      for r in (0.3, 0.7, 1.0, 2.5, 1e-3, 1e3, 1e-40, 3e38) for ax in (0, 1)],
    ("int_min_x", np.int32([GC.I32_MIN, -20, GC.I32_MIN + 300, 20]), 1.0, (GC.I32_MIN + 128, 0), 0),
    ("int_max_y", np.int32([-17, GC.I32_MAX - 300, 23, GC.I32_MAX]), 1.0, (0, GC.I32_MAX + 1 - 128), 1),
]
assert len({c[0] for c in POINT_CASES}) == len(POINT_CASES)


def _point_case(name):
    c = next(c for c in POINT_CASES if c[0] == name)
    _, box, reso, anchor, axis = c
    W, H = OG.dims(box)
    return box, np.zeros((W, H), np.uint8), reso, point_batch(box, reso, anchor, axis)


def _check_points(box, reso, sg, r):
    """the goal's cell is path point 0 and the start's the last; both must be the float64 rule's"""
    pre, (sx, sy, gx, gy) = pre_status64(box, sg, reso)
    for q in np.flatnonzero(r["status"] == OG.FOUND):
        L = int(r["path_len"][q])
        assert same(r["path"][:2, q], np.array([gx[q], gy[q]]).astype(F) * F(reso)), q
        assert same(r["path"][2 * L - 2:2 * L, q], np.array([sx[q], sy[q]]).astype(F) * F(reso)), q


def _degenerate_cases():
    """name -> (box, map, reso, sg, max_pts): 1 x 1 boxes, and corridors end to end at CRB_GRID_MAX_SIDE"""
    out = {}
    # the second box's cell (2^31 - 128, -2^31) is a float point; -2^31 + 128 is the next one above it
    for name, box in (("box_1x1", np.int32([-3, 8, -2, 9])),
                      ("box_1x1_int_ends", np.int32([GC.I32_MAX - 127, GC.I32_MIN, GC.I32_MAX - 126, GC.I32_MIN + 1]))):
        c = (F(box[0]), F(box[1]))
        sg = np.array([[c[0], c[1], c[0], c[1]], [c[0], c[1], c[0], F(box[1] + 128)]], F).T.copy()
        out[name] = (box, np.zeros((1, 1), np.uint8), 1.0, sg, 4)
    S = OG.MAX_SIDE
    for mp in (S, 1):
        out[f"corridor_{S}x1_max_pts{mp}"] = (np.int32([-100, 3, S - 100, 4]), np.zeros((S, 1), np.uint8), 0.5,
                                               np.array([[-50.0, 1.5, (S - 101) * 0.5, 1.5]], F).T.copy(), mp)
        out[f"corridor_1x{S}_max_pts{mp}"] = (np.int32([7, -S // 2, 8, S // 2]), np.zeros((1, S), np.uint8), 1.0,
                                               np.array([[7.0, S // 2 - 1, 7.0, -S // 2]], F).T.copy(), mp)
    return out


DEGENERATE = list(_degenerate_cases())


def _check_degenerate(name, algo, r):
    if name.startswith("box_1x1"):
        assert r["status"].tolist() == [OG.FOUND, OG.NO_PATH] and r["path_len"].tolist() == [1, 0]
        assert r["n_visited"].tolist() == [1, 1] and r["cost"][0] == 0
    else:
        assert r["status"][0] == OG.FOUND and r["path_len"][0] == OG.MAX_SIDE and r["n_visited"][0] == OG.MAX_SIDE
        if algo == OG.DIJKSTRA:
            assert r["cost"][0] == OG.MAX_SIDE - 1


def _maze_case(max_pts):
    m = GC.maze()
    W, H = m.shape
    box = np.int32([-100, 40, -100 + W, 40 + H])
    reso = 0.5
    sg = np.array([[-100 * reso, 40 * reso, (W - 101) * reso, 40 * reso],
                   [(W - 101) * reso, (40 + H - 1) * reso, -100 * reso, (40 + H - 1) * reso],
                   [-100 * reso, 40 * reso, -98 * reso, 41 * reso]], F).T.copy()
    return box, m, reso, sg, max_pts


MAZE_MAX_PTS = (1 << 15, 1000)


def _bytes_map(m, seed):
    """the blockage of m in bytes drawn from GC.MAP_BYTES"""
    b = np.random.default_rng(seed).choice(np.array(GC.MAP_BYTES, np.uint8), m.shape)
    return np.where(m != 0, b, 0).astype(np.uint8)


DIAG = F(1.41421354)


def map_cases():
    """(name, ox, oy, reso, rr, box) for the obstacle map: rectangular and offset boxes, n_obs across the 256-wide
    shared tile, obstacles outside the box and at .5, rr at reso * (float)sqrt(2) and its predecessor, 0 and < 0"""
    out = []
    boxes = (("tall", np.int32([-7, 5, 10, 66]), 0.3), ("wide", np.int32([5, -7, 66, 10]), 0.7),
             ("far", np.int32([-1000, 2000, -911, 2023]), 2.5), ("unit", np.int32([3, -40, 70, -9]), 1.0))
    for bname, box, reso in boxes:
        W, H = OG.dims(box)
        rng = np.random.default_rng(int(W * 1000 + H))
        for n_obs in (0, 1, 255, 256, 257, 513):
            # cells over the box and 3 cells past it on every side; a third of them at .5
            cx = rng.integers(box[0] - 3, box[2] + 3, n_obs).astype(np.float64)
            cy = rng.integers(box[1] - 3, box[3] + 3, n_obs).astype(np.float64)
            h = rng.random(n_obs) < 1 / 3
            cx[h] += rng.choice([-0.5, 0.5], int(h.sum()))
            cy[h] += rng.choice([-0.5, 0.5], int(h.sum()))
            ox, oy = F(cx) * F(reso), F(cy) * F(reso)
            diag = F(reso) * DIAG
            for rname, rr in (("diag", diag), ("below_diag", np.nextafter(diag, F(0))), ("zero", F(0)),
                              ("neg", F(-0.5) * F(reso)), ("wide", F(2.6) * F(reso))):
                if n_obs in (255, 257) and rname != "diag":
                    continue
                out.append((f"{bname}_n{n_obs}_{rname}", ox, oy, reso, float(rr), box))
    return out


MAP_CASES = map_cases()
MAP_NAMES = [c[0] for c in MAP_CASES]


def _map_case(name):
    return next(c for c in MAP_CASES if c[0] == name)[1:]


# ---- CPU: the checker against the float64 oracle -----------------------------------------------------------------
def test_float64_cell_rule_on_its_edges():
    """The rule itself: half away from zero, 0.49999997 stays, -0 is 0, overflow and the int range's ends."""
    c, ok = cells64(F([0.5, -0.5, 1.5, -2.5, 0.49999997, -0.49999997, -0.0, 2147483520.0, 2.0 ** 31, -2.0 ** 31,
                       np.inf, np.nan]), 1.0)
    assert c[:10].tolist() == [1, -1, 2, -3, 0, 0, 0, 2147483520, 0, -2 ** 31]
    assert ok.tolist() == [True] * 8 + [False, True, False, False]
    assert not cells64(F([1.0]), 1e-40)[1][0] and cells64(F([1e38]), 3e38)[0][0] == 0


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("name", BOX_NAMES)
def test_checker_meets_float64_oracle_on_boxes(name, n, algo):
    box, m, reso, sg = _box_plan_case(name, n)
    o = OG.plan(algo, box, m, reso, sg, max_pts=MAX_PTS)
    counts = check_plan(algo, box, m, reso, sg, o, MAX_PTS)
    if n == 4097:   # every status on a non-square, offset box
        assert (counts > 0).all(), counts


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("name", list(GC.int_end_cases()))
def test_checker_meets_float64_oracle_at_int_range_ends(name, algo):
    _, box, m, sg = GC.int_end_cases()[name]
    o = OG.plan(algo, box, m, 1.0, sg, max_pts=1024)
    counts = check_plan(algo, box, m, 1.0, sg, o, 1024)
    assert (counts > 0).all(), counts
    # the paths cross cells that share a float point
    found = np.flatnonzero(o["status"] == OG.FOUND)
    assert (o["path_len"][found] > 100).any()


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("name", [c[0] for c in POINT_CASES])
def test_checker_meets_float64_rule_for_points(name, algo):
    box, m, reso, sg = _point_case(name)
    o = OG.plan(algo, box, m, reso, sg, max_pts=512)
    counts = check_plan(algo, box, m, reso, sg, o, 512)
    _check_points(box, reso, sg, o)
    assert counts[OG.FOUND] > 0 and counts[OG.NO_PATH] + counts[OG.START_OUTSIDE] + counts[OG.BAD_POINT] > 0
    if reso == 1e-40:
        assert counts[OG.BAD_POINT] >= 4   # 1 m and -3 m overflow the quotient
    if name.startswith("tall_"):
        # +-0.5, +-1.5 and +-2.5 cells on the named axis, as goal and as start, plan inside the box (at reso 3e38
        # only +0.5 cell is finite)
        k = 2 if reso == 3e38 else 12
        assert (o["status"][:k] == OG.FOUND).all(), o["status"][:12]
        ax = 0 if name.endswith("_x") else 1
        assert (sg[2 + ax, 0:k:2] != 0).all() and (sg[ax, 1:k:2] != 0).all()


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("name", DEGENERATE)
def test_checker_meets_float64_oracle_on_degenerate_boxes(name, algo):
    box, m, reso, sg, mp = _degenerate_cases()[name]
    o = OG.plan(algo, box, m, reso, sg, max_pts=mp)
    check_plan(algo, box, m, reso, sg, o, mp)
    _check_degenerate(name, algo, o)


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("max_pts", MAZE_MAX_PTS)
def test_checker_meets_float64_oracle_in_a_maze(max_pts, algo):
    box, m, reso, sg, mp = _maze_case(max_pts)
    o = OG.plan(algo, box, m, reso, sg, max_pts=mp)
    check_plan(algo, box, m, reso, sg, o, mp)
    assert (o["status"] == OG.FOUND).all() and o["path_len"][:2].min() > 10 ** 4


@pytest.mark.parametrize("algo", ALGO_IDS)
def test_checker_any_nonzero_map_byte_blocks(algo):
    for name in ("tall_17x61", "winding_70x45"):
        box, m, reso, sg = _box_plan_case(name, 257)
        mb = _bytes_map(m, 0xB7)
        assert set(np.unique(mb).tolist()) == {0, *GC.MAP_BYTES}
        o = OG.plan(algo, box, m, reso, sg, max_pts=MAX_PTS)
        _bitwise(OG.plan(algo, box, mb, reso, sg, max_pts=MAX_PTS), o)
        check_plan(algo, box, mb, reso, sg, o, MAX_PTS)


@pytest.mark.parametrize("name", MAP_NAMES)
def test_checker_map_meets_float64_rule(name):
    ox, oy, reso, rr, box = _map_case(name)
    want = map64(ox, oy, reso, rr, box)
    assert np.array_equal(OG.obstacle_map(ox, oy, reso, rr, box) != 0, want)


def test_map_rr_cases_straddle_the_diagonal():
    """rr = reso * (float)sqrt(2) blocks an obstacle's diagonal neighbour at reso 1, its predecessor does not"""
    box = np.int32([0, 0, 3, 3])
    o = F([1.0])
    assert map64(o, o, 1.0, float(DIAG), box).all()
    m = map64(o, o, 1.0, float(np.nextafter(DIAG, F(0))), box)
    assert m.sum() == 5 and not m[0, 0] and m[1, 1]
    assert map64(o, o, 1.0, -0.0, box).sum() == 1 and not map64(o, o, 1.0, -1e-30, box).any()
    # and the box cases at reso 1 meet that boundary
    assert map64(*_map_case("unit_n513_diag")).sum() > map64(*_map_case("unit_n513_below_diag")).sum()


# ---- CPU: the checker against the reference text on the new square cases ----------------------------------------
@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("case", [c[0] for c in GC.square_cases()])
def test_square_cases_are_bitwise_the_reference_text(algo, case):
    L = GC.ref_lib(algo)
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle -f grid.mk)")
    _, ox, oy, reso, rr, sx, sy, gx, gy = next(c for c in GC.square_cases() if c[0] == case)
    box = OG.box_of_obstacles(ox, oy, reso)
    m = OG.obstacle_map(ox, oy, reso, rr, box)
    r = OG.plan(algo, box, m, reso, np.float32([[sx], [sy], [gx], [gy]]), max_pts=1 << 12)
    assert GC.check_ref_domain(algo, box, r["status"][0]), (box, r["status"])
    ref = GC.ref_run(L, sx, sy, gx, gy, ox, oy, reso, rr)
    assert np.array_equal(np.argwhere(m != 0), ref["map_cells"])
    assert np.array_equal(OG.trace(algo, box, m, reso, sx, sy, gx, gy), ref["trace"])
    n = int(r["path_len"][0])
    assert n == len(ref["path"])
    assert same(r["path"][:2 * n, 0].reshape(n, 2), ref["path"].astype(F) * F(reso))
    assert np.array_equal(m != 0, map64(ox, oy, reso, rr, box))


# ---- H100: the kernels against the checker, bitwise, and the float64 oracle --------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("name", BOX_NAMES)
def test_gpu_plan_on_boxes(engine, name, n, algo):
    box, m, reso, sg = _box_plan_case(name, n)
    r = _gpu_plan(engine, algo, box, m, reso, sg, MAX_PTS)
    _bitwise(r, OG.plan(algo, box, m, reso, sg, max_pts=MAX_PTS))
    counts = check_plan(algo, box, m, reso, sg, r, MAX_PTS)
    if n == 4097:
        assert (counts > 0).all(), counts


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
def test_gpu_plan_at_int_range_ends_points_and_degenerate_boxes(engine, algo):
    for name, (_, box, m, sg) in GC.int_end_cases().items():
        r = _gpu_plan(engine, algo, box, m, 1.0, sg, 1024)
        _bitwise(r, OG.plan(algo, box, m, 1.0, sg, max_pts=1024))
        assert (check_plan(algo, box, m, 1.0, sg, r, 1024) > 0).all(), name
    for name, *_ in POINT_CASES:
        box, m, reso, sg = _point_case(name)
        r = _gpu_plan(engine, algo, box, m, reso, sg, 512)
        _bitwise(r, OG.plan(algo, box, m, reso, sg, max_pts=512))
        check_plan(algo, box, m, reso, sg, r, 512)
        _check_points(box, reso, sg, r)
    for name, (box, m, reso, sg, mp) in _degenerate_cases().items():
        r = _gpu_plan(engine, algo, box, m, reso, sg, mp)
        _bitwise(r, OG.plan(algo, box, m, reso, sg, max_pts=mp))
        check_plan(algo, box, m, reso, sg, r, mp)
        _check_degenerate(name, algo, r)
    for mp in MAZE_MAX_PTS:
        box, m, reso, sg, _ = _maze_case(mp)
        r = _gpu_plan(engine, algo, box, m, reso, sg, mp)
        _bitwise(r, OG.plan(algo, box, m, reso, sg, max_pts=mp))
        check_plan(algo, box, m, reso, sg, r, mp)
        assert r["path_len"][:2].min() > 10 ** 4


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
def test_gpu_any_nonzero_map_byte_blocks(engine, algo):
    for name in ("tall_17x61", "winding_70x45"):
        box, m, reso, sg = _box_plan_case(name, 4097)
        o = OG.plan(algo, box, m, reso, sg, max_pts=MAX_PTS)
        _bitwise(_gpu_plan(engine, algo, box, _bytes_map(m, 0xB7), reso, sg, MAX_PTS), o)


def _check_max(algo, name, box, m, reso, sg, r):
    o = OG.plan(algo, box, m, reso, sg, max_pts=512)
    _bitwise(r, o)
    check_plan(algo, box, m, reso, sg, r, 512, d64=False)
    st = r["status"].tolist()
    assert st[:-1] == [OG.FOUND] * (len(st) - 1) and st[-1] == OG.NO_PATH and r["n_visited"][-1] == 64, (name, st)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("name", list(GC.MAX_BOXES))
def test_gpu_plan_at_max_cells(engine, name, algo):
    box, m, reso, sg = GC.max_case(name)
    slots = engine.grid_plan_slots(algo, _box(box), 1 << 20)
    assert slots == 3
    sg = np.ascontiguousarray(sg[:, np.arange(2 * slots + 1) % sg.shape[1]])
    r = _gpu_plan(engine, algo, box, m, reso, sg, 512)
    _check_max(algo, name, box, m, reso, sg, r)


@pytest.mark.gpu
def test_gpu_workspace_reuse_across_planners_and_sizes(engine):
    """A max-cells A* call, a small Dijkstra call, a max-cells Dijkstra call, a small A* call on one engine: stale
    slot state, or a slot layout of one planner used for the other, changes some bit."""
    big = GC.max_case("max_4096x4096")
    small = _box_plan_case("wide_61x17", 4097)
    for algo, (box, m, reso, sg) in ((OG.ASTAR, big), (OG.DIJKSTRA, small), (OG.DIJKSTRA, big), (OG.ASTAR, small)):
        r = _gpu_plan(engine, algo, box, m, reso, sg, 512)
        if sg.shape[1] == 7:
            _check_max(algo, "max_4096x4096", box, m, reso, sg, r)
        else:
            _bitwise(r, OG.plan(algo, box, m, reso, sg, max_pts=512))


@pytest.mark.gpu
def test_gpu_obstacle_map_on_boxes(engine):
    for name, ox, oy, reso, rr, box in MAP_CASES:
        want = OG.obstacle_map(ox, oy, reso, rr, box)
        assert np.array_equal(_gpu_map(engine, ox, oy, reso, rr, box), want), name
        assert np.array_equal(want != 0, map64(ox, oy, reso, rr, box)), name
    # at CRB_GRID_MAX_CELLS, 300 obstacles (the checker's cost is cells x obstacles)
    rng = np.random.default_rng(0x300)
    box = np.int32([-20000, 77, 12768, 589])
    cx = rng.integers(-20010, 12778, 300) + rng.choice([0.0, 0.5], 300)
    cy = rng.integers(67, 599, 300) + rng.choice([0.0, -0.5], 300)
    ox, oy = F(cx) * F(0.7), F(cy) * F(0.7)
    rr = float(F(3.3) * F(0.7))
    want = OG.obstacle_map(ox, oy, 0.7, rr, box)
    assert want.shape == (32768, 512) and want.any()
    assert np.array_equal(_gpu_map(engine, ox, oy, 0.7, rr, box), want)
