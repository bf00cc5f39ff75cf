"""The grid checker (oracle/grid.py) composed map by map, for crb_grid_obstacle_map_many and
crb_grid_plan_many_batched: every map of a table built, and every query planned, by the unchanged single-map checker.

TEST INFRASTRUCTURE ONLY, like oracle/grid.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import numpy as np

from . import grid as OG

# include/crb.h
BAD_MAP = 4
MAP_OK, MAP_BAD = 0, 1


def entry_ok(boxes, reso, map_off, n_cells, max_cells, m):
    """Whether table entry m is valid (crb.h): index, box limits, W * H <= max_cells, offsets, reso."""
    if not 0 <= m < len(reso):
        return False
    b = [int(v) for v in boxes[m]]
    W, H = b[2] - b[0], b[3] - b[1]
    if W < 1 or H < 1 or W > OG.MAX_SIDE or H > OG.MAX_SIDE or W * H > max_cells:
        return False
    lo, hi = int(map_off[m]), int(map_off[m + 1])
    if lo < 0 or hi < lo or hi > n_cells or hi - lo != W * H:
        return False
    r = np.float32(reso[m])
    return bool(np.isfinite(r) and r > 0)


def obstacle_map_many(ob, ob_off, ob_of, rr, boxes, reso, map_off, n_cells, max_cells, maps=None):
    """calc_obstacle_map for every map: map m from rows [ob_off[s], ob_off[s + 1]) of ob [n_rows, 2], s = ob_of[m], with
    reso[m] and rr[m].  Returns (maps uint8 [n_cells], status int32 [n_maps]); a BAD map's bytes keep the values of
    `maps` (zeros when not given)."""
    ob = np.asarray(ob, np.float32).reshape(-1, 2)
    out = np.zeros(n_cells, np.uint8) if maps is None else np.array(maps, np.uint8)
    n_maps = len(reso)
    status = np.full(n_maps, MAP_BAD, np.int32)
    for m in range(n_maps):
        if not entry_ok(boxes, reso, map_off, n_cells, max_cells, m) or not np.isfinite(np.float32(rr[m])):
            continue
        s = int(ob_of[m])
        if not 0 <= s < len(ob_off) - 1:
            continue
        lo, hi = int(ob_off[s]), int(ob_off[s + 1])
        if lo < 0 or hi < lo or hi > len(ob):
            continue
        out[int(map_off[m]):int(map_off[m + 1])] = OG.obstacle_map(ob[lo:hi, 0], ob[lo:hi, 1], reso[m], rr[m],
                                                                   boxes[m]).reshape(-1)
        status[m] = MAP_OK
    return out, status


def plan_many(algo, boxes, reso, map_off, maps, max_cells, map_of, sg, max_pts=0, path_fill=np.nan, nthreads=0):
    """The planners for sg [4, n], query q on map map_of[q] of the table: oracle.grid.plan once per map on its own
    queries, scattered back.  A query on an invalid entry gets BAD_MAP, path_len 0, cost NaN, n_visited 0 and an
    untouched path column (path_fill)."""
    sg = np.asarray(sg, np.float32)
    map_of = np.asarray(map_of, np.int32)
    maps = np.asarray(maps, np.uint8)
    n = sg.shape[1]
    out = dict(path=np.full((2 * max_pts, n), path_fill, np.float32), path_len=np.zeros(n, np.int32),
               cost=np.full(n, np.nan, np.float32), n_visited=np.zeros(n, np.int32),
               status=np.full(n, BAD_MAP, np.int32))
    order = np.argsort(map_of, kind="stable")
    sm = map_of[order]
    for m in np.unique(map_of):
        sel = order[np.searchsorted(sm, m, "left"):np.searchsorted(sm, m, "right")]
        if not entry_ok(boxes, reso, map_off, maps.size, max_cells, int(m)):
            continue
        W, H = OG.dims(boxes[m])
        r = OG.plan(algo, boxes[m], maps[int(map_off[m]):int(map_off[m + 1])].reshape(W, H), reso[m],
                    np.ascontiguousarray(sg[:, sel]), max_pts=max_pts, path_fill=path_fill, nthreads=nthreads)
        for k in out:
            out[k][..., sel] = r[k]
    return out
