"""Grid planning with a map per query: crb_grid_obstacle_map_many and crb_grid_plan_many_batched.

Every valid map must be bitwise crb_grid_obstacle_map on its own inputs, and every query's outputs bitwise those of
crb_grid_plan_batched run on its own map, and so those of the checker composed map by map (oracle/grid_many.py).
CPU: argument validation without a device, grid_map_table and the synth helpers, the composed checker on one map, the
compiler report and the C++ program.
H100 (-m gpu): maps at n_maps = 1, 7 and 1024; plans at n = 1 to 65536 in random order over them, both planners, with
max_pts 0, truncating and long; every way a table entry can be bad; NULL outputs, n = 0, graph capture, a workspace
shared with the single-map planner; a local-window fleet; the C++ program against the checker."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from cpprobotics_b200 import _lib, grid_map_table, synth
from oracle import grid as OG
from oracle import grid_many as GM
from toolchain import build_ref_program, kernel_sass_hashes, ptxas_kernels

INV = -1
KEYS = ("path", "path_len", "cost", "n_visited", "status")


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def fleet(n_maps, seed=0x6F1E):
    """grid_fleet_maps plus maps at reso 1e-3 and 1e3 (when there is room), with the table and the checker's maps."""
    f = synth.grid_fleet_maps(n_maps, seed=seed)
    if n_maps >= 7:
        f["lists"].append(np.float32([[0.0, 0.0], [0.01, 0.02], [0.02, 0.01], [0.03, 0.03]]))
        f["lists"].append(np.float32([[0.0, 0.0], [4000.0, 2000.0], [9000.0, 9000.0]]))
        f["ob_of"][-2:] = len(f["lists"]) - 2, len(f["lists"]) - 1
        f["boxes"][-2:] = (-2, -3, 40, 37), (0, 0, 10, 9)
        f["reso"][-2:] = 1e-3, 1e3
        f["rr"][-2:] = 2e-3, 1.5e3
    table = grid_map_table(f["boxes"], f["reso"])
    ob, off = synth.pack_obstacles(f["lists"], 2)
    maps, st = GM.obstacle_map_many(ob, off, f["ob_of"], f["rr"], *table[:3], int(table[2][-1]), table[3])
    assert (st == GM.MAP_OK).all()
    return f, table, (ob, off), maps


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is refused with CRB_ERR_INVALID_ARG before any device work; a valid call says
    CRB_ERR_NO_DEVICE on a machine without a GPU."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)
    big = _lib.CRB_GRID_MAX_CELLS

    def omap(**over):
        a = dict(dict(ctx=ctx, ob=d, rows=40, off=d, ns=3, of=d, rr=d, boxes=d, reso=d, moff=d, nm=5, nc=100, mc=20,
                      maps=d, st=d), **over)
        return L.crb_grid_obstacle_map_many(a["ctx"], a["ob"], a["rows"], a["off"], a["ns"], a["of"], a["rr"],
                                            a["boxes"], a["reso"], a["moff"], a["nm"], a["nc"], a["mc"], a["maps"],
                                            a["st"])

    def plan(**over):
        a = dict(dict(ctx=ctx, algo=0, boxes=d, reso=d, moff=d, nm=5, maps=d, nc=100, mc=20, n=7, of=d, sg=d, mp=4,
                      path=d), **over)
        return L.crb_grid_plan_many_batched(a["ctx"], a["algo"], a["boxes"], a["reso"], a["moff"], a["nm"], a["maps"],
                                            a["nc"], a["mc"], a["n"], a["of"], a["sg"], a["mp"], a["path"], d, d, d, d)

    def slots(**over):
        a = dict(dict(ctx=ctx, algo=1, mc=20, n=7, out=C.byref(C.c_int64())), **over)
        return L.crb_grid_plan_many_slots(a["ctx"], a["algo"], a["mc"], a["n"], a["out"])

    scal = (dict(nm=0), dict(nm=-1), dict(nc=-1), dict(mc=0), dict(mc=big + 1), dict(mc=-5))
    for kw in scal + (dict(ctx=None), dict(ns=0), dict(rows=-1), dict(ob=None), dict(off=None), dict(of=None),
                      dict(rr=None), dict(boxes=None), dict(reso=None), dict(moff=None), dict(maps=None)):
        assert omap(**kw) == INV, kw
    for kw in scal + (dict(ctx=None), dict(algo=2), dict(algo=-1), dict(n=-1), dict(n=(1 << 62) + 1), dict(mp=-1),
                      dict(n=1 << 40, mp=1 << 23), dict(boxes=None), dict(reso=None), dict(moff=None), dict(of=None),
                      dict(sg=None), dict(maps=None), dict(path=None)):
        assert plan(**kw) == INV, kw
    for kw in (dict(ctx=None), dict(out=None), dict(algo=2), dict(n=-1), dict(mc=0), dict(mc=big + 1)):
        assert slots(**kw) == INV, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert omap() == nd and omap(ob=None, rows=0) == nd and omap(maps=None, nc=0) == nd and omap(st=None) == nd
        assert omap(mc=big) == nd
        assert plan() == nd and plan(path=None, mp=0) == nd and plan(maps=None, nc=0) == nd
        assert plan(n=0, boxes=None, reso=None, moff=None, of=None, sg=None, maps=None, path=None) == nd
        assert slots() == nd and slots(mc=big, algo=0) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def test_map_table_offsets_are_the_cumulative_cells():
    boxes = np.int32([[0, 0, 60, 60], [-5, 7, -4, 8], [3, -9, 20, 40], [-32768, 0, 0, 512]])
    b, r, off, mc = grid_map_table(boxes, [1.0, 0.5, 2.0, 1e-3])
    W, H = boxes[:, 2] - boxes[:, 0], boxes[:, 3] - boxes[:, 1]
    assert b.dtype == np.int32 and same(b, boxes) and r.dtype == np.float32 and r.shape == (4,)
    assert off.dtype == np.int64 and off.tolist() == [0] + np.cumsum(W.astype(np.int64) * H).tolist()
    assert mc == 32768 * 512
    for bad in ([[0, 0, 0, 5]], [[3, 0, 2, 5]], [[0, 0, 32769, 1]], [[0, 0, 4097, 4096]]):
        with pytest.raises(ValueError):
            grid_map_table(bad, [1.0])
    with pytest.raises(ValueError):
        grid_map_table(boxes, [1.0])


def test_fleet_helpers_are_varied_and_deterministic():
    a, b = synth.grid_fleet_maps(200, seed=9), synth.grid_fleet_maps(200, seed=9)
    assert all(same(x, y) for x, y in zip(a["lists"], b["lists"])) and len(a["lists"]) == len(b["lists"])
    for k in ("ob_of", "boxes", "reso", "rr"):
        assert same(a[k], b[k]), k
    W, H = a["boxes"][:, 2] - a["boxes"][:, 0], a["boxes"][:, 3] - a["boxes"][:, 1]
    assert (W * H == 1).sum() >= 20 and (W != H).sum() > 100 and (a["boxes"][:, :2] < 0).any()
    assert (W * H % 256 != 0).mean() > 0.9 and (W * H > 256).any()
    assert a["reso"].min() < 0.03 and a["reso"].max() > 30 and (a["reso"] <= 100).all()
    assert len(np.unique(a["rr"] / a["reso"])) >= 4 and np.bincount(a["ob_of"]).max() >= 3
    assert any(len(x) == 0 for x in a["lists"]) and len({len(x) for x in a["lists"]}) > 20
    w = synth.grid_local_windows(300, side=200, win=64)
    assert (w["ob_of"] == 0).all() and len(w["lists"]) == 1 and w["boxes"].shape == (300, 4)
    assert ((w["boxes"][:, 2:] - w["boxes"][:, :2]) == 64).all() and w["boxes"].min() >= 0 and w["boxes"].max() <= 200
    assert same(w["boxes"], synth.grid_local_windows(300, side=200, win=64)["boxes"])
    f, table, _, maps = fleet(40)
    mo, sg = synth.grid_fleet_inputs(3000, table[0], table[1], maps, table[2], seed=4)
    mo2, sg2 = synth.grid_fleet_inputs(3000, table[0], table[1], maps, table[2], seed=4)
    assert same(mo, mo2) and same(sg, sg2) and mo.dtype == np.int32 and sg.shape == (4, 3000)
    assert len(np.unique(mo)) == 40 and not (np.diff(mo) >= 0).all() and np.isnan(sg).any()


def test_composed_checker_on_one_map_is_the_checker():
    ox, oy = synth.grid_demo_obstacles()
    gb = OG.box_of_obstacles(ox, oy, 1.0)
    m = OG.obstacle_map(ox, oy, 1.0, 1.0, gb)
    table = grid_map_table(gb[None], [1.0])
    mm, st = GM.obstacle_map_many(np.stack([ox, oy], 1), np.int64([0, ox.size]), np.int32([0]), np.float32([1.0]),
                                  *table[:3], m.size, table[3])
    assert st.tolist() == [0] and same(mm, m.reshape(-1))
    sg = synth.grid_inputs(300, gb, m, 1.0, seed=3)
    for algo in (OG.ASTAR, OG.DIJKSTRA):
        a = GM.plan_many(algo, *table[:3], mm, table[3], np.zeros(300, np.int32), sg, max_pts=40)
        b = OG.plan(algo, gb, m, 1.0, sg, max_pts=40)
        assert all(same(a[k], b[k]) for k in KEYS)


# sha256 of each single-map kernel's SASS (cuobjdump -sass, NVCC_FLAGS, CUDA 12.9) as they were before the many-map
# planner existed: moving their shared code into crb_grid_common.cuh must not change one instruction
SINGLE_MAP_SASS = {
    "_Z20crb_grid_plan_kernelILi1EEv12GridPlanArgs": "8dcae465b0b6eca72f0f08f73b6cb3032f38a9e90ddc3a123bc713eeb32fa775",
    "_Z20crb_grid_plan_kernelILi0EEv12GridPlanArgs": "824569cb039ba70b9c09ce18a3994efed167a975ec029f5cf6d6d244636cac46",
    "_Z19crb_grid_map_kernellPKfS0_ff12crb_grid_boxlPh":
        "e00c03e2ae961fa85b5911adf450a057cfafda3228e6a3b181074fa899ddd170",
}


def test_many_map_kernels_do_not_spill():
    kernels = ptxas_kernels("crb_grid_many.cu")
    assert sorted(kernels) == ["_Z24crb_grid_map_many_kernel11GridMapArgs",
                               "_Z25crb_grid_plan_many_kernelILi0EEv16GridPlanManyArgs",
                               "_Z25crb_grid_plan_many_kernelILi1EEv16GridPlanManyArgs"], kernels
    for f in kernels.values():
        assert (f.stack, f.spill_stores, f.spill_loads) == (0, 0, 0) and f.registers <= 56, f


def test_single_map_kernels_keep_their_machine_code():
    assert kernel_sass_hashes("crb_grid.cu") == SINGLE_MAP_SASS


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "grid_many_ref_api.cpp")


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _dtable(table):
    return tuple(_dev(a) for a in table[:3]) + (table[3],)


@pytest.fixture(scope="module")
def engine():
    from cpprobotics_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def gpu_maps(engine, f, table, store, sentinel=None):
    dob, doff = _dev(store[0]), _dev(store[1])
    n_cells = int(table[2][-1])
    import torch
    maps = torch.full((n_cells,), 0x5A if sentinel is None else sentinel, dtype=torch.uint8, device="cuda:0")
    maps, st = engine.grid_obstacle_map_many((dob, doff), _dev(f["ob_of"]), _dev(f["rr"]), _dtable(table), maps=maps)
    return maps.cpu().numpy(), st.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("n_maps", [1, 7, 1024])
def test_maps_are_the_single_map_builder_and_the_checker(engine, n_maps):
    f, table, store, want = fleet(n_maps, seed=0x600 + n_maps)
    got, st = gpu_maps(engine, f, table, store)
    assert (st == GM.MAP_OK).all() and same(got, want)
    ob, off = store
    for m in range(n_maps) if n_maps < 1024 else range(0, 1024, 37):
        s = f["ob_of"][m]
        lo, hi = int(off[s]), int(off[s + 1])
        box = _lib.GridBox(*[int(v) for v in f["boxes"][m]])
        one = engine.grid_obstacle_map(_dev(ob[lo:hi, 0]), _dev(ob[lo:hi, 1]), float(f["reso"][m]), float(f["rr"][m]),
                                       box)
        assert same(one.cpu().numpy().reshape(-1), got[table[2][m]:table[2][m + 1]]), m


def per_map_gpu(engine, algo, table, maps, map_of, sg, max_pts, fill=7.0):
    """crb_grid_plan_batched once per map on its own queries, scattered back"""
    import torch
    boxes, reso, off, _ = table
    n = sg.shape[1]
    out = dict(path=np.full((2 * max_pts, n), fill, np.float32), path_len=np.zeros(n, np.int32),
               cost=np.zeros(n, np.float32), n_visited=np.zeros(n, np.int32), status=np.zeros(n, np.int32))
    for m in np.unique(map_of):
        sel = np.nonzero(map_of == m)[0]
        W, H = OG.dims(boxes[m])
        path = torch.full((2 * max_pts, sel.size), fill, device="cuda:0") if max_pts else None
        r = engine.grid_plan(algo, _lib.GridBox(*[int(v) for v in boxes[m]]),
                             _dev(maps[off[m]:off[m + 1]].reshape(W, H)), float(reso[m]), _dev(sg[:, sel]),
                             max_pts=max_pts, path=path)
        for k in KEYS:
            if r[k] is not None:
                out[k][..., sel] = r[k].cpu().numpy()
    return out


def gpu_many(engine, algo, table, maps, map_of, sg, max_pts, fill=7.0):
    import torch
    n = sg.shape[1]
    path = torch.full((2 * max_pts, n), fill, device="cuda:0") if max_pts else None
    r = engine.grid_plan_many(algo, _dtable(table), _dev(maps), _dev(map_of), _dev(sg), max_pts=max_pts, path=path)
    out = {k: (v.cpu().numpy() if v is not None else np.full((0, n), fill, np.float32)) for k, v in r.items()}
    return out


@pytest.fixture(scope="module")
def fleet1024():
    return fleet(1024, seed=0x1024)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", [OG.ASTAR, OG.DIJKSTRA])
@pytest.mark.parametrize("n,max_pts", [(1, 0), (33, 3), (4097, 256), (65536, 24)])
def test_plans_are_the_single_map_planner_and_the_checker(engine, fleet1024, algo, n, max_pts):
    f, table, store, maps = fleet1024
    map_of, sg = synth.grid_fleet_inputs(n, table[0], table[1], maps, table[2], seed=n)
    got = gpu_many(engine, algo, table, maps, map_of, sg, max_pts)
    ref = per_map_gpu(engine, algo, table, maps, map_of, sg, max_pts)
    chk = GM.plan_many(algo, *table[:3], maps, table[3], map_of, sg, max_pts=max_pts, path_fill=7.0)
    for k in KEYS:
        assert same(got[k], ref[k]), k
        assert same(got[k], chk[k]), k
    if n >= 4097:
        assert len(np.unique(got["status"])) == 4       # found, no path, start outside and bad point all occur
        assert max_pts == 256 or (got["path_len"] > max_pts).any()


def bad_tables():
    """(name, boxes, reso, map_off, n_cells, max_cells, map index) for every way an entry can fail; entries 0 and 2
    stay valid (the 4 x 5 and 3 x 3 maps of the base table)"""
    boxes = np.int32([[0, 0, 4, 5], [2, 2, 8, 8], [-3, -3, 0, 0]])
    reso = np.float32([1.0, 1.0, 1.0])
    off = np.int64([0, 20, 56, 65])
    out = []

    def case(name, m=1, b=None, r=None, o=None, nc=65, mc=36):
        out.append((name, boxes if b is None else b, reso if r is None else r, off if o is None else o, nc, mc, m))
    case("index below range", m=-1)
    case("index above range", m=3)
    case("empty box", b=np.int32([[0, 0, 4, 5], [2, 2, 2, 8], [-3, -3, 0, 0]]))
    case("box over the side limit", b=np.int32([[0, 0, 4, 5], [0, 0, 32769, 1], [-3, -3, 0, 0]]), mc=1 << 24)
    case("W * H over max_cells", mc=35)
    case("map_off below 0", o=np.int64([0, -1, 56, 65]))
    case("map_off span not W * H", o=np.int64([0, 21, 56, 65]))
    case("map_off past n_cells", m=2, nc=64)
    case("map_off span not W * H for the last map", m=2, o=np.int64([0, 20, 56, 64]))
    case("reso zero", r=np.float32([1.0, 0.0, 1.0]))
    case("reso NaN", r=np.float32([1.0, np.nan, 1.0]))
    case("reso inf", r=np.float32([1.0, np.inf, 1.0]))
    return out


@pytest.mark.gpu
def test_bad_entries_give_bad_map_and_leave_neighbours_alone(engine):
    import torch
    ob = np.float32([[1.0, 1.0], [3.0, 4.0], [-2.0, -2.0], [5.0, 5.0]])
    for name, boxes, reso, off, nc, mc, m in bad_tables():
        table = (boxes, reso, off, mc)
        ob_of = np.int32([0, 0, 0])
        rr = np.float32([1.0, 1.0, 1.0])
        dmaps = torch.full((max(nc, 65),), 0xA5, dtype=torch.uint8, device="cuda:0")[:nc]
        st = engine.grid_obstacle_map_many((_dev(ob), _dev(np.int64([0, 4]))), _dev(ob_of), _dev(rr), _dtable(table),
                                           maps=dmaps)[1].cpu().numpy()
        hm = dmaps.cpu().numpy()
        want, wst = GM.obstacle_map_many(ob, np.int64([0, 4]), ob_of, rr, boxes, reso, off, nc, mc,
                                         maps=np.full(nc, 0xA5, np.uint8))
        assert same(st, wst) and same(hm, want), name
        assert st[1] == GM.MAP_BAD or m != 1, name
        for k in np.flatnonzero(st == GM.MAP_BAD):      # a refused map's bytes are untouched
            assert (hm[max(0, off[k]):max(0, min(off[k + 1], nc))] == 0xA5).all(), name
        for k in range(3):      # every valid entry is built, whatever its neighbours hold
            assert (st[k] == GM.MAP_OK) == (GM.entry_ok(boxes, reso, off, nc, mc, k)), (name, k)
        # the planner: queries on every map, the bad one and its neighbours
        base = np.zeros(65, np.uint8)
        sg = np.float32([[1, 3, 4, -2, 1, 2], [1, 4, 4, -2, 2, 3], [3, 7, 6, -1, 3, 1], [4, 6, 5, -1, 0, 1]])
        map_of = np.int32([0, m, m, 2, 0, m])
        if m == 1:
            sg[2, 2] = np.nan      # BAD_MAP wins over BAD_POINT
        for algo in (OG.ASTAR, OG.DIJKSTRA):
            got = gpu_many(engine, algo, table, base[:nc], map_of, sg, 8)
            chk = GM.plan_many(algo, boxes, reso, off, base[:nc], mc, map_of, sg, max_pts=8, path_fill=7.0)
            for k in KEYS:
                assert same(got[k], chk[k]), (name, k)
            bad = map_of == m
            assert (got["status"][bad] == _lib.CRB_GRID_BAD_MAP).all() and (got["path_len"][bad] == 0).all()
            assert np.isnan(got["cost"][bad]).all() and (got["n_visited"][bad] == 0).all()
            valid = np.array([GM.entry_ok(boxes, reso, off, nc, mc, int(k)) for k in map_of])
            assert (got["path"][:, bad] == 7.0).all() and (got["status"][valid] == OG.FOUND).all(), name
            assert (got["status"][~valid] == _lib.CRB_GRID_BAD_MAP).all(), name
    # the builder's own failures: a non-finite rr and bad list references
    table = grid_map_table(np.int32([[0, 0, 4, 5], [2, 2, 8, 8], [-3, -3, 0, 0]]), [1.0, 1.0, 1.0])
    for name, rr, ob_of, ob_off in (("rr NaN", [1, np.nan, 1], [0, 0, 0], [0, 4]),
                                    ("rr inf", [1, np.inf, 1], [0, 0, 0], [0, 4]),
                                    ("list index out of range", [1, 1, 1], [0, 1, 0], [0, 4]),
                                    ("list index negative", [1, 1, 1], [0, -1, 0], [0, 4]),
                                    ("list past n_rows", [1, 1, 1], [0, 1, 0], [0, 4, 9]),
                                    ("list offsets decreasing", [1, 1, 1], [0, 1, 0], [0, 4, 2])):
        rr, ob_of, ob_off = np.float32(rr), np.int32(ob_of), np.int64(ob_off)
        dmaps = torch.full((65,), 0xA5, dtype=torch.uint8, device="cuda:0")
        st = engine.grid_obstacle_map_many((_dev(ob), _dev(ob_off)), _dev(ob_of), _dev(rr), _dtable(table),
                                           maps=dmaps)[1].cpu().numpy()
        hm = dmaps.cpu().numpy()
        assert st.tolist() == [0, 1, 0] and (hm[20:56] == 0xA5).all(), name
        want, _ = GM.obstacle_map_many(ob, np.int64([0, 4]), np.int32([0, 0, 0]), np.float32([1, 1, 1]), *table[:3],
                                       65, table[3])
        assert same(hm[:20], want[:20]) and same(hm[56:], want[56:]), name


@pytest.mark.gpu
def test_launch_forms(engine):
    import torch
    f, table, store, maps = fleet(7, seed=0x77)
    map_of, sg = synth.grid_fleet_inputs(500, table[0], table[1], maps, table[2], seed=5)
    dt, dm = _dtable(table), _dev(maps)
    full = gpu_many(engine, OG.ASTAR, table, maps, map_of, sg, 16)
    # NULL outputs: only status, then nothing at all
    st = torch.empty(500, dtype=torch.int32, device="cuda:0")
    L = engine.lib
    dof, dsg = _dev(map_of), _dev(sg)
    args = lambda n, st_ptr: (engine.ctx, OG.ASTAR, dt[0].data_ptr(), dt[1].data_ptr(), dt[2].data_ptr(), 7,  # noqa
                              dm.data_ptr(), dm.numel(), table[3], n, dof.data_ptr(), dsg.data_ptr(), 0,
                              None, None, None, None, st_ptr)
    assert L.crb_grid_plan_many_batched(*args(500, st.data_ptr())) == 0
    assert L.crb_grid_plan_many_batched(*args(500, None)) == 0
    torch.cuda.synchronize()
    assert same(st.cpu().numpy(), full["status"])
    assert engine.grid_obstacle_map_many((_dev(store[0]), _dev(store[1])), _dev(f["ob_of"]), _dev(f["rr"]), dt,
                                         maps=torch.zeros_like(dm), map_status=None) is not None
    keep = [_dev(store[0]), _dev(store[1]), _dev(f["ob_of"]), _dev(f["rr"]), torch.zeros_like(dm)]
    assert L.crb_grid_obstacle_map_many(engine.ctx, keep[0].data_ptr(), store[0].shape[0], keep[1].data_ptr(),
                                        len(store[1]) - 1, keep[2].data_ptr(), keep[3].data_ptr(), dt[0].data_ptr(),
                                        dt[1].data_ptr(), dt[2].data_ptr(), 7, dm.numel(), table[3],
                                        keep[4].data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert same(keep[4].cpu().numpy(), maps)
    # n = 0 with maps and no queries, and no pointers at all
    assert L.crb_grid_plan_many_batched(*args(0, None)) == 0
    assert L.crb_grid_plan_many_batched(engine.ctx, 1, None, None, None, 7, None, 0, 5, 0, None, None, 0, None, None,
                                        None, None, None) == 0
    # the workspace shared with the single-map planner, in either order, then graph capture once it exists
    W, H = OG.dims(table[0][0])
    sel = np.nonzero(map_of == 0)[0]
    one = lambda: engine.grid_plan(OG.ASTAR, _lib.GridBox(*[int(v) for v in table[0][0]]),  # noqa: E731
                                   _dev(maps[:W * H].reshape(W, H)), float(table[1][0]), _dev(sg[:, sel]), max_pts=16,
                                   path=torch.full((32, sel.size), 7.0, device="cuda:0"))
    r1 = {k: v.cpu().numpy() for k, v in one().items()}
    assert all(same(r1[k], full[k][..., sel]) for k in KEYS)
    again = gpu_many(engine, OG.ASTAR, table, maps, map_of, sg, 16)
    r2 = {k: v.cpu().numpy() for k, v in one().items()}
    assert all(same(again[k], full[k]) and same(r2[k], r1[k]) for k in KEYS)
    outs = dict(path=torch.full((32, 500), 7.0, device="cuda:0"), path_len=torch.zeros(500, dtype=torch.int32,
                device="cuda:0"), cost=torch.zeros(500, device="cuda:0"),
                n_visited=torch.zeros(500, dtype=torch.int32, device="cuda:0"),
                status=torch.zeros(500, dtype=torch.int32, device="cuda:0"))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        engine.bind_current_stream()
        engine.grid_plan_many(OG.ASTAR, dt, dm, dof, dsg, max_pts=16, **outs)   # the workspace exists after this
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            engine.grid_plan_many(OG.ASTAR, dt, dm, dof, dsg, max_pts=16, **outs)
        for k, v in outs.items():      # the path's tail past path_len is left as it is: keep its fill
            v.fill_(7.0 if k == "path" else 0)
        g.replay()
        s.synchronize()
    engine.bind_current_stream()
    assert all(same(outs[k].cpu().numpy(), full[k]) for k in KEYS)


@pytest.mark.gpu
def test_local_windows_against_the_checker(engine):
    w = synth.grid_local_windows(2048, side=160, win=64)
    table = grid_map_table(w["boxes"], w["reso"])
    store = synth.pack_obstacles(w["lists"], 2)
    maps, st = gpu_maps(engine, w, table, store)
    assert (st == 0).all()
    ob = store[0]
    for m in range(0, 2048, 97):
        want = OG.obstacle_map(ob[:, 0], ob[:, 1], 1.0, 1.0, w["boxes"][m])
        assert same(maps[table[2][m]:table[2][m + 1]], want.reshape(-1)), m
    map_of = np.arange(2048, dtype=np.int32)
    sg = np.zeros((4, 2048), np.float32)
    for m in range(2048):
        sg[:, m:m + 1] = synth.grid_inputs(1, w["boxes"][m], maps[table[2][m]:table[2][m + 1]].reshape(64, 64), 1.0,
                                           seed=m)
    for algo in (OG.ASTAR, OG.DIJKSTRA):
        got = gpu_many(engine, algo, table, maps, map_of, sg, 32)
        chk = GM.plan_many(algo, *table[:3], maps, table[3], map_of, sg, max_pts=32, path_fill=7.0)
        assert all(same(got[k], chk[k]) for k in KEYS)
        assert (got["status"] == OG.FOUND).mean() > 0.8


@pytest.mark.gpu
def test_reference_style_program_matches_the_checker(tmp_path):
    exe = build_ref_program(tmp_path, "grid_many_ref_api.cpp")
    out = tmp_path / "out.bin"
    subprocess.check_call([exe, str(out)])
    got = np.fromfile(out, np.float32)
    ox, oy = synth.grid_demo_obstacles()
    t = np.arange(0, 41, dtype=np.float32) * np.float32(0.5)
    z, tw = np.zeros_like(t), np.full_like(t, 20.0)
    qx = np.stack([t, t, z, tw], 1).reshape(-1)
    qy = np.stack([z, tw, t, t], 1).reshape(-1)
    queries = [(ox, oy, 1.0, 1.0, (10, 10, 50, 50)), (ox, oy, 1.0, 0.5, (5, 55, 55, 5)),
               (qx, qy, 0.5, 0.5, (1, 1, 8, 18.5))]
    want = []
    for algo in (OG.ASTAR, OG.DIJKSTRA):
        for x, y, reso, rr, p in queries:
            gb = OG.box_of_obstacles(x, y, reso)
            m = OG.obstacle_map(x, y, reso, rr, gb)
            r = OG.plan(algo, gb, m, reso, np.float32(p).reshape(4, 1), max_pts=512)
            assert r["status"][0] == OG.FOUND
            k = int(r["path_len"][0])
            want += [np.float32([k]), r["path"][0:2 * k:2, 0], r["path"][1:2 * k:2, 0]]
    assert same(got, np.concatenate(want))
