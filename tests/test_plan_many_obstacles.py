"""Planning with an obstacle list per robot: crb_dwa_control_many_batched and crb_rrt_plan_many_batched.

Each robot's or query's outputs must be bitwise those of the shared-list entry point run with its own list, and so those
of the checker composed list by list (oracle/dwa.py dwa_control, oracle/rrt.py plan).
CPU: argument validation without a device, synth.pack_obstacles / dwa_neighbour_obstacles, composing the checker per
list, the compiler report and the C++ program.
H100 (-m gpu): the equivalence at n = 1, 33, 4097 and 65536 on empty, 1-row and 256-row lists with robots in random
order, at default and non-default parameters; bad list references; a NaN in one RRT list; NULL outputs, n = 0 and graph
capture; a 50-tick closed loop of a fleet that avoids itself; the C++ program against the checker."""
import ctypes as C
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import dwa_cases as D
import rrt_cases as RC
from cpprobotics_b200 import _lib, rrt_default_params, synth
from oracle import dwa as OD
from oracle import rrt as OR
from toolchain import build_ref_program, ptxas_kernels

INV = -1
DEMO = synth.RRT_DEMO
RRT_KEYS = ("path", "path_len", "tree", "parent", "n_nodes", "n_iter", "status")
DWA_KEYS = ("u", "cost", "best", "traj")


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def lib_params(p):
    return _lib.DwaParams(*[getattr(p, k) for k, _ in p._fields_])


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is refused with CRB_ERR_INVALID_ARG before any device work; a valid call says
    CRB_ERR_NO_DEVICE on a machine without a GPU."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)
    good = lib_params(OD.dwa_params())

    def dwa(params=None, **over):
        a = dict(dict(ctx=ctx, n=5, x=d, u=d, goal=d, ob=d, rows=40, off=d, ns=3, of=d, prm=C.byref(params or good)),
                 **over)
        return L.crb_dwa_control_many_batched(a["ctx"], a["n"], a["x"], a["u"], a["goal"], a["ob"], a["rows"], a["off"],
                                              a["ns"], a["of"], a["prm"], None, None, None, None)

    for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(x=None), dict(u=None), dict(goal=None), dict(ns=0),
               dict(ns=-1), dict(rows=-1), dict(off=None), dict(of=None), dict(ob=None)):
        assert dwa(**kw) == INV, kw
    for field, value in (("v_reso", 0.0), ("dt", np.nan), ("predict_time", 1.0e6), ("max_speed", np.inf)):
        p = OD.dwa_params()
        setattr(p, field, float(value))
        assert dwa(lib_params(p)) == INV and dwa(lib_params(p), n=0) == INV, field

    def rrt(po=None, **over):
        p = rrt_default_params()
        for k, v in (po or {}).items():
            setattr(p, k, v)
        a = dict(dict(ctx=ctx, prm=C.byref(p), ob=d, rows=40, off=d, ns=3, of=d, n=5, se=d, seed=d, mp=4, mn=4), **over)
        return L.crb_rrt_plan_many_batched(a["ctx"], a["prm"], a["ob"], a["rows"], a["off"], a["ns"], a["of"], a["n"],
                                           a["se"], a["seed"], a["mp"], d, d, a["mn"], d, d, d, d, d)

    nan, inf = float("nan"), float("inf")
    for po in (dict(rand_min=nan), dict(rand_min=3.0, rand_max=2.0), dict(expand_dis=inf), dict(max_iter=0),
               dict(max_iter=_lib.CRB_RRT_MAX_ITER + 1)):
        assert rrt(po) == INV and rrt(po, n=0) == INV, po
    for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(mp=-1), dict(mn=-1), dict(se=None), dict(seed=None),
               dict(ns=0), dict(rows=-1), dict(off=None), dict(of=None), dict(ob=None)):
        assert rrt(**kw) == INV, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert dwa() == nd and dwa(ob=None, rows=0) == nd
        assert dwa(n=0, x=None, u=None, goal=None, ob=None, off=None, of=None) == nd
        assert rrt() == nd and rrt(ob=None, rows=0) == nd
        assert rrt(n=0, se=None, seed=None, ob=None, off=None, of=None) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def test_pack_obstacles_round_trips_with_empty_lists():
    for k, lists in ((2, synth.dwa_fleet_obstacles(40, seed=3)), (3, synth.rrt_fleet_obstacles(40, seed=4))):
        ob, off = synth.pack_obstacles(lists, k)
        assert ob.dtype == np.float32 and ob.shape == (off[-1], k) and ob.flags["C_CONTIGUOUS"]
        assert off.dtype == np.int64 and off.shape == (41,) and off[0] == 0 and (np.diff(off) >= 0).all()
        for s, o in enumerate(lists):
            assert same(ob[off[s]:off[s + 1]], np.asarray(o, np.float32).reshape(-1, k)), (k, s)
        assert (np.diff(off) == 0).sum() >= 3
    ob, off = synth.pack_obstacles([], 2)
    assert ob.shape == (0, 2) and off.tolist() == [0]
    ob, off = synth.pack_obstacles([np.zeros((0, 3))] * 4, 3)
    assert ob.shape == (0, 3) and off.tolist() == [0] * 5


def test_fleet_obstacles_are_varied_and_deterministic():
    a = synth.dwa_fleet_obstacles(64, seed=11)
    assert all(same(x, y) for x, y in zip(a, synth.dwa_fleet_obstacles(64, seed=11)))
    lens = np.array([len(o) for o in a])
    assert (lens == 0).sum() == 4 and (lens == 1).sum() >= 4 and (lens == _lib.CRB_DWA_MAX_OBSTACLES).sum() == 4
    assert len(set(lens.tolist())) > 20 and lens.max() <= _lib.CRB_DWA_MAX_OBSTACLES
    spans = np.array([np.ptp(o[:, 0]) for o in a if len(o) > 30])
    assert spans.min() < 20 and spans.max() > 40          # different arenas
    r = synth.rrt_fleet_obstacles(64, seed=12)
    rl = np.array([len(o) for o in r])
    assert (rl == 0).sum() >= 4 and rl.max() <= 64 and len(set(rl.tolist())) > 20
    assert all(o.shape[1] == 3 and o.dtype == np.float32 for o in r)


def test_neighbour_lists_exclude_the_robot_are_nearest_first_and_capped():
    x, _, _ = synth.dwa_inputs(700, seed=21)
    st = synth.DWA_DEMO_OBSTACLES
    for radius, cap in ((5.0, 256), (2.0, 40), (1.0, 10), (3.0, 12)):
        ob, off = synth.dwa_neighbour_obstacles(x, st, radius, cap)
        assert off.shape == (701,) and (np.diff(off) <= cap).all()
        px, py = x[0].astype(np.float64), x[1].astype(np.float64)
        for i in range(0, 700, 7):
            lst = ob[off[i]:off[i + 1]]
            k = min(len(st), cap)
            assert same(lst[:k], st[:k])
            nb = lst[k:]
            d2 = (nb[:, 0].astype(np.float64) - px[i]) ** 2 + (nb[:, 1].astype(np.float64) - py[i]) ** 2
            assert (d2 <= radius * radius).all() and (np.diff(d2) >= 0).all()       # within radius, nearest first
            allj = (px - px[i]) ** 2 + (py - py[i]) ** 2
            others = np.delete(np.arange(700), i)
            want = others[np.lexsort((others, allj[others]))]
            want = want[allj[want] <= radius * radius][:cap - k]
            assert same(nb, np.stack([x[0, want], x[1, want]], axis=1).reshape(-1, 2))   # never the robot itself
    one = synth.dwa_neighbour_obstacles(x[:, :1], st, 5.0, 256)
    assert same(one[0], st) and one[1].tolist() == [0, 10]


def dwa_per_list(lists, ob_of, x, u, g, run):
    """run(ob, x, u, g) -> dict(u, cost, best, traj), once per list on its own robots, scattered back."""
    n = x.shape[1]
    out = None
    for s in np.unique(ob_of):
        sel = np.nonzero(ob_of == s)[0]
        r = run(lists[s], *(np.ascontiguousarray(a[:, sel]) for a in (x, u, g)))
        if out is None:
            out = {k: np.zeros(v.shape[:-1] + (n,), v.dtype) for k, v in r.items()}
        for k in out:
            out[k][..., sel] = r[k]
    return out


def rrt_per_list(lists, ob_of, se, seed, run):
    n = se.shape[1]
    out = None
    for s in np.unique(ob_of):
        sel = np.nonzero(ob_of == s)[0]
        r = run(lists[s], np.ascontiguousarray(se[:, sel]), seed[sel])
        if out is None:
            out = {k: np.zeros(np.asarray(r[k]).shape[:-1] + (n,), np.asarray(r[k]).dtype) for k in RRT_KEYS}
        for k in RRT_KEYS:
            out[k][..., sel] = r[k]
    return out


def dwa_checker(p=None):
    return lambda ob, x, u, g: {k: v for k, v in OD.dwa_control(x, u, g, ob, p).items()}


def rrt_checker(prm, max_pts=64, max_nodes=512):
    return lambda ob, se, seed: OR.plan(prm, ob, se, seed, max_pts=max_pts, max_nodes=max_nodes)


def test_checker_composed_per_list_is_the_checker_on_one_shared_list():
    x, u, g = D.batch(300, synth.DWA_DEMO_OBSTACLES, seed=5)
    ob_of = np.zeros(300, np.int32)
    ob_of[::3] = 1
    lists = [synth.DWA_DEMO_OBSTACLES, synth.DWA_DEMO_OBSTACLES.copy()]
    a = dwa_per_list(lists, ob_of, x, u, g, dwa_checker())
    b = OD.dwa_control(x, u, g, synth.DWA_DEMO_OBSTACLES)
    assert all(same(a[k], b[k]) for k in DWA_KEYS)
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    se, seed = synth.rrt_inputs(200, ob, DEMO["rand_min"], DEMO["rand_max"], seed=6)
    r = rrt_per_list([ob, ob.copy(), ob.copy()], np.arange(200, dtype=np.int32) % 3, se, seed, rrt_checker(prm))
    o = OR.plan(prm, ob, se, seed, max_pts=64, max_nodes=512)
    assert all(same(r[k], o[k]) for k in RRT_KEYS)


def test_changed_kernels_do_not_spill():
    found = []
    for src, kernel, max_regs in (("crb_dwa.cu", "crb_dwa_control_many_kernel", 64),
                                  ("crb_rrt.cu", "crb_rrt_plan_kernel", 58)):
        for name, f in ptxas_kernels(src).items():
            if kernel in name:
                found.append(kernel)
                assert (f.stack, f.spill_stores, f.spill_loads) == (0, 0, 0) and f.registers <= max_regs, f
    assert sorted(found) == ["crb_dwa_control_many_kernel", "crb_rrt_plan_kernel"]


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "plan_many_ref_api.cpp")


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    return None if t is None else t.cpu().numpy()


def dwa_lists():
    """Fleet lists (empty, 1-row and 256-row ones among them), the demo's list and a 256-row list, shuffled."""
    rng = np.random.default_rng(0xD3)
    lists = synth.dwa_fleet_obstacles(40, seed=3) + [synth.DWA_DEMO_OBSTACLES, synth.dwa_obstacles(256),
                                                     np.zeros((0, 2), np.float32)]
    return [lists[k] for k in rng.permutation(len(lists))]


def dwa_fleet(n, lists, seed, p=None):
    rng = np.random.default_rng(seed)
    ob_of = rng.integers(0, len(lists), n).astype(np.int32)
    x, u, g = D.batch(n, np.zeros((0, 2)), seed=seed, params=p)
    return ob_of, x, u, g


def gpu_dwa_many(engine, lists, ob_of, x, u, g, p=None, outputs=True, store=None):
    import torch
    n = x.shape[1]
    p = p or OD.dwa_params()
    ob, off = store if store is not None else synth.pack_obstacles(lists, 2)
    ud = _dev(u)
    cost = torch.full((n,), 7.0, device="cuda:0") if outputs else None
    best = torch.full((n,), 7, dtype=torch.int32, device="cuda:0") if outputs else None
    traj = torch.full((5 * OD.dwa_rollout_points(p), n), 7.0, device="cuda:0") if outputs else None
    st = engine.dwa_control_many(_dev(x), ud, _dev(g), (_dev(ob), _dev(off)), _dev(ob_of), lib_params(p), cost=cost,
                                 best=best, traj=traj)
    torch.cuda.synchronize()
    return dict(u=_host(ud), cost=_host(cost), best=_host(best), traj=_host(traj), status=_host(st))


def dwa_shared_gpu(engine, p=None):
    import torch

    def run(ob, x, u, g):
        p_ = p or OD.dwa_params()
        n = x.shape[1]
        ud = _dev(u)
        cost = torch.empty(n, device="cuda:0")
        best = torch.empty(n, dtype=torch.int32, device="cuda:0")
        traj = torch.empty((5 * OD.dwa_rollout_points(p_), n), device="cuda:0")
        engine.dwa_control(_dev(x), ud, _dev(g), _dev(np.asarray(ob, np.float32).reshape(-1, 2)), lib_params(p_),
                           cost=cost, best=best, traj=traj)
        torch.cuda.synchronize()
        return dict(u=_host(ud), cost=_host(cost), best=_host(best), traj=_host(traj))
    return run


def assert_dwa_same(got, want, keys=DWA_KEYS):
    for k in keys:
        assert same(got[k], want[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
def test_gpu_dwa_many_is_the_shared_entry_and_the_checker_per_list(engine, n):
    lists = dwa_lists()
    ob_of, x, u, g = dwa_fleet(n, lists, seed=0xD00 + n)
    got = gpu_dwa_many(engine, lists, ob_of, x, u, g)
    assert (got["status"] == _lib.CRB_DWA_OK).all()
    assert_dwa_same(got, dwa_per_list(lists, ob_of, x, u, g, dwa_shared_gpu(engine)))
    assert_dwa_same(got, dwa_per_list(lists, ob_of, x, u, g, dwa_checker()))
    if n >= 4097:
        lens = np.array([len(o) for o in lists])[ob_of]
        assert (lens == 0).any() and (lens == 1).any() and (lens == 256).any()
        assert (got["best"] < 0).any() and (got["best"] >= 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["distinct", "radius_zero", "zero_steps", "gains_overflow", "speed_cap"])
def test_gpu_dwa_many_with_non_default_params(engine, name):
    p = D.config(name)
    lists = dwa_lists()
    ob_of, x, u, g = dwa_fleet(4097, lists, seed=0xDA, p=p)
    got = gpu_dwa_many(engine, lists, ob_of, x, u, g, p)
    assert_dwa_same(got, dwa_per_list(lists, ob_of, x, u, g, dwa_shared_gpu(engine, p)))
    assert_dwa_same(got, dwa_per_list(lists, ob_of, x, u, g, dwa_checker(p)))


@pytest.mark.gpu
def test_gpu_dwa_many_bad_references(engine):
    lists = dwa_lists()
    ob, off = synth.pack_obstacles(lists, 2)
    nl = len(lists)
    rows = len(ob)
    # more lists in the store: nl = [rows, rows - 3) decreasing; nl + 1 = [rows - 3, rows) valid; nl + 2 = [rows,
    # rows + 257) over the cap; nl + 3 = [rows + 257, rows + 257) empty, valid; nl + 4 ends past n_rows
    ob2 = np.concatenate([ob, synth.dwa_obstacles(257)])
    off2 = np.concatenate([off, [rows - 3, rows, rows + 257, rows + 257, rows + 10 ** 6]])
    n = 4097
    ob_of, x, u, g = dwa_fleet(n, lists, seed=0xBAD)
    rng = np.random.default_rng(7)
    bad = rng.random(n) < 0.25
    kinds = np.int64([nl, nl + 2, nl + 4, -1, nl + 5, 2 ** 31 - 1, -(2 ** 31)])
    of = np.where(bad, kinds[rng.integers(0, kinds.size, n)], ob_of).astype(np.int32)
    got = gpu_dwa_many(engine, lists, of, x, u, g, store=(ob2, off2))
    assert (got["status"][bad] == _lib.CRB_DWA_BAD_OBSTACLES).all()
    assert (got["status"][~bad] == _lib.CRB_DWA_OK).all()
    assert np.isnan(got["u"][:, bad]).all() and np.isnan(got["cost"][bad]).all() and (got["best"][bad] == -1).all()
    assert np.isnan(got["traj"][:, bad]).all()
    want = dwa_per_list(lists, ob_of[~bad], *(a[:, ~bad] for a in (x, u, g)), run=dwa_checker())
    assert_dwa_same({k: v[..., ~bad] for k, v in got.items()}, want)
    # the valid extra lists, and an offset past n_rows on the last list only
    empty = np.zeros((0, 2), np.float32)
    ext = lists + [empty, ob2[rows - 3:rows], empty, empty]
    of = np.where(rng.random(n) < 0.3, rng.choice(np.int32([nl + 1, nl + 3]), n), ob_of).astype(np.int32)
    got = gpu_dwa_many(engine, ext, of, x, u, g, store=(ob2, off2))
    assert (got["status"] == _lib.CRB_DWA_OK).all()
    assert_dwa_same(got, dwa_per_list(ext, of, x, u, g, dwa_checker()))
    off_past = off.copy()
    off_past[-1] = rows + 1
    got = gpu_dwa_many(engine, lists, ob_of, x, u, g, store=(ob, off_past))
    assert ((got["status"] == _lib.CRB_DWA_BAD_OBSTACLES) == (ob_of == nl - 1)).all()


@pytest.mark.gpu
def test_gpu_dwa_many_launch_forms(engine):
    """NULL optional outputs, n = 0 and a graph-captured launch."""
    import torch
    lists = synth.dwa_fleet_obstacles(24, seed=8)
    ob, off = synth.pack_obstacles(lists, 2)
    ob_of, x, u, g = dwa_fleet(3000, lists, seed=0xF0)
    want = dwa_per_list(lists, ob_of, x, u, g, dwa_checker())
    got = gpu_dwa_many(engine, lists, ob_of, x, u, g, outputs=False)
    assert same(got["u"], want["u"]) and (got["status"] == 0).all()
    prm = lib_params(OD.dwa_params())
    obd, offd = _dev(ob), _dev(off)
    assert engine.lib.crb_dwa_control_many_batched(engine.ctx, 0, None, None, None, obd.data_ptr(), len(ob),
                                                   offd.data_ptr(), len(lists), None, C.byref(prm), None, None, None,
                                                   None) == 0
    e = torch.empty((5, 0), device="cuda:0")
    st = engine.dwa_control_many(e, e[:2], e[:2], (obd, offd), torch.empty(0, dtype=torch.int32, device="cuda:0"))
    assert st.shape == (0,)
    xd, ud, gd, ofd = _dev(x), _dev(u), _dev(g), _dev(ob_of)
    cost = torch.empty(3000, device="cuda:0")
    best = torch.empty(3000, dtype=torch.int32, device="cuda:0")
    traj = torch.empty((5 * OD.dwa_rollout_points(), 3000), device="cuda:0")
    stt = torch.empty(3000, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        eng = type(engine)(0)
        try:
            with torch.cuda.graph(gr, stream=s):
                eng.dwa_control_many(xd, ud, gd, (obd, offd), ofd, cost=cost, best=best, traj=traj, status=stt)
            gr.replay()
            torch.cuda.synchronize()
        finally:
            eng.close()
    assert_dwa_same(dict(u=_host(ud), cost=_host(cost), best=_host(best), traj=_host(traj)), want)
    assert (_host(stt) == 0).all()


def _checker_one_robot(args):
    x, u, g, ob = args
    return OD.dwa_control(x, u, g, ob, traj=False, nthreads=1)


@pytest.mark.gpu
def test_gpu_dwa_many_closed_loop_of_a_fleet_that_avoids_itself(engine):
    """1024 robots, 50 ticks: each tick the lists are rebuilt from the device states (the demo obstacles plus the other
    robots within 5 m, nearest first, capped at 256), dwa_control_many decides and crb_dwa_motion_batched advances;
    every tick's decisions are bitwise the checker's, robot by robot on its own list."""
    import torch
    n, ticks = 1024, 50
    x, u, g = synth.dwa_inputs(n, seed=0xF1EE)
    rng = np.random.default_rng(3)
    # about 10 neighbours within 5 m; a robot with a neighbour inside its radius (1 m) has no admissible sample
    x[:2] = rng.uniform(-40.0, 50.0, (2, n)).astype(np.float32)
    g = rng.uniform(-40.0, 50.0, (2, n)).astype(np.float32)
    xd, ud, gd = _dev(x), _dev(u), _dev(g)
    of = torch.arange(n, dtype=torch.int32, device="cuda:0")
    xo, uo = x.copy(), u.copy()
    longest = 0
    with ThreadPoolExecutor(max(1, min(32, len(os.sched_getaffinity(0))))) as pool:
        for tick in range(ticks):
            xs = _host(xd)
            ob, off = synth.dwa_neighbour_obstacles(xs, synth.DWA_DEMO_OBSTACLES, 5.0, 256)
            longest = max(longest, int(np.diff(off).max()))
            st = engine.dwa_control_many(xd, ud, gd, (_dev(ob), _dev(off)), of)
            engine.dwa_motion(xd, ud)
            assert same(xs, xo), tick
            parts = list(pool.map(_checker_one_robot, [(xo[:, i:i + 1], uo[:, i:i + 1], g[:, i:i + 1],
                                                        ob[off[i]:off[i + 1]]) for i in range(n)]))
            uo = np.concatenate([r["u"] for r in parts], axis=1)
            xo = OD.dwa_motion(xo, uo)
            torch.cuda.synchronize()
            assert (_host(st) == 0).all() and same(_host(ud), uo), tick
    assert same(_host(xd), xo) and longest > 15
    assert (np.hypot(xo[0] - x[0], xo[1] - x[1]) > 0.5).mean() > 0.25


# ---- H100: RRT --------------------------------------------------------------------------------------------------
def _rrt_params(prm):
    p = rrt_default_params()
    for k in ("rand_min", "rand_max", "expand_dis", "goal_sample_rate", "max_iter"):
        setattr(p, k, prm[k])
    return p


def rrt_fleet(n, lists, lo, hi, seed):
    rng = np.random.default_rng(seed)
    ob_of = rng.integers(0, len(lists), n).astype(np.int32)
    se, sd = np.zeros((4, n), np.float32), np.zeros(n, np.uint32)
    for s in np.unique(ob_of):
        sel = np.nonzero(ob_of == s)[0]
        se[:, sel], sd[sel] = synth.rrt_inputs(sel.size, lists[s], lo, hi, seed=int(seed * 31 + s))
    return ob_of, se, sd


def gpu_rrt_many(engine, prm, lists, ob_of, se, seed, max_pts=64, max_nodes=512, store=None, **kw):
    ob, off = store if store is not None else synth.pack_obstacles(lists, 3)
    sd = _dev(np.asarray(seed, np.uint32).view(np.int32))
    r = engine.rrt_plan_many((_dev(ob), _dev(off)), _dev(ob_of), _dev(se), sd, _rrt_params(prm), max_pts=max_pts,
                             max_nodes=max_nodes, **kw)
    return {k: _host(v) for k, v in r.items()}


def rrt_shared_gpu(engine, prm, max_pts=64, max_nodes=512):
    def run(ob, se, seed):
        r = engine.rrt_plan(_dev(np.asarray(ob, np.float32).reshape(-1, 3)), _dev(se),
                            _dev(np.asarray(seed, np.uint32).view(np.int32)), _rrt_params(prm), max_pts=max_pts,
                            max_nodes=max_nodes)
        return {k: _host(v) for k, v in r.items()}
    return run


def rrt_lists(lo, hi):
    rng = np.random.default_rng(0x77)
    lists = synth.rrt_fleet_obstacles(30, seed=5, lo=lo, hi=hi) + [synth.rrt_demo_obstacles()]
    return [lists[k] for k in rng.permutation(len(lists))]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
def test_gpu_rrt_many_is_the_shared_entry_and_the_checker_per_list(engine, n):
    prm = RC.demo_prm()
    lists = rrt_lists(DEMO["rand_min"], DEMO["rand_max"])
    ob_of, se, seed = rrt_fleet(n, lists, DEMO["rand_min"], DEMO["rand_max"], seed=n)
    got = gpu_rrt_many(engine, prm, lists, ob_of, se, seed)
    assert (got["status"] != _lib.CRB_RRT_BAD_OBSTACLES).all()
    want = rrt_per_list(lists, ob_of, se, seed, rrt_shared_gpu(engine, prm))
    assert all(same(got[k], want[k]) for k in RRT_KEYS)
    want = rrt_per_list(lists, ob_of, se, seed, rrt_checker(prm))
    for k in RRT_KEYS:
        assert same(got[k], want[k]), k
    if n >= 4097:
        assert (got["status"] == OR.FOUND).mean() > 0.9


@pytest.mark.gpu
def test_gpu_rrt_many_with_non_default_params(engine):
    for prm, _, _, _, _, _, sd in list(RC.scattered_maps(4, seed=0xAB)):
        prm = dict(prm, max_iter=2048)
        lo, hi = float(prm["rand_min"]), float(prm["rand_max"])
        lists = synth.rrt_fleet_obstacles(12, seed=sd & 0xFFFF, lo=lo, hi=hi, max_k=40)
        ob_of, se, seed = rrt_fleet(4097, lists, lo, hi, seed=sd & 0xFFF)
        got = gpu_rrt_many(engine, prm, lists, ob_of, se, seed)
        want = rrt_per_list(lists, ob_of, se, seed, rrt_checker(prm))
        for k in RRT_KEYS:
            assert same(got[k], want[k]), (prm, k)
        want = rrt_per_list(lists, ob_of, se, seed, rrt_shared_gpu(engine, prm))
        assert all(same(got[k], want[k]) for k in RRT_KEYS)


@pytest.mark.gpu
def test_gpu_rrt_many_bad_references_and_a_nan_in_one_list(engine):
    prm = RC.demo_prm(max_iter=1024)
    lists = rrt_lists(DEMO["rand_min"], DEMO["rand_max"])
    nl = len(lists)
    ob, off = synth.pack_obstacles(lists, 3)
    rows = len(ob)
    off2 = np.concatenate([off, [rows - 3, rows + 10 ** 6]])   # nl: decreasing; nl + 1: past n_rows
    n = 4097
    ob_of, se, seed = rrt_fleet(n, lists, DEMO["rand_min"], DEMO["rand_max"], seed=0xBAD)
    rng = np.random.default_rng(9)
    bad = rng.random(n) < 0.25
    kinds = np.int64([nl, nl + 1, nl + 2, -1, 2 ** 31 - 1])
    of = np.where(bad, kinds[rng.integers(0, kinds.size, n)], ob_of).astype(np.int32)
    got = gpu_rrt_many(engine, prm, lists, of, se, seed, store=(ob, off2))
    assert (got["status"][bad] == _lib.CRB_RRT_BAD_OBSTACLES).all()
    for k in ("n_nodes", "n_iter", "path_len"):
        assert (got[k][bad] == 0).all(), k
    assert np.isnan(got["path"][:, bad]).all() and np.isnan(got["tree"][:, bad]).all()
    assert (got["parent"][:, bad] == -1).all()
    want = rrt_per_list(lists, ob_of[~bad], se[:, ~bad], seed[~bad], rrt_checker(prm))
    assert all(same(got[k][..., ~bad], want[k]) for k in RRT_KEYS)
    # a NaN in one list: BAD_INPUT for the queries on that list only, as the shared entry gives it on that list
    big = int(np.argmax([len(o) for o in lists]))
    nan_lists = [o.copy() for o in lists]
    nan_lists[big][len(nan_lists[big]) // 2, 2] = np.nan
    got = gpu_rrt_many(engine, prm, nan_lists, ob_of, se, seed)
    on = ob_of == big
    assert on.any() and (got["status"][on] == OR.BAD_INPUT).all() and (got["n_nodes"][on] == 0).all()
    assert (got["status"][~on] != OR.BAD_INPUT).mean() > 0.9
    want = rrt_per_list(nan_lists, ob_of, se, seed, rrt_checker(prm))
    assert all(same(got[k], want[k]) for k in RRT_KEYS)
    want = rrt_per_list(nan_lists, ob_of, se, seed, rrt_shared_gpu(engine, prm))
    assert all(same(got[k], want[k]) for k in RRT_KEYS)


@pytest.mark.gpu
def test_gpu_rrt_many_launch_forms(engine):
    """NULL outputs, n = 0, and a graph-captured launch after the first call on the context."""
    import torch
    prm = RC.demo_prm()
    lists = rrt_lists(DEMO["rand_min"], DEMO["rand_max"])
    ob, off = synth.pack_obstacles(lists, 3)
    ob_of, se, seed = rrt_fleet(3000, lists, DEMO["rand_min"], DEMO["rand_max"], seed=44)
    full = rrt_per_list(lists, ob_of, se, seed, rrt_checker(prm, 8, 40))
    obs, ofd, sed, sdd = (_dev(ob), _dev(off)), _dev(ob_of), _dev(se), _dev(seed.view(np.int32))
    p = _rrt_params(prm)
    for k in ("path_len", "n_nodes", "n_iter", "status"):
        buf = torch.empty(3000, dtype=torch.int32, device="cuda:0")
        res = engine.rrt_plan_many(obs, ofd, sed, sdd, p, **{k: buf})
        assert same(_host(res[k]), full[k]) and res["path"] is None and res["tree"] is None, k
    z = torch.empty(0, dtype=torch.int32, device="cuda:0")
    e = engine.rrt_plan_many(obs, z, torch.empty((4, 0), device="cuda:0"), z, p, max_pts=4)
    assert e["status"].shape == (0,) and e["path"].shape == (8, 0)
    out = {k: torch.full_like(v, -1) for k, v in engine.rrt_plan_many(obs, ofd, sed, sdd, p, max_pts=8,
                                                                        max_nodes=40).items()}
    torch.cuda.synchronize()
    for v in out.values():
        v.fill_(float("nan") if v.is_floating_point() else -1)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        engine.bind_current_stream()
        with torch.cuda.graph(g, stream=s):
            engine.rrt_plan_many(obs, ofd, sed, sdd, p, max_pts=8, max_nodes=40, **out)
    engine.bind_current_stream()
    g.replay()
    torch.cuda.synchronize()
    for k in RRT_KEYS:
        assert same(_host(out[k]), full[k]), k


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_the_checker(tmp_path):
    exe = build_ref_program(tmp_path, "plan_many_ref_api.cpp")
    lists = synth.dwa_fleet_obstacles(6, seed=13)
    m = 6
    x, u, g = synth.dwa_inputs(m, seed=14)
    blob = [np.float32([m])]
    for i in range(m):
        blob += [x[:, i], u[:, i], g[:, i], np.float32([len(lists[i])]), lists[i].reshape(-1)]
    rl = [synth.rrt_demo_obstacles(), np.zeros((0, 3), np.float32)] + synth.rrt_fleet_obstacles(3, seed=15)[1:]
    q = len(rl)
    se, seed = np.zeros((4, q), np.float32), np.arange(1, q + 1, dtype=np.uint32)
    for i in range(q):
        se[:, i:i + 1] = synth.rrt_inputs(1, rl[i], DEMO["rand_min"], DEMO["rand_max"], seed=20 + i)[0]
    blob.append(np.float32([q]))
    for i in range(q):
        blob += [se[:, i], seed[i:i + 1].view(np.float32), np.float32([len(rl[i])]), rl[i].reshape(-1)]
    np.concatenate(blob).astype(np.float32).tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    p = 0
    for i in range(m):
        o = OD.dwa_control(x[:, i:i + 1], u[:, i:i + 1], g[:, i:i + 1], lists[i])
        assert same(out[p:p + 2], o["u"][:, 0]); p += 2
        k = int(out[p]); p += 1
        assert k == (0 if o["best"][0] < 0 else OD.dwa_rollout_points())
        assert same(out[p:p + 5 * k], o["traj"][:, 0][:5 * k]); p += 5 * k
    prm = RC.demo_prm(max_iter=_lib.CRB_RRT_MAX_ITER)
    for i in range(q):
        c = RC.checker_one(prm, rl[i], *se[:, i], int(seed[i]))
        k = int(out[p]); p += 1
        assert c["status"] == OR.FOUND and k == len(c["path"])
        assert same(out[p:p + 2 * k], c["path"].reshape(-1)), i
        p += 2 * k
    assert p == out.size
