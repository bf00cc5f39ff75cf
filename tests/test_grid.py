"""Grid A* and Dijkstra (src/a_star.cpp, src/dijkstra.cpp).
CPU: the checker's restated heap pops ties in the order of the host's std::priority_queue; the checker is bitwise the
reference's own text (obstacle map, expansion trace and path) on the demo, seeded scenarios and corner cases; the
golden fixture; statuses where the reference is undefined; layouts, validation without a device, the reference-style
program compiles, and the kernels do not spill.  H100: crb_grid_obstacle_map and crb_grid_plan_batched are bitwise
the checker (every output, several batch sizes and maps, more queries than slots, short path buffers, n = 0, split
batches, a CUDA graph), the golden fixture, and the reference-style C++ program."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import grid_cases as GC
from grid_cases import same
from cpprobotics_b200 import _lib, grid_box_of_obstacles, synth
from oracle import grid as OG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "grid_golden.npz")
CPP_API = os.path.join(ROOT, "tests", "cpp", "grid_ref_api.cpp")
CPP_HEAP = os.path.join(ROOT, "tests", "cpp", "grid_heap_pin.cpp")
ALGO_IDS = [a for a, _ in GC.ALGOS]


def _ref(algo):
    L = GC.ref_lib(algo)
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
    return L


def _setup(ox, oy, reso, rr):
    box = OG.box_of_obstacles(ox, oy, reso)
    return box, OG.obstacle_map(ox, oy, reso, rr, box)


def _path_cells(r, q, reso):
    n = int(r["path_len"][q])
    return r["path"][:2 * n, q].reshape(n, 2)


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_heap_pops_ties_in_the_order_of_std_priority_queue(tmp_path):
    exe = str(tmp_path / "heap_pin")
    subprocess.check_call(["g++", "-std=c++11", "-O2", "-Wall", "-Werror", CPP_HEAP, "-o", exe])
    rng = np.random.default_rng(0x4EA9)
    n = 100000
    keys = rng.integers(0, 6, n).astype(np.float32) * np.float32(0.5)   # six distinct keys: ties everywhere
    op = np.zeros(n, np.uint8)
    size = 0
    for i, u in enumerate(rng.random(n)):   # pushes and pops interleaved, the heap growing and shrinking
        push = size == 0 or u < (0.62 if i % 20000 < 12000 else 0.4)
        op[i] = push
        size += 1 if push else -1
    rec = np.zeros(n, dtype=[("op", np.uint8), ("key", np.float32)])
    rec["op"], rec["key"] = op, keys
    (tmp_path / "ops.bin").write_bytes(rec.tobytes())
    subprocess.check_call([exe, str(tmp_path / "ops.bin"), str(tmp_path / "out.bin")])
    want = np.fromfile(tmp_path / "out.bin", np.int32)
    got = OG.heap_run(op, keys)
    assert want.size == (op == 0).sum() > 40000
    assert np.array_equal(got, want)


def _compare_with_reference(algo, L, ox, oy, reso, rr, sx, sy, gx, gy):
    """False when the reference does not define the query (nothing compared), True after a bitwise comparison."""
    box, m = _setup(ox, oy, reso, rr)
    r = OG.plan(algo, box, m, reso, np.float32([[sx], [sy], [gx], [gy]]), max_pts=1 << 14)
    if not GC.check_ref_domain(algo, box, r["status"][0]):
        return False
    ref = GC.ref_run(L, sx, sy, gx, gy, ox, oy, reso, rr)
    assert np.array_equal(np.argwhere(m != 0), ref["map_cells"])
    assert np.array_equal(OG.trace(algo, box, m, reso, sx, sy, gx, gy), ref["trace"])
    assert r["path_len"][0] == len(ref["path"]) and r["n_visited"][0] >= 1
    assert same(_path_cells(r, 0, reso), ref["path"].astype(np.float32) * np.float32(reso))
    return True


@pytest.mark.parametrize("algo", ALGO_IDS)
def test_demo_is_bitwise_the_reference_text(algo):
    L = _ref(algo)
    ox, oy, reso, rr, sg = GC.demo()
    assert _compare_with_reference(algo, L, ox, oy, reso, rr, *sg[:, 0])
    box, m = _setup(ox, oy, reso, rr)
    assert list(box) == [0, 0, 60, 60] and m.shape == (60, 60)


@pytest.mark.parametrize("algo", ALGO_IDS)
def test_seeded_scenarios_are_bitwise_the_reference_text(algo):
    L = _ref(algo)
    done = sum(_compare_with_reference(algo, L, *s) for s in GC.seeded_scenarios(algo, 240, seed=0x5EED + algo))
    assert done >= 200


@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("case", [c[0] for c in GC.corner_cases()])
def test_corner_cases_are_bitwise_the_reference_text(algo, case):
    L = _ref(algo)
    c = next(c for c in GC.corner_cases() if c[0] == case)
    assert _compare_with_reference(algo, L, *c[1:])
    box, m = _setup(*c[1:5])
    r = OG.plan(algo, box, m, c[3], np.float32([[c[5]], [c[6]], [c[7]], [c[8]]]))
    if case == "start_is_goal":
        assert r["path_len"][0] == 1 and r["n_visited"][0] == 1 and r["cost"][0] == 0
    if case == "start_on_obstacle":
        assert m[21, 5] and r["status"][0] == OG.FOUND
    if case == "goal_adjacent":
        assert r["path_len"][0] == 2


def test_oracle_reproduces_the_golden_fixture():
    d = np.load(GOLDEN)
    for algo, name in GC.ALGOS:
        ox, oy, reso, rr, sg = GC.demo()
        box, m = _setup(ox, oy, reso, rr)
        assert np.array_equal(np.argwhere(m != 0), d[f"demo_{name}_map_cells"])
        assert np.array_equal(OG.trace(algo, box, m, reso, *sg[:, 0]), d[f"demo_{name}_trace"])
        r = OG.plan(algo, box, m, reso, sg, max_pts=256)
        assert same(_path_cells(r, 0, reso), d[f"demo_{name}_path"].astype(np.float32) * np.float32(reso))
        p = o = 0
        for k, (no, pl) in enumerate(zip(d[f"seeded_{name}_n_obs"], d[f"seeded_{name}_path_len"])):
            v = d[f"seeded_{name}_inputs"][p:p + 6 + 2 * no]
            p += 6 + 2 * no
            box, m = _setup(v[6:6 + no], v[6 + no:], v[0], v[1])
            r = OG.plan(algo, box, m, v[0], v[2:6].reshape(4, 1), max_pts=int(pl))
            want = d[f"seeded_{name}_path"][o:o + pl].astype(np.float32) * np.float32(v[0])
            o += pl
            assert r["status"][0] == OG.FOUND and same(_path_cells(r, 0, v[0]), want), (name, k)
        assert k == 23


def _walk_ok(path, n, reso, box, m):
    """A path of adjacent, in-box cells whose cells after the start are free."""
    cells = np.rint(path[:2 * n].reshape(n, 2) / np.float32(reso)).astype(np.int64)
    steps = np.abs(np.diff(cells, axis=0))
    inside = ((cells[:, 0] >= box[0]) & (cells[:, 0] < box[2]) & (cells[:, 1] >= box[1]) & (cells[:, 1] < box[3]))
    free = m[cells[:-1, 0] - box[0], cells[:-1, 1] - box[1]] == 0
    return inside.all() and (steps.max(axis=1) == 1).all() and free.all()


@pytest.mark.parametrize("algo", ALGO_IDS)
def test_checker_statuses_where_the_reference_is_undefined(algo):
    ox, oy, reso, rr, _ = GC.demo()
    box, m = _setup(ox, oy, reso, rr)
    # a goal on an obstacle and one outside the box (every free cell visited), a start outside, NaN / inf / huge points
    sg = np.float32([[10, 10, 10, 70, np.nan, 10, 1e20, 10],
                     [10, 10, 10, 10, 10, 10, 10, -0.5],
                     [50, 20, 61, 50, 50, 50, 50, np.inf],
                     [50, 10, 50, 50, 50, 50, 50, 50]])
    r = OG.plan(algo, box, m, reso, sg, max_pts=8)
    assert r["status"].tolist() == [OG.FOUND, OG.NO_PATH, OG.NO_PATH, OG.START_OUTSIDE, OG.BAD_POINT,
                                    OG.FOUND, OG.BAD_POINT, OG.BAD_POINT]
    bad = r["status"] != OG.FOUND
    assert (r["path_len"][bad] == 0).all() and np.isnan(r["cost"][bad]).all()
    assert (r["n_visited"][[1, 2]] == (m == 0).sum()).all() and (r["n_visited"][[3, 4, 6, 7]] == 0).all()
    assert r["n_visited"][0] > 1 and np.isnan(r["path"][:, bad]).all()
    walled = OG.obstacle_map(ox, oy, reso, 12.0, box)   # rr 12 closes the gaps the inner walls leave
    r = OG.plan(algo, box, walled, reso, sg[:, :1])
    assert r["status"][0] == OG.NO_PATH and r["n_visited"][0] > 0
    # a rectangular box, and a box away from the origin: defined here by the box-relative indexing
    for ox2, oy2 in ((np.float32([-7, 30, 3, 4]), np.float32([5, 17, 9, 12])),
                     (np.float32([100, 140, 120]), np.float32([-80, -40, -60]))):
        box2, m2 = _setup(ox2, oy2, 1.0, 1.5)
        W, H = OG.dims(box2)
        sg2 = synth.grid_inputs(64, box2, m2, 1.0, seed=3)
        r = OG.plan(algo, box2, m2, 1.0, sg2, max_pts=W * H)
        ok = np.flatnonzero(r["status"] == OG.FOUND)
        assert len(ok) >= 40
        for q in ok:
            assert _walk_ok(r["path"][:, q], r["path_len"][q], 1.0, box2, m2), q
            assert same(r["path"][:2, q], np.float32([np.rint(sg2[2, q]), np.rint(sg2[3, q])]) + np.float32(0))   # cell * reso: +0, never -0


def test_box_and_layout_on_the_host(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){printf("%zu %zu %zu %zu '
                   '%d %d %d %d %d %d %d %d %zu\\n",sizeof(crb_grid_box),offsetof(crb_grid_box,min_y),'
                   'offsetof(crb_grid_box,max_x),offsetof(crb_grid_box,max_y),CRB_GRID_MAX_SIDE,CRB_GRID_MAX_CELLS,'
                   'CRB_GRID_ASTAR,CRB_GRID_DIJKSTRA,CRB_GRID_FOUND,CRB_GRID_NO_PATH,CRB_GRID_START_OUTSIDE,'
                   'CRB_GRID_BAD_POINT,CRB_GRID_WS_BUDGET);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    B = _lib.GridBox
    assert got[:4] == [C.sizeof(B), B.min_y.offset, B.max_x.offset, B.max_y.offset]
    assert got[4:] == [_lib.CRB_GRID_MAX_SIDE, _lib.CRB_GRID_MAX_CELLS, _lib.CRB_GRID_ASTAR, _lib.CRB_GRID_DIJKSTRA,
                       _lib.CRB_GRID_FOUND, _lib.CRB_GRID_NO_PATH, _lib.CRB_GRID_START_OUTSIDE,
                       _lib.CRB_GRID_BAD_POINT, _lib.CRB_GRID_WS_BUDGET]
    assert got[4:12] == [OG.MAX_SIDE, OG.MAX_CELLS, OG.ASTAR, OG.DIJKSTRA, OG.FOUND, OG.NO_PATH, OG.START_OUTSIDE,
                         OG.BAD_POINT]
    # the box needs no device and is the checker's
    ox, oy = synth.grid_demo_obstacles()
    for reso in (1.0, 0.5, 2.0, 0.3):
        b = grid_box_of_obstacles(ox, oy, reso)
        assert [b.min_x, b.min_y, b.max_x, b.max_y] == OG.box_of_obstacles(ox, oy, reso).tolist()
    h = grid_box_of_obstacles(np.float32([0.5, -0.5, 2.5]), np.float32([1.5, -1.5, -2.5]), 1.0)
    assert [h.min_x, h.min_y, h.max_x, h.max_y] == [-1, -3, 3, 2]   # round: half away from zero


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE on a machine without
    a GPU.  The context handle is an opaque non-NULL buffer that these paths never dereference."""
    import torch
    L = _lib.load_library()
    inv = -1
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)
    good = _lib.GridBox(0, 0, 60, 60)
    f = np.float32([1.0, 2.0])
    out = _lib.GridBox()

    def box(n=2, x=f, y=f, reso=1.0, o=C.byref(out)):
        return L.crb_grid_box_of_obstacles(n, None if x is None else x.ctypes.data, None if y is None else y.ctypes.data,
                                           reso, o)

    def omap(**over):
        a = dict(dict(ctx=ctx, n=5, ox=d, oy=d, reso=1.0, rr=1.0, box=C.byref(good), map=d), **over)
        return L.crb_grid_obstacle_map(a["ctx"], a["n"], a["ox"], a["oy"], a["reso"], a["rr"], a["box"], a["map"])

    def plan(**over):
        a = dict(dict(ctx=ctx, algo=0, box=C.byref(good), map=d, reso=1.0, n=5, sg=d, mp=4, path=d), **over)
        return L.crb_grid_plan_batched(a["ctx"], a["algo"], a["box"], a["map"], a["reso"], a["n"], a["sg"], a["mp"],
                                       a["path"], d, d, d, d)
    assert box() == 0
    for kw in (dict(n=0), dict(x=None), dict(o=None), dict(reso=0.0), dict(reso=-1.0), dict(reso=float("nan")),
               dict(reso=float("inf")), dict(x=np.float32([np.nan, 1])), dict(y=np.float32([1, 3e9]))):
        assert box(**kw) == inv, kw
    assert box(x=np.float32([1, 2.1e9])) == 0 and box(x=np.float32([1, 2.2e9])) == inv
    bad_boxes = [_lib.GridBox(0, 0, 0, 5), _lib.GridBox(3, 0, 2, 5), _lib.GridBox(0, 0, 32769, 1),
                 _lib.GridBox(0, 0, 4097, 4096), _lib.GridBox(-2147483648, 0, 2147483647, 2)]
    for b in bad_boxes:
        assert omap(box=C.byref(b)) == inv and plan(box=C.byref(b)) == inv
        assert L.crb_grid_plan_slots(ctx, 0, C.byref(b), 5, C.byref(C.c_int64())) == inv
    for kw in (dict(ctx=None), dict(n=-1), dict(reso=0.0), dict(reso=float("nan")), dict(rr=float("nan")),
               dict(rr=float("inf")), dict(box=None), dict(map=None), dict(ox=None)):
        assert omap(**kw) == inv, kw
    for kw in (dict(ctx=None), dict(algo=2), dict(algo=-1), dict(reso=0.0), dict(reso=float("inf")), dict(n=-1),
               dict(mp=-1), dict(box=None), dict(map=None), dict(sg=None), dict(path=None)):
        assert plan(**kw) == inv, kw
    assert L.crb_grid_plan_slots(ctx, 2, C.byref(good), 5, C.byref(C.c_int64())) == inv
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert omap() == nd and plan() == nd and plan(n=0, map=None, sg=None, path=None) == nd
        assert plan(path=None, mp=0) == nd and omap(n=0, ox=None, oy=None) == nd
        assert plan(box=C.byref(_lib.GridBox(-5, 7, 32763, 8))) == nd   # a 32768 x 1 box is within the limits
        assert b"no CPU fallback" in L.crb_last_error_string()
        assert L.crb_grid_plan_slots(ctx, 1, C.byref(good), 5, C.byref(C.c_int64())) == nd


def _build_api(tmp_path):
    exe = str(tmp_path / "grid_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           CPP_API, "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


def test_reference_style_program_compiles(tmp_path):
    _build_api(tmp_path)


def test_new_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-c", os.path.join(ROOT, "cpprobotics_b200", "csrc", "crb_grid.cu"),
                          "-o", str(tmp_path / "grid.o")], capture_output=True, text=True, check=True).stderr
    blocks = out.split("Compiling entry function")[1:]
    kernels = [b for b in blocks if "crb_grid_" in b.splitlines()[0]]
    assert len(kernels) == 3
    for b in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in b and "0 bytes stack frame" in b, b


# ---- H100 -----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _box(b):
    return _lib.GridBox(*[int(v) for v in b])


def _maps():
    """name -> (ox, oy, reso, rr): the demo and the seeded 128 x 128 scatter"""
    ox, oy, reso, rr, _ = GC.demo()
    sx, sy = synth.grid_scatter_obstacles(128)
    return {"demo": (ox, oy, reso, rr), "scatter128": (sx, sy, 1.0, 1.0)}


def _gpu_map(engine, ox, oy, reso, rr, box):
    return engine.grid_obstacle_map(_dev(ox), _dev(oy), reso, rr, _box(box)).cpu().numpy()


def _gpu_plan(engine, algo, box, m, reso, sg, max_pts):
    r = engine.grid_plan(algo, _box(box), _dev(m), reso, _dev(sg), max_pts=max_pts)
    return {k: (None if v is None else v.cpu().numpy()) for k, v in r.items()}


KEYS = ("path", "path_len", "cost", "n_visited", "status")


@pytest.mark.gpu
def test_gpu_obstacle_map_is_bitwise_the_checker(engine):
    cases = [GC.demo()[:4]] + [c[1:5] for c in GC.corner_cases()]
    for side, per, reso, rr in ((128, 1 / 40, 1.0, 1.0), (300, 1 / 30, 0.5, 0.8), (512, 1 / 64, 1.0, 2.5),
                                (512, 1 / 20, 2.0, 0.0)):
        ox, oy = synth.grid_scatter_obstacles(side, reso, per, seed=side + int(1 / per))
        cases.append((ox, oy, reso, rr))
    ox, oy = synth.grid_scatter_obstacles(200, 1.0, 1 / 50)
    cases.append((np.concatenate([ox, [np.nan, 3e9]]).astype(np.float32), np.concatenate([oy, [5, 5]]).astype(np.float32),
                  1.0, 1.5))   # two obstacles that round to nothing block nothing
    for ox, oy, reso, rr in cases:
        box = OG.box_of_obstacles(ox[np.isfinite(ox) & (np.abs(ox) < 1e9)], oy[np.isfinite(ox) & (np.abs(ox) < 1e9)],
                                  reso)
        want = OG.obstacle_map(ox, oy, reso, rr, box)
        assert np.array_equal(_gpu_map(engine, ox, oy, reso, rr, box), want), (len(ox), reso, rr)
    assert len(cases[-2][0]) > 13000 and want.any() and not want.all()


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
@pytest.mark.parametrize("which", ["demo", "scatter128"])
def test_gpu_plan_is_bitwise_the_checker(engine, algo, n, which):
    ox, oy, reso, rr = _maps()[which]
    box, m = _setup(ox, oy, reso, rr)
    assert np.array_equal(_gpu_map(engine, ox, oy, reso, rr, box), m)
    sg = synth.grid_inputs(n, box, m, reso, seed=0x900 + n)
    o = OG.plan(algo, box, m, reso, sg, max_pts=64)
    r = _gpu_plan(engine, algo, box, m, reso, sg, 64)
    for k in KEYS:
        assert same(r[k], o[k]), k
    if n >= 4097:
        st = np.bincount(o["status"], minlength=4)
        assert st[OG.FOUND] > 0.9 * n and st[OG.NO_PATH] > 0 and st[OG.START_OUTSIDE] > 0 and st[OG.BAD_POINT] > 0
        assert (o["path_len"] > 64).any()   # paths longer than the buffer: path_len still counts them


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGO_IDS)
def test_gpu_more_queries_than_slots(engine, algo):
    ox, oy = synth.grid_scatter_obstacles(256, 1.0, 1 / 40, seed=77)
    box, m = _setup(ox, oy, 1.0, 1.0)
    slots = engine.grid_plan_slots(algo, _box(box), 1 << 20)
    assert 1 <= slots < 4096
    n = 2 * slots + 1
    sg = synth.grid_inputs(n, box, m, 1.0, seed=78)
    o = OG.plan(algo, box, m, 1.0, sg, max_pts=32)
    r = _gpu_plan(engine, algo, box, m, 1.0, sg, 32)
    for k in KEYS:
        assert same(r[k], o[k]), k
    assert engine.grid_plan_slots(algo, _box(box), 7) == 7


@pytest.mark.gpu
def test_gpu_short_path_buffers_empty_batches_split_batches_and_a_graph(engine):
    import torch
    ox, oy, reso, rr, _ = GC.demo()
    box, m = _setup(ox, oy, reso, rr)
    sg = synth.grid_inputs(3000, box, m, reso, seed=5)
    md = _dev(m)
    for algo in ALGO_IDS:
        o = OG.plan(algo, box, m, reso, sg, max_pts=3)
        r = _gpu_plan(engine, algo, box, m, reso, sg, 3)
        assert all(same(r[k], o[k]) for k in KEYS) and (o["path_len"] > 3).any()
        # outputs requested one at a time, path without max_pts
        full = OG.plan(algo, box, m, reso, sg)
        sgd = _dev(sg)
        for k in ("path_len", "cost", "n_visited", "status"):
            buf = torch.empty(3000, dtype=torch.float32 if k == "cost" else torch.int32, device="cuda:0")
            res = engine.grid_plan(algo, _box(box), md, reso, sgd, **{k: buf})
            assert same(res[k].cpu().numpy(), full[k]), k
        # two launches over the halves give the same bits as one
        a = _gpu_plan(engine, algo, box, m, reso, np.ascontiguousarray(sg[:, :1234]), 16)
        b = _gpu_plan(engine, algo, box, m, reso, np.ascontiguousarray(sg[:, 1234:]), 16)
        w = _gpu_plan(engine, algo, box, m, reso, sg, 16)
        for k in KEYS:
            assert same(np.concatenate([a[k], b[k]], axis=-1), w[k]), k
        # n = 0 enqueues nothing
        e = engine.grid_plan(algo, _box(box), md, reso, torch.empty((4, 0), device="cuda:0"), max_pts=4)
        assert e["status"].shape == (0,) and e["path"].shape == (8, 0)
        # a launch captured in a CUDA graph after a warm call at this map size
        out = {k: torch.full_like(v, -1) for k, v in engine.grid_plan(algo, _box(box), md, reso, sgd, max_pts=8).items()}
        torch.cuda.synchronize()
        for v in out.values():   # path slots past path_len are left as they are: NaN, as the checker's
            v.fill_(float("nan") if v.is_floating_point() else -1)
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            engine.bind_current_stream()
            with torch.cuda.graph(g, stream=s):
                engine.grid_plan(algo, _box(box), md, reso, sgd, max_pts=8, **out)
        engine.bind_current_stream()
        g.replay()
        torch.cuda.synchronize()
        want = OG.plan(algo, box, m, reso, sg, max_pts=8)
        for k in KEYS:
            assert same(out[k].cpu().numpy(), want[k]), k
    with pytest.raises(_lib.CrbError):
        engine.grid_plan(2, _box(box), md, reso, _dev(sg))


@pytest.mark.gpu
def test_gpu_reproduces_the_golden_fixture(engine):
    d = np.load(GOLDEN)
    for algo, name in GC.ALGOS:
        ox, oy, reso, rr, sg = GC.demo()
        box, _ = _setup(ox, oy, reso, rr)
        m = _gpu_map(engine, ox, oy, reso, rr, box)
        assert np.array_equal(np.argwhere(m != 0), d[f"demo_{name}_map_cells"])
        r = _gpu_plan(engine, algo, box, m, reso, sg, 256)
        assert same(_path_cells(r, 0, reso), d[f"demo_{name}_path"].astype(np.float32) * np.float32(reso))
        p = o = 0
        for no, pl in zip(d[f"seeded_{name}_n_obs"], d[f"seeded_{name}_path_len"]):
            v = d[f"seeded_{name}_inputs"][p:p + 6 + 2 * no]
            p += 6 + 2 * no
            box = OG.box_of_obstacles(v[6:6 + no], v[6 + no:], v[0])
            m = _gpu_map(engine, v[6:6 + no], v[6 + no:], v[0], v[1], box)
            r = _gpu_plan(engine, algo, box, m, v[0], v[2:6].reshape(4, 1), int(pl))
            want = d[f"seeded_{name}_path"][o:o + pl].astype(np.float32) * np.float32(v[0])
            o += pl
            assert r["status"][0] == OG.FOUND and same(_path_cells(r, 0, v[0]), want)


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_checker(tmp_path):
    exe = _build_api(tmp_path)
    subprocess.check_call([exe, str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    ox, oy, reso, rr, _ = GC.demo()
    box, m = _setup(ox, oy, reso, rr)
    single = np.float32([[10], [10], [50], [50]])
    batch = np.float32([[10, 5, 30], [10, 55, 30], [50, 55, 30], [50, 5, 30]])
    p = 0
    for algo, sg in ((0, single), (1, single), (0, batch), (1, batch)):
        r = OG.plan(algo, box, m, reso, sg, max_pts=512)
        for q in range(sg.shape[1]):
            n = int(out[p]); p += 1
            assert n == r["path_len"][q]
            pts = _path_cells(r, q, reso)
            assert same(out[p:p + n], pts[:, 0]) and same(out[p + n:p + 2 * n], pts[:, 1])
            p += 2 * n
    assert p == out.size
