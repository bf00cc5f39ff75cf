"""RRT (include/rrt.h).
CPU: the checker's mt19937 and both distributions are libstdc++'s (crafted values included), its atanf is the host
atanf on every non-negative float and its atan2f the host atan2f on dense pairs and every special quadrant; the checker
is bitwise the reference's own text (tree, parents, path, draws) on the demo, scattered maps, corner cases and the
rare-branch seeds; the golden fixture; statuses where the reference is undefined; layouts, validation without a device,
the reference-style program compiles, and the kernel does not spill.  H100: crb_rrt_plan_batched is bitwise the checker
(every output, batch sizes, maps, truncation, NULL outputs, split batches, a CUDA graph, the max_iter limits, the
rare-branch seeds), crb_atan2f_libm is the checker's, the golden fixture, and the reference-style C++ program."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rrt_cases as RC
from cpprobotics_b200 import _lib, rrt_default_params, synth
from oracle import rrt as OR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "rrt_golden.npz")
CPP_API = os.path.join(ROOT, "tests", "cpp", "rrt_ref_api.cpp")
CPP_PIN = os.path.join(ROOT, "tests", "cpp", "rrt_dist_pin.cpp")
DEMO = synth.RRT_DEMO
KEYS = ("path", "path_len", "tree", "parent", "n_nodes", "n_iter", "status")


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _ref():
    L = RC.ref_lib()
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
    return L


@pytest.fixture(scope="module")
def pin(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("pin") / "rrt_dist_pin")
    subprocess.check_call(["g++", "-std=c++11", "-O2", "-Wall", "-Werror", CPP_PIN, "-o", exe])

    def run(mode, values, *extra):
        d = tmp_path_factory.mktemp("io")
        np.ascontiguousarray(values, np.uint32).tofile(d / "in.bin")
        subprocess.check_call([exe, mode, str(d / "in.bin"), str(d / "out.bin")] + [str(x) for x in extra])
        return np.fromfile(d / "out.bin", np.uint32)
    return run


def _demo_se(n=1):
    return np.tile(np.float32([[DEMO["sx"]], [DEMO["sy"]], [DEMO["gx"]], [DEMO["gy"]]]), (1, n))


def _same_run(c, r):
    return (same(c["tree"], r["tree"]) and np.array_equal(c["parent"], r["parent"]) and same(c["path"], r["path"])
            and c["draws"] == r["draws"])


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_mt19937_is_std_mt19937(pin):
    seeds = np.uint32([0, 1, 5489, 0xFFFFFFFF, 0x80000000, 12345, 0xDEADBEEF, 7, 624, 4242424242])
    want = pin("mt", seeds).reshape(seeds.size, 100000)
    for s, w in zip(seeds, want):
        assert np.array_equal(OR.mt_run(int(s), 100000), w), s


def test_distributions_are_libstdcxx_on_crafted_values(pin):
    rng = np.random.default_rng(0xD157)
    inv101 = pow(101, -1, 1 << 32)
    low = np.uint32([(k * inv101) % (1 << 32) for k in range(68)])          # low word k < 68: a redraw
    edge = np.uint32([(k * inv101) % (1 << 32) for k in range(68, 110)])     # 68 <= low < 110: no redraw
    top = np.arange(0xFFFFFF00, 0x100000000, dtype=np.uint64).astype(np.uint32)   # around 2^32 - 128
    u = np.concatenate([rng.integers(0, 1 << 32, 4000, dtype=np.uint64).astype(np.uint32), low, edge, top,
                        np.uint32([0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFF7F, 0xFFFFFF80])])
    u = u[rng.permutation(u.size)]
    u = np.concatenate([u, low[:5]])   # redraws at the very end: the last draw runs dry
    got, used = OR.dist_run(0, u)
    want = pin("int", u).reshape(-1, 2)
    assert np.array_equal(got, want[:, 0]) and np.array_equal(used, want[:, 1].astype(np.int32))
    assert (used > 1).sum() > 50 and got.max() == 100 and got.min() == 0
    for a, b in ((-2.0, 15.0), (0.0, 1.0), (-1e30, 3e30), (5.0, 5.0), (-7.25, -0.5)):
        got, used = OR.dist_run(1, u, a, b)
        want = pin("real", u, repr(a), repr(b)).reshape(-1, 2)
        assert np.array_equal(got, want[:, 0]) and (used == 1).all() and used.size == u.size, (a, b)
    got, _ = OR.dist_run(1, top, 0.0, 1.0)
    assert (got[top >= 0xFFFFFF80] == 0x3F7FFFFF).all()   # nextafterf(1, 0)


def test_atanf_is_the_host_atanf_on_every_non_negative_float():
    assert OR.atanf_census(0, 0x80000000) == 0


def test_atan2f_is_the_host_atan2f_on_pairs_and_every_special_quadrant():
    rng = np.random.default_rng(0xA7A2)
    n = 4_000_000
    mag = lambda: rng.choice(np.float32([1e-30, 1e-6, 1e-2, 1, 10, 1e3, 1e8, 1e30]), n)  # noqa: E731
    y = (rng.standard_normal(n) * mag()).astype(np.float32)
    x = (rng.standard_normal(n) * mag()).astype(np.float32)
    assert OR.atan2f_pairs(y, x) == 0
    bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    assert OR.atan2f_pairs(bits.view(np.float32), np.roll(bits, 1).view(np.float32)) == 0   # any bit patterns
    sp = np.float32([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 3.0, -2.5, 1e-40, -1e-40, 3e38, -3e38, 1e-20,
                     1e20, 2.0 ** 61, -(2.0 ** -61)])
    Y, X = np.meshgrid(sp, sp)
    assert OR.atan2f_pairs(Y.ravel(), X.ravel()) == 0
    z = rng.standard_normal(100000).astype(np.float32)
    assert OR.atan2f_pairs(z, np.ones_like(z)) == 0   # the x == 1 shortcut


def test_demo_is_bitwise_the_reference_text_for_2000_seeds():
    L = _ref()
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    for s in range(1, 2001):
        c = RC.checker_one(prm, ob, DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"], s)
        assert c["status"] == OR.FOUND, s
        r = RC.ref_run(L, prm, ob, DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"], s, prm["max_iter"] + 1)
        assert r is not None and _same_run(c, r), s


def test_rare_branch_seeds_are_bitwise_the_reference_text():
    L = _ref()
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    seeds = RC.REDRAW_SEEDS + RC.CANONICAL_ONE_SEEDS
    o = OR.plan(prm, ob, _demo_se(len(seeds)), np.uint32(seeds))
    k = len(RC.REDRAW_SEEDS)
    assert ((o["branches"][:k] & 1) != 0).all() and ((o["branches"][k:] & 2) != 0).all()
    for s in seeds:
        c = RC.checker_one(prm, ob, DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"], s)
        r = RC.ref_run(L, prm, ob, DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"], s, prm["max_iter"] + 1)
        assert c["status"] == OR.FOUND and _same_run(c, r), s


def test_scattered_maps_are_bitwise_the_reference_text():
    L = _ref()
    done = 0
    for prm, ob, sx, sy, gx, gy, seed in RC.scattered_maps(80, seed=0x5EED):
        c = RC.checker_one(prm, ob, sx, sy, gx, gy, seed)
        if c["status"] != OR.FOUND:
            continue
        r = RC.ref_run(L, prm, ob, sx, sy, gx, gy, seed, prm["max_iter"] + 1)
        assert r is not None and _same_run(c, r), seed
        done += 1
    assert done >= 60


@pytest.mark.parametrize("case", ["start_is_goal", "start_inside_obstacle", "goal_sample_rate_100"])
def test_corner_cases_are_bitwise_the_reference_text(case):
    L = _ref()
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    sx, sy, gx, gy = DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"]
    if case == "start_is_goal":
        gx, gy = sx, sy
    elif case == "start_inside_obstacle":
        sx, sy = 5.0, 4.3   # 0.7 from the centre of the obstacle (5, 5, 1)
    else:
        prm = dict(prm, goal_sample_rate=100)   # always the goal: a straight run past the obstacles
        sx, sy, gx, gy = -2.0, 12.0, 6.0, 14.0
    for s in range(1, 41):
        c = RC.checker_one(prm, ob, sx, sy, gx, gy, s)
        assert c["status"] == OR.FOUND, s
        r = RC.ref_run(L, prm, ob, sx, sy, gx, gy, s, prm["max_iter"] + 1)
        assert _same_run(c, r), s
    if case == "start_is_goal":   # atan2f(0, 0) = 0 when the goal is drawn
        assert OR.atan2f(0.0, 0.0) == 0.0


def test_oracle_reproduces_the_golden_fixture():
    d = np.load(GOLDEN)
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    t = p = 0
    for s, (nn, pl) in enumerate(zip(d["demo_n_nodes"], d["demo_path_len"]), start=1):
        c = RC.checker_one(prm, ob, DEMO["sx"], DEMO["sy"], DEMO["gx"], DEMO["gy"], s)
        assert same(c["tree"], d["demo_tree"][t:t + nn]) and np.array_equal(c["parent"], d["demo_parent"][t:t + nn])
        assert same(c["path"], d["demo_path"][p:p + pl])
        t, p = t + nn, p + pl
    assert s == 32
    i = p = 0
    for no, pl in zip(d["scattered_n_ob"], d["scattered_path_len"]):
        v = d["scattered_inputs"][i:i + 9 + 3 * no]
        i += 9 + 3 * no
        prm = dict(rand_min=v[0], rand_max=v[1], expand_dis=v[2], goal_sample_rate=int(v[3]), max_iter=8192)
        c = RC.checker_one(prm, v[9:].reshape(no, 3), *v[4:8], int(v[8:9].view(np.uint32)[0]))
        assert c["status"] == OR.FOUND and same(c["path"], d["scattered_path"][p:p + pl])
        p += pl
    assert len(d["scattered_n_ob"]) == 16


def test_checker_statuses_where_the_reference_is_undefined():
    ob = synth.rrt_demo_obstacles()
    prm = RC.demo_prm(max_iter=300)
    # a goal inside an obstacle's reach only through it, a goal enclosed, NaN / inf points
    se = np.float32([[0, 0, np.nan, 0, 0, 0],
                     [0, 0, 0, np.inf, 0, 0],
                     [6, 5, 6, 6, 6, 6],
                     [9, 5, 9, 9, 9, 9]])
    o = OR.plan(prm, ob, se, np.uint32([1, 2, 3, 4, 5, 6]), max_pts=8, max_nodes=400)
    assert o["status"].tolist()[:4] == [OR.FOUND, OR.MAX_ITER, OR.BAD_INPUT, OR.BAD_INPUT]
    assert (o["n_iter"][1] == 300) and o["n_nodes"][1] > 1 and o["path_len"][1] == 0 and np.isnan(o["path"][:, 1]).all()
    assert (o["n_nodes"][1] == (o["parent"][:, 1] >= 0).sum() + 1) and o["parent"][0, 1] == -1
    assert (o["n_nodes"][[2, 3]] == 0).all() and (o["n_iter"][[2, 3]] == 0).all() and (o["path_len"][[2, 3]] == 0).all()
    # a non-finite obstacle makes every query BAD_INPUT
    bad = ob.copy()
    bad[3, 2] = np.inf
    assert (OR.plan(prm, bad, se, np.uint32([1, 2, 3, 4, 5, 6]))["status"] == OR.BAD_INPUT).all()
    # a rand area so wide that every distance overflows: no nearest node
    wide = dict(prm, rand_min=-3e38, rand_max=3e38, goal_sample_rate=-1)
    w = OR.plan(wide, ob, _demo_se(8), np.arange(8, dtype=np.uint32))
    assert (w["status"] == OR.BAD_INPUT).any() and (w["n_iter"] >= 1).all()
    # max_iter = 1: one pass
    one = OR.plan(dict(prm, max_iter=1), ob, _demo_se(64), np.arange(64, dtype=np.uint32))
    assert (one["n_iter"] == 1).all() and (one["status"] == OR.MAX_ITER).all() and set(one["n_nodes"]) <= {1, 2}


def test_params_and_layout_on_the_host(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){crb_rrt_params p;'
                   'crb_rrt_default_params(&p);printf("%zu %zu %zu %zu %zu %d %d %d %d %g %g %g %d %d\\n",'
                   'sizeof(crb_rrt_params),offsetof(crb_rrt_params,rand_max),offsetof(crb_rrt_params,expand_dis),'
                   'offsetof(crb_rrt_params,goal_sample_rate),offsetof(crb_rrt_params,max_iter),CRB_RRT_MAX_ITER,'
                   'CRB_RRT_FOUND,CRB_RRT_MAX_ITER_REACHED,CRB_RRT_BAD_INPUT,p.rand_min,p.rand_max,p.expand_dis,'
                   'p.goal_sample_rate,p.max_iter);return 0;}\n')
    exe = tmp_path / "sz"
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe), "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}"])
    got = subprocess.check_output([str(exe)]).split()
    P = _lib.RrtParams
    assert [int(x) for x in got[:5]] == [C.sizeof(P), P.rand_max.offset, P.expand_dis.offset,
                                         P.goal_sample_rate.offset, P.max_iter.offset]
    assert [int(x) for x in got[5:9]] == [_lib.CRB_RRT_MAX_ITER, _lib.CRB_RRT_FOUND, _lib.CRB_RRT_MAX_ITER_REACHED,
                                          _lib.CRB_RRT_BAD_INPUT]
    assert [int(x) for x in got[5:9]] == [OR.MAX_ITER_LIMIT, OR.FOUND, OR.MAX_ITER, OR.BAD_INPUT]
    assert [float(x) for x in got[9:12]] == [-2.0, 15.0, 1.0] and [int(x) for x in got[12:]] == [5, 500]
    p = rrt_default_params()
    assert (p.rand_min, p.rand_max, p.expand_dis, p.goal_sample_rate, p.max_iter) == (-2.0, 15.0, 1.0, 5, 500)


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE on a machine without
    a GPU.  The context handle is an opaque non-NULL buffer that these paths never dereference."""
    import torch
    L = _lib.load_library()
    inv = -1
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)

    def plan(prm_over=None, **over):
        p = rrt_default_params()
        for k, v in (prm_over or {}).items():
            setattr(p, k, v)
        a = dict(dict(ctx=ctx, prm=C.byref(p), ob=d, n_ob=6, n=5, se=d, seed=d, mp=4, path=d, mn=4, tree=d), **over)
        return L.crb_rrt_plan_batched(a["ctx"], a["prm"], a["ob"], a["n_ob"], a["n"], a["se"], a["seed"], a["mp"],
                                      a["path"], d, a["mn"], a["tree"], d, d, d, d)
    nan, inf = float("nan"), float("inf")
    for po in (dict(rand_min=nan), dict(rand_max=inf), dict(rand_min=-inf), dict(rand_min=3.0, rand_max=2.0),
               dict(expand_dis=nan), dict(expand_dis=inf), dict(max_iter=0), dict(max_iter=-5),
               dict(max_iter=_lib.CRB_RRT_MAX_ITER + 1)):
        assert plan(po) == inv, po
    for kw in (dict(ctx=None), dict(prm=None), dict(n=-1), dict(n_ob=-1), dict(mp=-1), dict(mn=-1), dict(se=None),
               dict(seed=None), dict(ob=None)):
        assert plan(**kw) == inv, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert plan() == nd and plan(n=0, se=None, seed=None, ob=None) == nd and plan(ob=None, n_ob=0) == nd
        assert plan(dict(max_iter=_lib.CRB_RRT_MAX_ITER, rand_min=5.0, rand_max=5.0, expand_dis=-1.0)) == nd
        assert plan(path=None, tree=None) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def _build_api(tmp_path):
    exe = str(tmp_path / "rrt_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           CPP_API, "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


def test_reference_style_program_compiles(tmp_path):
    _build_api(tmp_path)


def test_new_kernel_does_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-c", os.path.join(ROOT, "cpprobotics_b200", "csrc", "crb_rrt.cu"),
                          "-o", str(tmp_path / "rrt.o")], capture_output=True, text=True, check=True).stderr
    blocks = out.split("Compiling entry function")[1:]
    kernels = [b for b in blocks if "crb_rrt_plan_kernel" in b.splitlines()[0]]
    assert len(kernels) == 1
    assert "0 bytes spill stores, 0 bytes spill loads" in kernels[0] and "0 bytes stack frame" in kernels[0]
    for b in out.split("Function properties for")[1:]:   # the out-of-line atanf / sin-cos reduction too
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in b.splitlines()[1], b


# ---- H100 -----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _params(prm):
    p = rrt_default_params()
    for k in ("rand_min", "rand_max", "expand_dis", "goal_sample_rate", "max_iter"):
        setattr(p, k, prm[k])
    return p


def _gpu(engine, prm, ob, se, seed, max_pts=64, max_nodes=512, **kw):
    r = engine.rrt_plan(_dev(ob), _dev(se), _dev(np.asarray(seed, np.uint32).view(np.int32)), _params(prm),
                        max_pts=max_pts, max_nodes=max_nodes, **kw)
    return {k: (None if v is None else v.cpu().numpy()) for k, v in r.items()}


def _maps():
    """name -> (prm, ob, lo, hi): the demo, and a dense seeded map of 64 obstacles over [-20, 40)^2"""
    dense = synth.rrt_scatter_obstacles(64, -20.0, 40.0)
    return {"demo": (RC.demo_prm(), synth.rrt_demo_obstacles(), DEMO["rand_min"], DEMO["rand_max"]),
            "dense64": (dict(rand_min=-20.0, rand_max=40.0, expand_dis=1.0, goal_sample_rate=5, max_iter=4096), dense,
                        -20.0, 40.0)}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 4096, 65536])
@pytest.mark.parametrize("which", ["demo", "dense64"])
def test_gpu_plan_is_bitwise_the_checker(engine, n, which):
    prm, ob, lo, hi = _maps()[which]
    se, seed = synth.rrt_inputs(n, ob, lo, hi, seed=0x700 + n)
    o = OR.plan(prm, ob, se, seed, max_pts=64, max_nodes=512)
    r = _gpu(engine, prm, ob, se, seed)
    for k in KEYS:
        assert same(r[k], o[k]), k
    if n >= 4096:
        assert (o["status"] == OR.FOUND).mean() > 0.9
        assert (o["path_len"] > 64).any() or (o["n_nodes"] > 512).any()   # truncated buffers are exercised


@pytest.mark.gpu
def test_gpu_rare_branch_seeds_and_max_iter_limits(engine):
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    seeds = np.uint32(RC.REDRAW_SEEDS + RC.CANONICAL_ONE_SEEDS)
    for p in (prm, dict(prm, max_iter=1), dict(prm, max_iter=_lib.CRB_RRT_MAX_ITER), dict(prm, max_iter=300)):
        o = OR.plan(p, ob, _demo_se(seeds.size), seeds, max_pts=128, max_nodes=p["max_iter"] + 1)
        r = _gpu(engine, p, ob, _demo_se(seeds.size), seeds, max_pts=128, max_nodes=p["max_iter"] + 1)
        for k in KEYS:
            assert same(r[k], o[k]), (p["max_iter"], k)
    # statuses where the reference is undefined, and a non-finite obstacle
    se = np.float32([[0, 0, np.nan, 0], [0, 0, 0, np.inf], [6, 5, 6, 6], [9, 5, 9, 9]])
    wide = dict(prm, rand_min=-3e38, rand_max=3e38, goal_sample_rate=-1, max_iter=300)
    bad = ob.copy()
    bad[0, 0] = np.nan
    for p, o_ in ((dict(prm, max_iter=300), ob), (wide, ob), (prm, bad)):
        sd = np.arange(4, dtype=np.uint32)
        o = OR.plan(p, o_, se, sd, max_pts=16, max_nodes=301)
        r = _gpu(engine, p, o_, se, sd, max_pts=16, max_nodes=301)
        for k in KEYS:
            assert same(r[k], o[k]), k


@pytest.mark.gpu
def test_gpu_null_outputs_empty_and_split_batches_and_a_graph(engine):
    import torch
    prm, ob, lo, hi = _maps()["demo"]
    se, seed = synth.rrt_inputs(3000, ob, lo, hi, seed=5)
    full = OR.plan(prm, ob, se, seed, max_pts=8, max_nodes=40)
    obd, sed, sdd = _dev(ob), _dev(se), _dev(seed.view(np.int32))
    p = _params(prm)
    # outputs requested one at a time, the others NULL
    for k in ("path_len", "n_nodes", "n_iter", "status"):
        buf = torch.empty(3000, dtype=torch.int32, device="cuda:0")
        res = engine.rrt_plan(obd, sed, sdd, p, **{k: buf})
        assert same(res[k].cpu().numpy(), full[k]) and res["path"] is None and res["tree"] is None, k
    only_tree = engine.rrt_plan(obd, sed, sdd, p, max_nodes=40)
    assert same(only_tree["tree"].cpu().numpy(), full["tree"]) and same(only_tree["parent"].cpu().numpy(), full["parent"])
    # two launches over the parts give the same bits as one
    a = _gpu(engine, prm, ob, se[:, :1234], seed[:1234], 8, 40)
    b = _gpu(engine, prm, ob, se[:, 1234:], seed[1234:], 8, 40)
    for k in KEYS:
        assert same(np.concatenate([a[k], b[k]], axis=-1), full[k]), k
    # n = 0 enqueues nothing
    e = engine.rrt_plan(obd, torch.empty((4, 0), device="cuda:0"), torch.empty(0, dtype=torch.int32, device="cuda:0"),
                        p, max_pts=4)
    assert e["status"].shape == (0,) and e["path"].shape == (8, 0)
    # a launch captured in a CUDA graph (the counter exists after the calls above)
    out = {k: torch.full_like(v, -1) for k, v in engine.rrt_plan(obd, sed, sdd, p, max_pts=8, max_nodes=40).items()}
    torch.cuda.synchronize()
    for v in out.values():
        v.fill_(float("nan") if v.is_floating_point() else -1)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        engine.bind_current_stream()
        with torch.cuda.graph(g, stream=s):
            engine.rrt_plan(obd, sed, sdd, p, max_pts=8, max_nodes=40, **out)
    engine.bind_current_stream()
    g.replay()
    torch.cuda.synchronize()
    for k in KEYS:
        assert same(out[k].cpu().numpy(), full[k]), k
    with pytest.raises(_lib.CrbError):
        engine.rrt_plan(obd, sed, sdd, _params(dict(prm, max_iter=0)))


ATAN2F_CU = r"""
// crb_atan2f_libm on the device: mode 0 gives atanf (atan2f(y, 1)) for every non-negative float in [lo, hi), in chunks,
// checked by the checker's crb_oracle_rrt_atanf_check; mode 1 gives atan2f of the pairs in argv[4] (y[n], x[n] as
// float32), checked by crb_oracle_rrt_atan2f_check (argv[3] = liboracle_rrt.so).  Prints the number of mismatches.
#include <dlfcn.h>
#include <vector>

#include "crb_common.cuh"
__global__ void atanf_k(unsigned lo, unsigned long long count, float* out) {
  for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x)
    out[k] = crb_atan2f_libm(__uint_as_float(lo + (unsigned)k), 1.0f);
}
__global__ void atan2f_k(long long n, const float* y, const float* x, float* out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
    out[k] = crb_atan2f_libm(y[k], x[k]);
}
int main(int argc, char** argv) {
  if (argc < 4) return 2;
  void* so = dlopen(argv[3], RTLD_NOW);
  if (!so) return 2;
  long long bad = 0;
  if (argv[1][0] == '0') {
    const unsigned lo = (unsigned)strtoul(argv[2], 0, 0), hi = 0x80000000u;
    typedef long long (*check_fn)(unsigned, unsigned, const float*);
    check_fn check = (check_fn)dlsym(so, "crb_oracle_rrt_atanf_check");
    const unsigned chunk = 1u << 27;
    float *d, *h;
    if (!check || cudaMalloc(&d, chunk * 4ull) != cudaSuccess || cudaMallocHost(&h, chunk * 4ull) != cudaSuccess) return 3;
    for (unsigned a = lo; a < hi; a = (hi - a > chunk) ? a + chunk : hi) {
      const unsigned b = (hi - a > chunk) ? a + chunk : hi;
      atanf_k<<<2048, 256>>>(a, b - a, d);
      if (cudaMemcpy(h, d, (b - a) * 4ull, cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
      bad += check(a, b, h);
    }
  } else {
    FILE* f = fopen(argv[4], "rb");
    if (!f) return 2;
    std::vector<float> v;
    float t;
    while (fread(&t, 4, 1, f) == 1) v.push_back(t);
    fclose(f);
    const long long n = (long long)v.size() / 2;
    typedef long long (*check_fn)(long long, const float*, const float*, const float*);
    check_fn check = (check_fn)dlsym(so, "crb_oracle_rrt_atan2f_check");
    float* d;
    if (!check || cudaMalloc(&d, v.size() * 4 + n * 4) != cudaSuccess) return 3;
    cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    atan2f_k<<<2048, 256>>>(n, d, d + n, d + 2 * n);
    std::vector<float> out(n);
    if (cudaMemcpy(out.data(), d + 2 * n, n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
    bad = check(n, v.data(), v.data() + n, out.data());
  }
  printf("%lld\n", bad);
  return 0;
}
"""


@pytest.mark.gpu
def test_gpu_atan2f_is_the_checkers(tmp_path):
    """crb_atan2f_libm on the device against the checker's restatement (itself pinned to the host libm by the CPU
    tests): atanf on every non-negative float, atan2f on dense pairs and every special quadrant."""
    src = tmp_path / "atan2f.cu"
    src.write_text(ATAN2F_CU)
    exe = tmp_path / "atan2f"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-I", os.path.join(ROOT, "cpprobotics_b200", "csrc"), str(src), "-o", str(exe), "-ldl"])
    assert int(subprocess.check_output([str(exe), "0", "0x0", OR.LIB_PATH], text=True).strip()) == 0
    rng = np.random.default_rng(0xA7A3)
    n = 4_000_000
    bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    y = np.concatenate([(rng.standard_normal(n) * 10).astype(np.float32), bits])
    x = np.concatenate([(rng.standard_normal(n) * 10).astype(np.float32), np.roll(bits, 1)])
    sp = np.float32([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 3.0, -2.5, 1e-40, 3e38, 2.0 ** 61])
    Y, X = np.meshgrid(sp, sp)
    np.concatenate([y, Y.ravel(), x, X.ravel()]).astype(np.float32).tofile(tmp_path / "pairs.bin")
    out = subprocess.check_output([str(exe), "1", "0", OR.LIB_PATH, str(tmp_path / "pairs.bin")], text=True)
    assert int(out.strip()) == 0


@pytest.mark.gpu
def test_gpu_reproduces_the_golden_fixture(engine):
    d = np.load(GOLDEN)
    prm, ob = RC.demo_prm(), synth.rrt_demo_obstacles()
    k = len(d["demo_n_nodes"])
    r = _gpu(engine, prm, ob, _demo_se(k), np.arange(1, k + 1, dtype=np.uint32), max_pts=512, max_nodes=4097)
    t = p = 0
    for q, (nn, pl) in enumerate(zip(d["demo_n_nodes"], d["demo_path_len"])):
        assert r["n_nodes"][q] == nn and r["path_len"][q] == pl
        assert same(r["tree"][:2 * nn, q].reshape(nn, 2), d["demo_tree"][t:t + nn])
        assert np.array_equal(r["parent"][:nn, q], d["demo_parent"][t:t + nn])
        assert same(r["path"][:2 * pl, q].reshape(pl, 2), d["demo_path"][p:p + pl])
        t, p = t + nn, p + pl
    i = p = 0
    for no, pl in zip(d["scattered_n_ob"], d["scattered_path_len"]):
        v = d["scattered_inputs"][i:i + 9 + 3 * no]
        i += 9 + 3 * no
        prm = dict(rand_min=v[0], rand_max=v[1], expand_dis=v[2], goal_sample_rate=int(v[3]), max_iter=8192)
        r = _gpu(engine, prm, v[9:].reshape(no, 3), v[4:8].reshape(4, 1), v[8:9].view(np.uint32), max_pts=int(pl),
                 max_nodes=0)
        assert r["status"][0] == OR.FOUND and same(r["path"][:, 0].reshape(pl, 2), d["scattered_path"][p:p + pl])
        p += pl


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_checker(tmp_path):
    exe = _build_api(tmp_path)
    subprocess.check_call([exe, str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    ob = synth.rrt_demo_obstacles()
    prm = RC.demo_prm(max_iter=_lib.CRB_RRT_MAX_ITER)
    p = 0
    for (sx, sy), s in (((0.0, 0.0), 7), ((0.0, 0.0), 1), ((12.0, 2.0), 2), ((6.0, 9.0), 3)):
        c = RC.checker_one(prm, ob, sx, sy, 6.0, 9.0, s)
        m = int(out[p]); p += 1
        assert c["status"] == OR.FOUND and m == len(c["path"])
        assert same(out[p:p + 2 * m], c["path"].reshape(-1)), s   # and the parent chain is whole (no -1 marks)
        p += 2 * m
    assert p == out.size
