"""State lattice planner (src/state_lattice_planner.cpp): terminal-state samplers, lookup-table search, generate_path.
CPU: the checker is bitwise the reference's own text (the demo's 78 states end to end, seeded queries per sampler,
corner cases of the samplers and the search), slp_load_table is the reference's CSV reading, the golden fixture,
defaults, layouts and argument validation.  H100: crb_slp_sample_states_batched and crb_slp_search_nearest_batched,
and the search + optimizer composition, are bitwise the checker; the golden fixture, shard invariance, n = 0 and the
reference-style C++ program."""
import ctypes as C
import os
import subprocess
from decimal import Decimal, localcontext

import numpy as np
import pytest

import slp_cases as SC
from cpprobotics_b200 import _lib, slp_default_params, slp_load_table, synth
from oracle import mptg as OM
from oracle import slp as OS
from toolchain import build_ref_program, ptxas_kernels, run_layout_probe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "slp_golden.npz")
NAMES = ((OS.UNIFORM, "uniform"), (OS.BIASED, "biased"), (OS.LANE, "lane"))


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN (NaN payloads are not specified by either side)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _ref():
    L = SC.ref_lib()
    if L is None:
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle)")
    return L


def _lib_sampler(s):
    return _lib.SlpSampler(s.kind, s.nxy, s.nh, s.ns, s.d)


# ---- CPU ------------------------------------------------------------------------------------------------------
def _compare_samples(L, s, qp):
    o = OS.sample(s, qp)
    t, cnt = SC.ref_sample(L, s, qp)
    ok = o["status"] == OS.OK   # an out-of-range query is this library's refusal, not the reference's answer
    S = OS.states_per_query(s)
    cols = np.repeat(ok, S)
    assert np.array_equal(o["n_states"][ok], cnt[ok])
    assert same(o["target"][:, cols], t[:, cols])
    assert (o["n_states"][~ok] == 0).all() and np.isnan(o["target"][:, ~cols]).all()
    return o


def test_demo_is_bitwise_the_reference_text_end_to_end():
    L = _ref()
    tb = SC.table()
    total = 0
    for kind, name in NAMES:
        s, qp = SC.demo(kind)
        o = _compare_samples(L, s, qp)
        n = int(o["n_states"][0])
        total += n
        tg = o["target"][:, :n]
        sr = OS.search(tg, tb)
        ref_p = SC.ref_search(L, tg, tb)
        assert same(sr["param"], ref_p) and (sr["row"] >= 0).all()
        g = OS.generate_path(tg, tb, max_pts=256)
        traj, ln = SC.ref_demo(L, kind, tb, 256)
        assert same(g["traj"], traj) and np.array_equal(g["traj_len"], ln), name
        assert (g["status"] == OM.CONVERGED).all() and ln.max() <= 256
    assert total == 78


@pytest.mark.parametrize("kind", [k for k, _ in NAMES])
def test_oracle_is_bitwise_the_reference_text_on_seeded_queries(kind):
    L = _ref()
    fields, qp = synth.slp_inputs(2100, kind, seed=0xA11 + kind)
    o = _compare_samples(L, SC.sampler_of(fields), qp)
    assert (o["status"] == OS.OK).sum() >= 2000 and (o["status"] == OS.OUT_OF_RANGE).sum() > 0
    # the search over every valid state, and generate_path for a sample of the ones the reference defines
    tb = SC.table()
    S = OS.states_per_query(SC.sampler_of(fields))
    fin = np.flatnonzero(np.isfinite(o["target"]).all(axis=0))
    tg = np.ascontiguousarray(o["target"][:, fin])
    assert same(OS.search(tg, tb)["param"], SC.ref_search(L, tg, tb))
    pick = np.ascontiguousarray(tg[:, ::max(1, tg.shape[1] // 96)])
    g = OS.generate_path(pick, tb, max_pts=512)
    keep = np.flatnonzero(g["status"] <= OM.MAX_ITER_REACHED)
    assert len(keep) >= 32   # lanes behind the start often leave the defined cases
    traj, ln = SC.ref_generate_path(L, np.ascontiguousarray(pick[:, keep]), tb, 0.0, 512)
    assert same(g["traj"][:, keep], traj) and np.array_equal(g["traj_len"][keep], ln)
    assert S > 0


@pytest.mark.parametrize("case", [c[0] for c in SC.sampler_sets()])
def test_sampler_corner_cases_are_bitwise_the_reference_text(case):
    L = _ref()
    name, s, qp = next(c for c in SC.sampler_sets() if c[0] == case)
    o = _compare_samples(L, s, qp)
    ok = o["status"] == OS.OK
    if case.endswith("_nxy1") and s.kind != OS.LANE:   # 0 / 0: every angle NaN; the search finds no row
        if s.kind == OS.UNIFORM:
            assert (o["n_states"][ok] == s.nh).all() and np.isnan(o["target"]).all()
            sr = OS.search(o["target"][:, :3], SC.table())
            assert (sr["row"] == -1).all() and np.isnan(sr["param"]).all()
        else:
            assert (o["n_states"] == 0).all()
    if case in ("biased_ns0", "biased_ns1"):
        assert (o["n_states"] == 0).all()
    if case == "biased_duplicates":   # the back-step li = j - 1 lets the scan match the same j again
        t = o["target"][:, :o["n_states"][2]]
        assert len(np.unique(t[0])) < t.shape[1] // s.nh
        assert (o["n_states"][ok] < OS.states_per_query(s)).all()   # late position samples find no j


@pytest.mark.parametrize("case", [c[0] for c in SC.search_sets()])
def test_search_corner_cases_are_bitwise_the_reference_text(case):
    L = _ref()
    name, t, tb = next(c for c in SC.search_sets() if c[0] == case)
    o = OS.search(t, tb)
    assert same(o["param"], SC.ref_search(L, t, tb))
    if case == "equidistant":
        assert o["row"].tolist() == [0]
    elif case == "equal_roots":   # the larger square ties in sqrtf: the first row wins
        assert o["row"].tolist() == [0]
    elif case == "nan_row":
        assert 0 not in o["row"] and 1 not in o["row"]
    elif case == "one_row":
        assert o["row"].tolist() == [0, 0]


def test_search_k0_and_no_row():
    tb = SC.table()
    t = np.float32([[5.0, np.nan], [1.0, 0.0], [0.1, 0.0]])
    o = OS.search(t, tb, k0=np.float32([0.25, 0.5]))
    assert o["param"][1, 0] == np.float32(0.25) and o["row"][1] == -1 and np.isnan(o["param"][:, 1]).all()
    g = OS.generate_path(t, tb)
    assert g["status"][1] == OM.EMPTY_TRAJ and g["traj_len"][1] == 0
    p0, v = OS.slp_params()
    p0.max_iter = 0
    g = OS.generate_path(t, tb, params=p0)
    assert g["status"][1] == OM.MAX_ITER_REACHED and g["traj_len"][1] == 0


def _double_rounding_decimals(k=64):
    """Decimal strings just above the midpoint of two adjacent floats whose lower one is even: strtod rounds them to
    the midpoint, which the narrowing to float rounds down (ties to even), while strtof rounds them up."""
    rng = np.random.default_rng(5)
    out = []
    while len(out) < k:
        f = np.float32(rng.uniform(-30, 30))
        if f.view(np.uint32) & 1:
            continue
        g = np.nextafter(f, np.float32(np.inf) if f > 0 else np.float32(-np.inf))
        with localcontext() as ctx:
            ctx.prec = 200   # the midpoint and the nudge exactly
            mid = (Decimal(float(f)) + Decimal(float(g))) / 2
            out.append(str(mid + (Decimal(1).scaleb(-40) if f > 0 else -Decimal(1).scaleb(-40))))
    return out


def test_load_table_is_the_reference_reading(tmp_path):
    libc = C.CDLL(None)
    libc.strtof.restype, libc.strtof.argtypes = C.c_float, [C.c_char_p, C.c_void_p]
    libc.strtod.restype, libc.strtod.argtypes = C.c_double, [C.c_char_p, C.c_void_p]
    dec = _double_rounding_decimals()
    assert all(np.float32(libc.strtod(s.encode(), None)) != np.float32(libc.strtof(s.encode(), None)) for s in dec)
    p = tmp_path / "t.csv"
    rows = [",".join(dec[6 * r:6 * r + 6]) for r in range(len(dec) // 6)]
    p.write_text("x,y,yaw,s,km,kf\n" + "\n".join(rows) + "\n")
    got = slp_load_table(p)
    want = np.float32([[libc.strtod(s.encode(), None) for s in dec[6 * r:6 * r + 6]] for r in range(len(rows))])
    assert same(got, want)
    assert same(slp_load_table(SC.TABLE_CSV)[:, :], np.float32([[float(v) for v in ln.split(",")]
                                                                for ln in open(SC.TABLE_CSV).read().split()[1:]]))
    bad = tmp_path / "bad.csv"
    bad.write_text("h\n1,2,3\n")
    with pytest.raises(ValueError):
        slp_load_table(bad)
    L = SC.ref_lib()
    if L is not None:
        assert same(slp_load_table(p), SC.ref_read_csv(L, p))
        assert same(slp_load_table(SC.TABLE_CSV), SC.ref_read_csv(L, SC.TABLE_CSV))


def test_oracle_reproduces_the_golden_fixture():
    d = np.load(GOLDEN)
    tb = d["table"]
    assert same(tb, SC.table())
    for kind, name in NAMES:
        s, qp = SC.demo(kind)
        o = OS.sample(s, qp)
        n = int(o["n_states"][0])
        g = OS.generate_path(o["target"][:, :n], tb, max_pts=256)
        assert same(g["traj"], d[f"demo_{name}_traj"]) and np.array_equal(g["traj_len"], d[f"demo_{name}_len"])
        fields, _ = synth.slp_inputs(1, kind)
        o = OS.sample(SC.sampler_of(fields), d[f"seeded_{name}_qp"])
        ok = np.repeat(o["status"] == OS.OK, OS.states_per_query(SC.sampler_of(fields)))
        assert same(o["target"][:, ok], d[f"seeded_{name}_target"][:, ok])
        t = np.ascontiguousarray(o["target"][:, d[f"seeded_{name}_cols"]])
        assert same(OS.search(t, tb)["param"], d[f"seeded_{name}_param"])
        g = OS.generate_path(t, tb, max_pts=256)
        assert same(g["traj"], d[f"seeded_{name}_traj"]) and np.array_equal(g["traj_len"], d[f"seeded_{name}_len"])


def test_defaults_and_layout(tmp_path):
    p, v = slp_default_params()
    q, w = OS.slp_params()
    assert (p.base_l, p.ds, p.max_iter, p.cost_th, list(p.h_step), v) == \
        (q.base_l, q.ds, q.max_iter, q.cost_th, list(q.h_step), w)
    assert np.float32(p.h_step[0]) == np.float32(0.5) and np.float32(p.h_step[1]) == np.float32(0.02)
    got = run_layout_probe(
        tmp_path, '#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){printf("%zu %zu %zu %zu '
        '%zu %d %d %d %d %d %d %d %d %d\\n",sizeof(crb_slp_sampler),offsetof(crb_slp_sampler,nxy),'
        'offsetof(crb_slp_sampler,nh),offsetof(crb_slp_sampler,ns),offsetof(crb_slp_sampler,d),'
        'CRB_SLP_UNIFORM,CRB_SLP_BIASED,CRB_SLP_LANE,CRB_SLP_MAX_NXY,CRB_SLP_MAX_NH,CRB_SLP_MAX_NS,'
        'CRB_SLP_MAX_STATES,CRB_SLP_OK,CRB_SLP_OUT_OF_RANGE);return 0;}\n')
    S = _lib.SlpSampler
    assert got[:5] == [C.sizeof(S), S.nxy.offset, S.nh.offset, S.ns.offset, S.d.offset]
    assert got[5:] == [_lib.CRB_SLP_UNIFORM, _lib.CRB_SLP_BIASED, _lib.CRB_SLP_LANE, _lib.CRB_SLP_MAX_NXY,
                       _lib.CRB_SLP_MAX_NH, _lib.CRB_SLP_MAX_NS, _lib.CRB_SLP_MAX_STATES, _lib.CRB_SLP_OK,
                       _lib.CRB_SLP_OUT_OF_RANGE]
    assert got[5:] == [OS.UNIFORM, OS.BIASED, OS.LANE, OS.MAX_NXY, OS.MAX_NH, OS.MAX_NS, OS.MAX_STATES, OS.OK,
                       OS.OUT_OF_RANGE]
    L = _lib.load_library()
    for (kind, nxy, nh, ns), want in [((0, 5, 3, 0), 15), ((1, 30, 2, 100), 58), ((2, 5, 0, 0), 5),
                                      ((1, 1, 4, 0), 0), ((0, 256, 256, 0), 65536), ((0, 257, 256, 0), -1),
                                      ((3, 5, 1, 0), -1), ((0, 0, 1, 0), -1), ((1, 5, 0, 0), -1), ((1, 5, 1, -1), -1),
                                      ((2, 4097, 1, 0), -1)]:
        s = _lib.SlpSampler(kind, nxy, nh, ns, 20)
        assert L.crb_slp_states_per_query(C.byref(s)) == want, (kind, nxy, nh, ns)
        if want >= 0:
            assert OS.states_per_query(OS.sampler(kind, nxy, nh, ns, 20)) == want


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE on a machine without
    a GPU.  The context handle is an opaque non-NULL buffer that these paths never dereference."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)
    good = _lib.SlpSampler(1, 30, 2, 100, 20)
    inv = -1

    def samp(**over):
        a = dict(dict(ctx=ctx, n=1, s=C.byref(good), qp=d, t=d, ns=d), **over)
        return L.crb_slp_sample_states_batched(a["ctx"], a["n"], a["s"], a["qp"], a["t"], a["ns"], d)

    def srch(**over):
        a = dict(dict(ctx=ctx, n=1, t=d, tb=d, rows=24, p=d), **over)
        return L.crb_slp_search_nearest_batched(a["ctx"], a["n"], a["t"], a["tb"], a["rows"], None, a["p"], d)
    for k in ("ctx", "s", "qp", "t", "ns"):
        assert samp(**{k: None}) == inv, k
    for k in ("ctx", "t", "tb", "p"):
        assert srch(**{k: None}) == inv, k
    for bad in [(3, 30, 2, 100, 20), (-1, 30, 2, 100, 20), (1, 0, 2, 100, 20), (1, 4097, 2, 100, 20),
                (1, 30, 0, 100, 20), (1, 30, 1025, 100, 20), (1, 30, 2, -1, 20), (1, 30, 2, (1 << 20) + 1, 20),
                (0, 1024, 1024, 0, 0)]:
        assert samp(s=C.byref(_lib.SlpSampler(*bad))) == inv, bad
    assert samp(n=-1) == inv and srch(n=-1) == inv
    assert srch(rows=0) == inv and srch(rows=-5) == inv and srch(n=0, t=None, tb=None, p=None, rows=0) == inv
    if not torch.cuda.is_available():
        assert samp() == _lib.CRB_ERR_NO_DEVICE and srch() == _lib.CRB_ERR_NO_DEVICE
        assert samp(n=0, qp=None, t=None, ns=None) == _lib.CRB_ERR_NO_DEVICE
        assert srch(n=0, t=None, tb=None, p=None) == _lib.CRB_ERR_NO_DEVICE
        assert b"no CPU fallback" in L.crb_last_error_string()
        for s in ((0, 5, 3, 0, 20), (2, 5, 0, 0, 0), (1, 1, 1, 0, 0)):
            assert samp(s=C.byref(_lib.SlpSampler(*s))) == _lib.CRB_ERR_NO_DEVICE


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "slp_ref_api.cpp")


def test_new_kernels_do_not_spill():
    kernels = [f for k, f in ptxas_kernels("crb_slp.cu").items() if "crb_slp_" in k]
    assert len(kernels) == 2
    for f in kernels:
        assert (f.spill_stores, f.spill_loads) == (0, 0), f


# ---- H100 -----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _gpu_sample(engine, s, qp):
    t, ns, st = engine.slp_sample_states(_lib_sampler(s), _dev(qp))
    return dict(target=t.cpu().numpy(), n_states=ns.cpu().numpy(), status=st.cpu().numpy())


def _same_dict(r, o, keys):
    return all(same(r[k], o[k]) for k in keys)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [k for k, _ in NAMES])
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
def test_gpu_sampler_is_bitwise_the_oracle(engine, kind, n):
    fields, qp = synth.slp_inputs(n, kind, seed=0xB00 + n)
    s = SC.sampler_of(fields)
    assert _same_dict(_gpu_sample(engine, s, qp), OS.sample(s, qp), ("target", "n_states", "status"))


@pytest.mark.gpu
def test_gpu_sampler_corner_cases_are_bitwise_the_oracle(engine):
    for name, s, qp in SC.sampler_sets():
        assert _same_dict(_gpu_sample(engine, s, qp), OS.sample(s, qp), ("target", "n_states", "status")), name


def _gpu_search(engine, t, tb, k0=None):
    p, r = engine.slp_search_nearest(_dev(t), _dev(tb), None if k0 is None else _dev(k0))
    return dict(param=p.cpu().numpy(), row=r.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 24, 5000])
def test_gpu_search_is_bitwise_the_oracle(engine, rows):
    tb = SC.table() if rows == 24 else synth.slp_table(rows, seed=rows)
    fields, qp = synth.slp_inputs(4097, OS.BIASED, seed=9)
    t = OS.sample(SC.sampler_of(fields), qp)["target"]          # includes NaN slots: row -1
    k0 = synth.uniform(3, 160, np.arange(t.shape[1], dtype=np.uint64), -0.1, 0.1).astype(np.float32)
    for kk in (None, k0):
        o = OS.search(t, tb, kk)
        assert _same_dict(_gpu_search(engine, t, tb, kk), o, ("param", "row"))
    assert (o["row"] == -1).any() and (o["row"] >= 0).any()
    for name, t, tb in SC.search_sets():
        assert _same_dict(_gpu_search(engine, t, tb), OS.search(t, tb), ("param", "row")), name


def _gpu_generate(engine, t, tb, max_pts, k0=None, params=None):
    r = engine.slp_generate_path(_dev(t), _dev(tb), None if k0 is None else _dev(k0), params=params, max_pts=max_pts)
    return {k: (None if v is None else v.cpu().numpy()) for k, v in r.items()}


@pytest.mark.gpu
def test_gpu_generate_path_is_bitwise_the_oracle(engine):
    tb = SC.table()
    for kind, name in NAMES:
        fields, qp = synth.slp_inputs(700, kind, seed=0xC0 + kind)
        t = OS.sample(SC.sampler_of(fields), qp)["target"]
        k0 = synth.uniform(4, 161, np.arange(t.shape[1], dtype=np.uint64), -0.05, 0.05).astype(np.float32)
        for kk in (None, k0):
            o = OS.generate_path(t, tb, kk, max_pts=96)
            r = _gpu_generate(engine, t, tb, 96, kk)
            assert _same_dict(r, o, ("param", "traj", "traj_len", "cost", "status", "iters", "row")), name
        assert (o["status"] == OM.CONVERGED).any() and (o["row"] == -1).any() and (o["traj_len"] > 96).any()


@pytest.mark.gpu
def test_gpu_reproduces_the_golden_fixture(engine):
    d = np.load(GOLDEN)
    tb = d["table"]
    for kind, name in NAMES:
        s, qp = SC.demo(kind)
        g = _gpu_sample(engine, s, qp)
        n = int(g["n_states"][0])
        r = _gpu_generate(engine, g["target"][:, :n], tb, 256)
        assert same(r["traj"], d[f"demo_{name}_traj"]) and np.array_equal(r["traj_len"], d[f"demo_{name}_len"])
        fields, _ = synth.slp_inputs(1, kind)
        s = SC.sampler_of(fields)
        g = _gpu_sample(engine, s, d[f"seeded_{name}_qp"])
        ok = np.repeat(g["status"] == OS.OK, OS.states_per_query(s))
        assert same(g["target"][:, ok], d[f"seeded_{name}_target"][:, ok])
        t = np.ascontiguousarray(g["target"][:, d[f"seeded_{name}_cols"]])
        assert same(_gpu_search(engine, t, tb)["param"], d[f"seeded_{name}_param"])
        r = _gpu_generate(engine, t, tb, 256)
        assert same(r["traj"], d[f"seeded_{name}_traj"]) and np.array_equal(r["traj_len"], d[f"seeded_{name}_len"])


@pytest.mark.gpu
def test_gpu_shard_invariance(engine):
    fields, qp = synth.slp_inputs(3000, OS.BIASED, seed=41)
    s = SC.sampler_of(fields)
    S = OS.states_per_query(s)
    full = _gpu_sample(engine, s, qp)
    i0, i1 = 1001, 2417
    _, shard = synth.slp_inputs(i1 - i0, OS.BIASED, seed=41, i0=i0)
    assert same(shard, np.ascontiguousarray(qp[:, i0:i1]))
    part = _gpu_sample(engine, s, shard)
    assert same(part["target"], np.ascontiguousarray(full["target"][:, i0 * S:i1 * S]))
    assert same(part["n_states"], full["n_states"][i0:i1]) and same(part["status"], full["status"][i0:i1])
    tb = SC.table()
    t = full["target"]
    a = _gpu_generate(engine, t, tb, 32)
    b = _gpu_generate(engine, np.ascontiguousarray(t[:, 5000:40000]), tb, 32)
    for k in ("param", "traj"):
        assert same(b[k], np.ascontiguousarray(a[k][:, 5000:40000])), k
    for k in ("traj_len", "cost", "status", "iters", "row"):
        assert same(b[k], a[k][5000:40000]), k


@pytest.mark.gpu
def test_gpu_n_zero_is_a_no_op(engine):
    import torch
    e = torch.empty((5, 0), dtype=torch.float32, device="cuda:0")
    t, ns, st = engine.slp_sample_states(_lib_sampler(OS.sampler(OS.BIASED, 30, 2, 100, 20)), e)
    assert t.shape == (3, 0) and ns.shape == (0,)
    p, r = engine.slp_search_nearest(e[:3], _dev(SC.table()))
    g = engine.slp_generate_path(e[:3], _dev(SC.table()))
    torch.cuda.synchronize()
    assert p.shape == (4, 0) and g["status"].shape == (0,)


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_oracle(tmp_path):
    exe = build_ref_program(tmp_path, "slp_ref_api.cpp")
    tb = SC.table()
    tb.tofile(tmp_path / "table.bin")
    subprocess.check_call([exe, str(tmp_path / "table.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    p = 0
    for kind, name in NAMES:
        s, qp = SC.demo(kind)
        o = OS.sample(s, qp)
        n = int(o["n_states"][0])
        g = OS.generate_path(o["target"][:, :n], tb, max_pts=512)
        assert int(out[p]) == n
        p += 1
        for i in range(n):
            k = int(out[p]); p += 1
            assert k == g["traj_len"][i]
            assert same(out[p:p + 3 * k], g["traj"][:3 * k, i]); p += 3 * k
    s, qp = SC.demo(OS.UNIFORM)
    want = OS.search(OS.sample(s, qp)["target"][:, :1], tb)["param"][:, 0]
    assert same(out[p:p + 4], want) and p + 4 == out.size
