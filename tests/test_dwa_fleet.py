"""Dynamic window approach for a mixed fleet: crb_dwa_control_fleet_batched (a Config record per robot from a device
table) and crb_dwa_motion_fleet_batched (a dt per robot).

Each robot's outputs must be bitwise those of crb_dwa_control_many_batched run with its own record, and so those of the
checker (oracle/dwa.py) composed per (config, list); traj keeps the first min(n_pts, max_pts) points and leaves the rest
untouched.  The device decides a record with the host's own function, so a robot's status is CRB_DWA_OK exactly when
crb_dwa_rollout_points accepts its record.
CPU: argument validation without a device, the record layout, the compiler report of the new kernels, the C++ programs
and the synthetic fleet.  H100 (-m gpu): the equivalence at n = 1, 31, 4097 and 2^16 + 3 over every tests/dwa_cases.py
configuration; the device record check against the host's at and past its limits; bad config and list references;
max_pts below, at and above a robot's point count, and traj offsets past 2^31; NULL outputs, n = 0, graph capture and a
one-record table; motion with a dt per robot; a 100-tick closed loop; the C++ program against the checker."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import dwa_cases as D
from cpprobotics_b200 import _lib, dwa_config_table, synth
from oracle import dwa as OD
from toolchain import build_ref_program, ptxas_kernels, run_layout_probe

INV = -1
FIELDS = [k for k, _ in _lib.DwaParams._fields_]
SENT = np.float32(7.0)            # fill of traj rows a launch must leave untouched


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
    return _lib.DwaParams(*[float(getattr(p, k)) for k in FIELDS])


def rollout_points(p):
    """crb_dwa_rollout_points: the point count, or None when the record is refused."""
    n = C.c_int(0)
    rc = _lib.load_library().crb_dwa_rollout_points(C.byref(lib_params(p)), C.byref(n))
    return n.value if rc == 0 else None


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is CRB_ERR_INVALID_ARG before any device work; a valid call is CRB_ERR_NO_DEVICE on a
    machine without a GPU."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)

    def ctl(**over):
        a = dict(dict(ctx=ctx, n=5, x=d, u=d, goal=d, ob=d, rows=40, off=d, ns=3, of=d, cfg=d, nc=4, cof=d, mp=32),
                 **over)
        return L.crb_dwa_control_fleet_batched(a["ctx"], a["n"], a["x"], a["u"], a["goal"], a["ob"], a["rows"],
                                               a["off"], a["ns"], a["of"], a["cfg"], a["nc"], a["cof"], a["mp"], None,
                                               None, None, None, None)

    for kw in (dict(ctx=None), dict(n=-1), dict(x=None), dict(u=None), dict(goal=None), dict(ns=0), dict(ns=-1),
               dict(rows=-1), dict(off=None), dict(of=None), dict(ob=None), dict(nc=0), dict(nc=-1), dict(cfg=None),
               dict(cof=None), dict(mp=-1), dict(mp=_lib.CRB_DWA_MAX_STEPS + 2), dict(n=0, nc=0),
               dict(n=0, mp=-1), dict(n=0, ns=0)):
        assert ctl(**kw) == INV, kw

    def mot(**over):
        a = dict(dict(ctx=ctx, n=5, x=d, u=d, dt=d), **over)
        return L.crb_dwa_motion_fleet_batched(a["ctx"], a["n"], a["x"], a["u"], a["dt"])

    for kw in (dict(ctx=None), dict(n=-1), dict(x=None), dict(u=None), dict(dt=None)):
        assert mot(**kw) == INV, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert ctl() == nd and ctl(ob=None, rows=0) == nd and ctl(mp=0) == nd
        assert ctl(mp=_lib.CRB_DWA_MAX_STEPS + 1) == nd
        assert ctl(n=0, x=None, u=None, goal=None, ob=None, off=None, of=None, cfg=None, cof=None) == nd
        assert mot() == nd and mot(n=0, x=None, u=None, dt=None) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def test_config_record_layout(tmp_path):
    """A table row is one crb_dwa_params: 48 bytes, the twelve floats at 4-byte steps in Config's order."""
    fields = ", ".join(f"(int)offsetof(crb_dwa_params, {k})" for k in FIELDS)
    fmt = " ".join(["%d"] * 13)
    got = run_layout_probe(tmp_path, '#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){'
                           f'printf("{fmt}\\n", (int)sizeof(crb_dwa_params), {fields}); return 0;}}\n')
    assert got == [48] + [4 * k for k in range(12)]
    assert C.sizeof(_lib.DwaParams) == 48
    ps = synth.dwa_fleet_configs(9, seed=1)
    t = dwa_config_table(ps)
    assert t.dtype == np.float32 and t.shape == (9, 12) and t.flags["C_CONTIGUOUS"]
    assert t.tobytes() == b"".join(bytes(p) for p in ps)
    with pytest.raises(ValueError):
        dwa_config_table([])


def test_new_kernels_do_not_spill():
    ks = ptxas_kernels("crb_dwa_fleet.cu")
    names = sorted(k for k in ks if "crb_dwa_" in k)
    assert len(names) == 2 and any("control_fleet" in k for k in names) and any("motion_fleet" in k for k in names)
    for name in names:
        f = ks[name]
        assert (f.stack, f.spill_stores, f.spill_loads) == (0, 0, 0) and f.registers <= 64, f


def test_reference_style_programs_compile(tmp_path):
    """The std::vector<Config> overload and the dt-per-robot motion, and programs that only use the single-Config
    overloads."""
    for cpp in ("dwa_fleet_ref_api.cpp", "dwa_ref_api.cpp", "plan_many_ref_api.cpp"):
        build_ref_program(tmp_path, cpp)


def test_synthetic_fleet_is_deterministic_and_accepted():
    a, b = synth.dwa_fleet_configs(40, seed=3), synth.dwa_fleet_configs(40, seed=3)
    assert [bytes(p) for p in a] == [bytes(p) for p in b]
    assert [bytes(p) for p in a] != [bytes(p) for p in synth.dwa_fleet_configs(40, seed=4)]
    pts = [rollout_points(p) for p in a]
    assert all(k is not None for k in pts)
    assert [k == OD.dwa_rollout_points(p) for k, p in zip(pts, a)] == [True] * 40
    assert len({bytes(p) for p in a}) == 40 and min(pts) < 20 and max(pts) > 60
    t = dwa_config_table(a)
    assert np.ptp(t[:, FIELDS.index("robot_radius")]) > 1.0 and np.ptp(t[:, FIELDS.index("v_reso")]) > 0.01
    of = np.random.default_rng(0).integers(0, 40, 3000).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(a, of, seed=9)
    x2, u2, g2 = synth.dwa_fleet_inputs(a, of, seed=9)
    assert same(x, x2) and same(u, u2) and same(g, g2)
    lo, hi, w = t[of, 1], t[of, 0], t[of, 2]
    assert ((x[3] >= lo) & (x[3] <= hi)).all() and (np.abs(x[4]) <= w).all()
    assert (x[3] == hi).mean() > 0.08 and (x[4] == -w).mean() > 0.08
    assert same(u, x[3:5])


# ---- H100 -----------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    return None if t is None else t.cpu().numpy()


def fleet_lists():
    """Fleet lists (empty, 1-row and 256-row ones among them) and the demo's list."""
    return synth.dwa_fleet_obstacles(40, seed=3) + [synth.DWA_DEMO_OBSTACLES]


def gpu_fleet(engine, lists, ob_of, configs, config_of, x, u, g, max_pts=None, outputs=True, store=None, table=None):
    """One crb_dwa_control_fleet_batched launch; outputs filled with sentinels first."""
    import torch
    n = x.shape[1]
    ob, off = store if store is not None else synth.pack_obstacles(lists, 2)
    tab = table if table is not None else dwa_config_table(configs)
    if max_pts is None:
        max_pts = max([rollout_points(p) or 0 for p in configs] + [0])
    ud = _dev(u)
    dev = "cuda:0"
    cost = torch.full((n,), 3.0, device=dev) if outputs else None
    best = torch.full((n,), 7, dtype=torch.int32, device=dev) if outputs else None
    traj = torch.full((5 * max_pts, n), float(SENT), device=dev) if outputs else None
    tl = torch.full((n,), 7, dtype=torch.int32, device=dev) if outputs else None
    st = engine.dwa_control_fleet(_dev(x), ud, _dev(g), (_dev(ob), _dev(off)), _dev(ob_of), _dev(tab),
                                  _dev(config_of), max_pts=max_pts, cost=cost, best=best, traj=traj, traj_len=tl)
    torch.cuda.synchronize()
    return dict(u=_host(ud), cost=_host(cost), best=_host(best), traj=_host(traj), traj_len=_host(tl),
                status=_host(st), max_pts=max_pts)


def many_per_config(engine, lists, ob_of, configs, config_of, x, u, g):
    """crb_dwa_control_many_batched once per config on its own robots, scattered back: dict(u, cost, best, traj (a
    list of each robot's [5 n_pts] column))."""
    import torch
    n = x.shape[1]
    ob, off = synth.pack_obstacles(lists, 2)
    obd, offd = _dev(ob), _dev(off)
    out = dict(u=np.zeros((2, n), np.float32), cost=np.zeros(n, np.float32), best=np.zeros(n, np.int32),
               traj=[None] * n)
    for c in np.unique(config_of):
        sel = np.nonzero(config_of == c)[0]
        p = lib_params(configs[c])
        m = sel.size
        ud = _dev(u[:, sel])
        cost = torch.empty(m, device="cuda:0")
        best = torch.empty(m, dtype=torch.int32, device="cuda:0")
        traj = torch.empty((5 * rollout_points(p), m), device="cuda:0")
        engine.dwa_control_many(_dev(x[:, sel]), ud, _dev(g[:, sel]), (obd, offd), _dev(ob_of[sel]), p, cost=cost,
                                best=best, traj=traj)
        torch.cuda.synchronize()
        out["u"][:, sel], out["cost"][sel], out["best"][sel] = _host(ud), _host(cost), _host(best)
        tr = _host(traj)
        for j, i in enumerate(sel):
            out["traj"][i] = tr[:, j]
    return out


def checker_per_pair(lists, ob_of, configs, config_of, x, u, g):
    """The checker composed per (config, list), in the layout of many_per_config."""
    n = x.shape[1]
    out = dict(u=np.zeros((2, n), np.float32), cost=np.zeros(n, np.float32), best=np.zeros(n, np.int32),
               traj=[None] * n)
    keys = config_of.astype(np.int64) * (len(lists) + 1) + ob_of
    for key in np.unique(keys):
        sel = np.nonzero(keys == key)[0]
        c, s = int(config_of[sel[0]]), int(ob_of[sel[0]])
        o = OD.dwa_control(*(np.ascontiguousarray(a[:, sel]) for a in (x, u, g)), lists[s], configs[c])
        out["u"][:, sel], out["cost"][sel], out["best"][sel] = o["u"], o["cost"], o["best"]
        for j, i in enumerate(sel):
            out["traj"][i] = o["traj"][:, j]
    return out


def assert_fleet_is(got, want, config_of, configs, cols=None):
    """Robots cols of a fleet launch are want's (u, cost, best bitwise; the first min(n_pts, max_pts) points of traj;
    rows past them untouched; traj_len n_pts)."""
    cols = np.arange(got["u"].shape[1]) if cols is None else cols
    assert same(got["u"][:, cols], want["u"][:, cols]) and same(got["cost"][cols], want["cost"][cols])
    assert same(got["best"][cols], want["best"][cols])
    pts = np.array([rollout_points(configs[c]) for c in range(len(configs))])
    assert same(got["traj_len"][cols], pts[config_of[cols]].astype(np.int32))
    mp = got["max_pts"]
    for i in cols:
        k = min(int(pts[config_of[i]]), mp)
        assert same(got["traj"][:5 * k, i], want["traj"][i][:5 * k]), i
        assert (got["traj"][5 * k:, i] == SENT).all(), i


def mixed_fleet(n, configs_names, n_lists, seed):
    """n robots shuffled over the named dwa_cases configurations and n_lists lists; each robot's state from its
    configuration's config_batch (quirk robots and start yaws included)."""
    rng = np.random.default_rng(seed)
    config_of = rng.integers(0, len(configs_names), n).astype(np.int32)
    ob_of = rng.integers(0, n_lists, n).astype(np.int32)
    x, u, g = (np.zeros((k, n), np.float32) for k in (5, 2, 2))
    for c, name in enumerate(configs_names):
        sel = np.nonzero(config_of == c)[0]
        if sel.size:
            x[:, sel], u[:, sel], g[:, sel] = D.config_batch(name, sel.size, np.zeros((0, 2)), seed=seed + c)
    return config_of, ob_of, x, u, g


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 4097, 2 ** 16 + 3])
def test_gpu_mixed_fleet_is_many_per_config_and_the_checker(engine, n):
    names = [k for k in D.CONFIGS if n <= 31 or not D.heavy(k)]
    configs = [D.config(k) for k in names]
    lists = fleet_lists()
    config_of, ob_of, x, u, g = mixed_fleet(n, names, len(lists), seed=0xF1 + n)
    got = gpu_fleet(engine, lists, ob_of, configs, config_of, x, u, g)
    assert (got["status"] == _lib.CRB_DWA_OK).all()
    assert_fleet_is(got, many_per_config(engine, lists, ob_of, configs, config_of, x, u, g), config_of, configs)
    assert_fleet_is(got, checker_per_pair(lists, ob_of, configs, config_of, x, u, g), config_of, configs)
    if n >= 4097:
        assert len(np.unique(config_of)) == len(names) and (got["best"] < 0).any() and (got["best"] >= 0).any()


def record_sweep():
    """Records around the limits: the near-cap sweep of test_dwa_params.test_sample_count_rule_is_sound (every other
    magnitude), BEYOND_CAP, a NaN or inf in each field, and v_reso, yawrate_reso or dt at 0 or below."""
    VCAP, WCAP = _lib.CRB_DWA_MAX_SPEED_SAMPLES, _lib.CRB_DWA_MAX_YAWRATE_SAMPLES
    f32 = np.float32
    recs = []
    for m in np.float32(np.logspace(-3, 7, 21)):
        ulp = float(np.spacing(m))
        for r in (0.5, 0.51, 0.6, 0.75, 1.0, 1.5, 2.0, 3.0, 7.0, 33.0, 1e3, 1e4):
            reso = f32(r * ulp)
            for dl in (-1.0, -0.5, 0.0, 0.5, 1.0):
                for axis, cap in (("v", VCAP), ("w", WCAP)):
                    width = float(f32((cap - 2 + dl) * float(reso)))
                    if axis == "v":
                        recs += [dict(max_speed=m, min_speed=float(f32(m - width)), max_accel=float(m) * 4.0, dt=1.0,
                                      v_reso=float(reso), max_dyawrate=0.0),
                                 dict(max_speed=m, min_speed=-m, max_accel=width / 2.0, dt=1.0, v_reso=float(reso),
                                      max_dyawrate=0.0)]
                    else:
                        recs += [dict(max_yawrate=m, max_dyawrate=width / 2.0, dt=1.0, yawrate_reso=float(reso),
                                      max_accel=0.0),
                                 dict(max_yawrate=float(f32(width / 2.0)), max_dyawrate=float(m) * 4.0, dt=1.0,
                                      yawrate_reso=float(reso), max_accel=0.0)]
    ps = [OD.dwa_params(**kw) for kw in recs]
    ps += [OD.dwa_params(**kw) for kw in (
        dict(max_speed=1e5, min_speed=99999.4, max_accel=10.0, dt=0.1, v_reso=0.01, predict_time=0.3),
        dict(max_yawrate=1e4, max_dyawrate=10.0, dt=0.02525, yawrate_reso=0.001),
        dict(max_speed=1e6, min_speed=1e6 - 0.6, max_accel=3.0, v_reso=0.01),
        dict(dt=0.0625, predict_time=62.4375), dict(dt=0.0625, predict_time=62.5))]
    for k in FIELDS:
        for v in (np.nan, np.inf, -np.inf):
            ps.append(OD.dwa_params(**{k: float(v)}))
    for k in ("v_reso", "yawrate_reso", "dt"):
        for v in (0.0, -0.0, -1e-45, -0.01):
            ps.append(OD.dwa_params(**{k: v}))
    ps += [D.config(k) for k in D.CONFIGS]
    return ps


@pytest.mark.gpu
def test_gpu_device_record_check_is_the_host_check(engine):
    configs = record_sweep()
    pts = [rollout_points(p) for p in configs]
    n = len(configs)
    assert 500 < sum(k is not None for k in pts) < n - 100
    config_of = np.arange(n, dtype=np.int32)
    x = np.zeros((5, n), np.float32)
    t = dwa_config_table(configs)
    x[3] = np.clip(np.float32(0.0), t[:, 1], t[:, 0])
    x[3] = np.where(np.isfinite(x[3]), x[3], 0.0)
    u = np.ascontiguousarray(x[3:5])
    g = np.full((2, n), 5.0, np.float32)
    lists = [np.zeros((0, 2), np.float32)]
    got = gpu_fleet(engine, lists, np.zeros(n, np.int32), configs, config_of, x, u, g, max_pts=2)
    ok = np.array([k is not None for k in pts])
    assert np.array_equal(got["status"] == _lib.CRB_DWA_OK, ok)
    assert (got["status"][~ok] == _lib.CRB_DWA_BAD_CONFIG).all()
    assert np.array_equal(got["traj_len"], np.array([k if k is not None else 0 for k in pts], np.int32))
    assert np.isnan(got["u"][:, ~ok]).all() and np.isnan(got["cost"][~ok]).all() and (got["best"][~ok] == -1).all()
    assert (got["traj"][:, ~ok] == SENT).all()


@pytest.mark.gpu
def test_gpu_bad_config_and_list_references(engine):
    configs = synth.dwa_fleet_configs(8, seed=2) + [OD.dwa_params(v_reso=0.0)]   # the last record is refused
    nc = len(configs)
    lists = fleet_lists()
    nl = len(lists)
    n = 4097
    rng = np.random.default_rng(5)
    config_of = rng.integers(0, nc - 1, n).astype(np.int32)
    ob_of = rng.integers(0, nl, n).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=6)
    kind = rng.integers(0, 8, n)   # 0-3 good; 4 bad config; 5 refused record; 6 bad list; 7 both bad
    cof, oof = config_of.copy(), ob_of.copy()
    bad_c = (kind == 4) | (kind == 7)
    cof[bad_c] = rng.choice(np.int32([-1, nc, 2 ** 31 - 1, -(2 ** 31)]), bad_c.sum())
    cof[kind == 5] = nc - 1
    bad_l = (kind == 6) | (kind == 7)
    oof[bad_l] = rng.choice(np.int32([-1, nl, 2 ** 31 - 1]), bad_l.sum())
    got = gpu_fleet(engine, lists, oof, configs, cof, x, u, g)
    bc, bl = bad_c | (kind == 5), kind == 6
    good = ~(bc | bl)
    assert (got["status"][bc] == _lib.CRB_DWA_BAD_CONFIG).all()
    assert (got["status"][bl] == _lib.CRB_DWA_BAD_OBSTACLES).all() and (got["status"][good] == 0).all()
    for m in (bc, bl):
        assert np.isnan(got["u"][:, m]).all() and np.isnan(got["cost"][m]).all() and (got["best"][m] == -1).all()
    assert (got["traj_len"][bc] == 0).all() and (got["traj"][:, bc] == SENT).all()
    pts = np.array([rollout_points(p) or 0 for p in configs])
    assert np.array_equal(got["traj_len"][bl], pts[cof[bl]])
    for i in np.nonzero(bl)[0]:
        k = min(int(pts[cof[i]]), got["max_pts"])
        assert np.isnan(got["traj"][:5 * k, i]).all() and (got["traj"][5 * k:, i] == SENT).all()
    # every other robot is what it is in a batch without the bad ones
    sub = np.nonzero(good)[0]
    alone = gpu_fleet(engine, lists, ob_of[sub], configs, config_of[sub], *(a[:, sub] for a in (x, u, g)))
    for k in ("u", "traj"):
        assert same(got[k][:, sub], alone[k]), k
    for k in ("cost", "best", "traj_len", "status"):
        assert same(got[k][sub], alone[k]), k


@pytest.mark.gpu
def test_gpu_max_pts_clips_traj(engine):
    configs = synth.dwa_fleet_configs(8, seed=7)     # 32, 16, 27, 32, 21, 13, 82 and 32 points
    pts = [rollout_points(p) for p in configs]
    lists = fleet_lists()
    n = 3001
    rng = np.random.default_rng(8)
    config_of = rng.integers(0, 8, n).astype(np.int32)
    ob_of = rng.integers(0, len(lists), n).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=9)
    want = many_per_config(engine, lists, ob_of, configs, config_of, x, u, g)
    for mp in (27, 0, 1, max(pts), _lib.CRB_DWA_MAX_STEPS + 1):
        got = gpu_fleet(engine, lists, ob_of, configs, config_of, x, u, g, max_pts=mp)
        assert got["traj"].shape == (5 * mp, n)
        assert_fleet_is(got, want, config_of, configs)
    assert min(pts) < 27 < max(pts) and 27 in pts


@pytest.mark.gpu
def test_gpu_traj_offsets_past_2_31_elements(engine):
    """2^19 + 3 robots, one in four on a 1000-step one-sample record, the rest on the reference Config, with max_pts
    1001: traj is 5005 x (2^19 + 3) floats, and its element offsets pass 2^31 from row 4096."""
    import torch
    if torch.cuda.mem_get_info()[0] < 12 * 2 ** 30:
        pytest.skip("needs 12 GiB of free device memory")
    long = OD.dwa_params(max_accel=0.0, max_dyawrate=0.0, dt=0.0625, predict_time=62.4375)
    configs = [OD.dwa_params(), long]
    n = 2 ** 19 + 3
    config_of = (np.arange(n) % 4 == 1).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=31)
    ob_of = np.zeros(n, np.int32)
    ob, off = synth.pack_obstacles([synth.DWA_DEMO_OBSTACLES], 2)
    dev = torch.device("cuda:0")
    ud = _dev(u)
    tl = torch.empty(n, dtype=torch.int32, device=dev)
    traj = torch.full((5 * 1001, n), float(SENT), device=dev)
    try:
        engine.dwa_control_fleet(_dev(x), ud, _dev(g), (_dev(ob), _dev(off)), _dev(ob_of),
                                 _dev(dwa_config_table(configs)), _dev(config_of), traj=traj, traj_len=tl)
        row0 = (2 ** 31) // n
        rows = np.r_[0, 1, row0 - 2:row0 + 3, 5 * 1001 - 5:5 * 1001]
        c0 = 2 ** 31 - row0 * n
        cols = np.unique(np.r_[0:1000, c0 - 1000:c0 + 1000, n - 1000:n])
        got = traj.index_select(0, torch.from_numpy(rows).to(dev)).index_select(1, torch.from_numpy(cols).to(dev))
        got = got.cpu().numpy()
        gu, gl = ud.cpu().numpy(), tl.cpu().numpy()
    finally:
        del traj
        torch.cuda.empty_cache()
    assert np.array_equal(gl, np.where(config_of == 1, 1001, 32).astype(np.int32))
    for c in (0, 1):
        sel = cols[config_of[cols] == c]
        o = OD.dwa_control(*(np.ascontiguousarray(a[:, sel]) for a in (x, u, g)), synth.DWA_DEMO_OBSTACLES,
                           configs[c])
        assert same(gu[:, sel], o["u"])
        k = 5 * (1001 if c else 32)
        gsel = got[:, np.isin(cols, sel)]
        r_in = rows < k
        assert same(gsel[r_in], np.ascontiguousarray(o["traj"][rows[r_in]])) and (gsel[~r_in] == SENT).all()


@pytest.mark.gpu
def test_gpu_launch_forms(engine):
    """NULL optional outputs, n = 0, a graph-captured launch, and a one-record table against the many entry point."""
    import torch
    configs = synth.dwa_fleet_configs(8, seed=10)
    lists = synth.dwa_fleet_obstacles(24, seed=8)
    ob, off = synth.pack_obstacles(lists, 2)
    n = 3000
    rng = np.random.default_rng(11)
    config_of = rng.integers(0, 8, n).astype(np.int32)
    ob_of = rng.integers(0, len(lists), n).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=12)
    want = gpu_fleet(engine, lists, ob_of, configs, config_of, x, u, g)
    ud = _dev(u)
    tab, obd, offd = _dev(dwa_config_table(configs)), _dev(ob), _dev(off)
    engine.dwa_control_fleet(_dev(x), ud, _dev(g), (obd, offd), _dev(ob_of), tab, _dev(config_of))
    torch.cuda.synchronize()
    assert same(_host(ud), want["u"])
    assert engine.lib.crb_dwa_control_fleet_batched(engine.ctx, 0, None, None, None, None, 0, None, 1, None, None, 1,
                                                    None, 0, None, None, None, None, None) == 0
    e = torch.empty((5, 0), device="cuda:0")
    i0 = torch.empty(0, dtype=torch.int32, device="cuda:0")
    assert engine.dwa_control_fleet(e, e[:2], e[:2], (obd, offd), i0, tab, i0).shape == (0,)
    engine.dwa_motion_fleet(e, e[:2], e[0])
    # graph capture and replay
    mp = want["max_pts"]
    xd, ud, gd, ofd, cfd = _dev(x), _dev(u), _dev(g), _dev(ob_of), _dev(config_of)
    cost = torch.empty(n, device="cuda:0")
    best = torch.empty(n, dtype=torch.int32, device="cuda:0")
    traj = torch.full((5 * mp, n), float(SENT), device="cuda:0")
    tl = torch.empty(n, dtype=torch.int32, device="cuda:0")
    stt = torch.empty(n, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        eng = type(engine)(0)
        try:
            with torch.cuda.graph(gr, stream=s):
                eng.dwa_control_fleet(xd, ud, gd, (obd, offd), ofd, tab, cfd, max_pts=mp, cost=cost, best=best,
                                      traj=traj, traj_len=tl, status=stt)
            gr.replay()
            torch.cuda.synchronize()
        finally:
            eng.close()
    for k, t in (("u", ud), ("cost", cost), ("best", best), ("traj", traj), ("traj_len", tl), ("status", stt)):
        assert same(_host(t), want[k]), k
    # one record for everyone is crb_dwa_control_many_batched
    for p in (OD.dwa_params(), D.config("distinct")):
        one = np.zeros(n, np.int32)
        xs, us, gs = synth.dwa_fleet_inputs([p], one, seed=13)
        got = gpu_fleet(engine, lists, ob_of, [p], one, xs, us, gs)
        assert_fleet_is(got, many_per_config(engine, lists, ob_of, [p], one, xs, us, gs), one, [p])


@pytest.mark.gpu
def test_gpu_motion_with_a_dt_per_robot(engine):
    """Bitwise crb_dwa_motion_batched per distinct dt; NaN, 0 and negative dt as the checker's motion."""
    import torch
    n = 5003
    rng = np.random.default_rng(14)
    x, u, _ = synth.dwa_inputs(n, seed=15)
    x[2, ::7] = np.float32(130.25)                     # sinf / cosf's large reduction
    good = np.float32([0.1, 0.05, 0.2, 0.0625, 0.08, 1e-3, 3.0])
    odd = np.float32([np.nan, 0.0, -0.0, -0.1, np.inf, -np.inf])
    dt = rng.choice(np.concatenate([good, odd]), n).astype(np.float32)
    xd = _dev(x)
    engine.dwa_motion_fleet(xd, _dev(u), _dev(dt))
    torch.cuda.synchronize()
    got = _host(xd)
    for v in np.concatenate([good, odd]):
        sel = np.nonzero(dt.view(np.uint32) == np.float32(v).view(np.uint32))[0]
        if v in good:
            xs = _dev(x[:, sel])
            engine.dwa_motion(xs, _dev(u[:, sel]), dt=float(v))
            torch.cuda.synchronize()
            assert same(got[:, sel], _host(xs)), v
        assert same(got[:, sel], OD.dwa_motion(x[:, sel], u[:, sel], float(v))), v


@pytest.mark.gpu
def test_gpu_closed_loop_of_a_mixed_fleet(engine):
    """3000 robots over 8 classes and 40 lists, 100 ticks of dwa_control_fleet then dwa_motion_fleet with dt =
    configs.dt[config_of]; a seeded sample of 96 robots is run by the checker alongside, bitwise at every tick."""
    import torch
    configs = synth.dwa_fleet_configs(8, seed=16)
    lists = fleet_lists()
    ob, off = synth.pack_obstacles(lists, 2)
    n = 3000
    rng = np.random.default_rng(17)
    config_of = rng.integers(0, 8, n).astype(np.int32)
    ob_of = rng.integers(0, len(lists), n).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=18)
    tab = _dev(dwa_config_table(configs))
    dtd = tab[:, FIELDS.index("dt")][_dev(config_of).long()].contiguous()
    xd, ud, gd, obd, offd, ofd, cfd = (_dev(a) for a in (x, u, g, ob, off, ob_of, config_of))
    sample = np.sort(rng.choice(n, 96, replace=False))
    xo, uo = x[:, sample].copy(), u[:, sample].copy()
    for tick in range(100):
        st = engine.dwa_control_fleet(xd, ud, gd, (obd, offd), ofd, tab, cfd)
        engine.dwa_motion_fleet(xd, ud, dtd)
        for j, i in enumerate(sample):
            p = configs[config_of[i]]
            o = OD.dwa_control(xo[:, j:j + 1], uo[:, j:j + 1], g[:, i:i + 1], lists[ob_of[i]], p, traj=False)
            uo[:, j:j + 1] = o["u"]
            xo[:, j:j + 1] = OD.dwa_motion(xo[:, j:j + 1], o["u"], p.dt)
        torch.cuda.synchronize()
        assert (_host(st) == 0).all(), tick
        assert same(_host(ud)[:, sample], uo) and same(_host(xd)[:, sample], xo), tick
    assert (np.hypot(xo[0] - x[0, sample], xo[1] - x[1, sample]) > 0.5).mean() > 0.25


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_the_checker(tmp_path):
    exe = build_ref_program(tmp_path, "dwa_fleet_ref_api.cpp")
    configs = synth.dwa_fleet_configs(8, seed=19) + [D.config("distinct")]
    lists = fleet_lists()
    m = 72
    rng = np.random.default_rng(20)
    config_of = rng.integers(0, len(configs), m).astype(np.int32)
    config_of[0] = len(configs) - 1
    ob_of = rng.integers(0, len(lists), m).astype(np.int32)
    x, u, g = synth.dwa_fleet_inputs(configs, config_of, seed=21)
    t = dwa_config_table(configs)
    parts = [np.float32([m])]
    for i in range(m):
        o = lists[ob_of[i]]
        parts += [x[:, i], u[:, i], g[:, i], t[config_of[i]], np.float32([len(o)]), o.reshape(-1)]
    np.concatenate(parts).astype(np.float32).tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    q = 0
    for i in range(m):
        p = configs[config_of[i]]
        o = OD.dwa_control(x[:, i:i + 1], u[:, i:i + 1], g[:, i:i + 1], lists[ob_of[i]], p)
        assert same(out[q:q + 2], o["u"][:, 0]); q += 2
        k = int(out[q]); q += 1
        assert k == (OD.dwa_rollout_points(p) if o["best"][0] >= 0 else 0)
        assert same(out[q:q + 5 * k], o["traj"][:5 * k, 0]); q += 5 * k
        assert same(out[q:q + 5], OD.dwa_motion(x[:, i:i + 1], o["u"], p.dt)[:, 0]); q += 5
    # the single-Config call resolves to the one-Config fleet overload: every robot on robot 0's Config
    for i in range(m):
        o = OD.dwa_control(x[:, i:i + 1], u[:, i:i + 1], g[:, i:i + 1], lists[ob_of[i]], configs[config_of[0]],
                           traj=False)
        assert same(out[q:q + 2], o["u"][:, 0]); q += 2
    assert q == out.size
