"""Problem sets for tests/test_mptg.py, tests/test_mptg_params.py and tests/golden/make_mptg_golden.py: seeded
problems around the demo and the reference's corner cases, each with the parameters it needs.  Every set is
(name, state, target, param, params); limit_sets() adds the statuses each problem is built to end with."""
import functools

import numpy as np

from cpprobotics_b200 import synth
from oracle import mptg as OM

f32 = np.float32
BELOW_120 = np.nextafter(f32(120.0), f32(0.0))   # the largest float below 120


def demo(m=1):
    st = np.tile(np.float32(synth.MPTG_DEMO_STATE)[:, None], (1, m))
    tg = np.tile(np.float32(synth.MPTG_DEMO_TARGET)[:, None], (1, m))
    pa = np.tile(np.float32(synth.MPTG_DEMO_PARAM)[:, None], (1, m))
    return st, tg, pa


def quirk_sets():
    """Corner cases of optimizer_traj, each a set the reference defines (no empty nominal, no endless loop)."""
    sets = []
    st, tg, pa = demo()
    # target = the end of the initial parameter's roll-out: converged at iteration 0
    last = OM.generate(st, pa)["last"]
    sets.append(("converged_at_0", st, last.copy(), pa, OM.mptg_params()))
    # the same target with cost_th 0: dc = 0, dp = -0, both line-search candidates are p: a tie (alpha 1.5)
    sets.append(("ls_tie", st, last.copy(), pa, OM.mptg_params(cost_th=0.0, max_iter=3)))
    # max_iter exhausted: the returned trajectory is the one of the parameter before the last update
    sets.append(("max_iter_2", st, tg, pa, OM.mptg_params(max_iter=2)))
    # max_iter = 0: nothing is rolled out, the returned Traj is empty
    sets.append(("max_iter_0", st, tg, pa, OM.mptg_params(max_iter=0)))
    # h_step[1] so small that steering[1] +- h rolls out the same end: J has a zero column and a non-finite
    # inverse, dp and the parameter become NaN (both candidates roll out nothing: a tie); one iteration keeps the
    # returned Traj defined
    sets.append(("singular_j", st, tg, pa, OM.mptg_params(h_step=(0.2, 1e-30, 0.005), max_iter=1)))
    # a target yaw of NaN: every cost is NaN, so is J; both line-search costs are NaN and alpha stays 1.0
    tn = tg.copy()
    tn[2, 0] = np.float32(np.nan)
    sets.append(("nan_costs", st, tn, pa, OM.mptg_params(max_iter=1)))
    # steering beyond pi/4 from the start: glibc's tanf range reduction (exact below |kp| = 120)
    sw = pa.copy()
    sw[1:, 0] = (0.9, -1.0, 1.3)
    sets.append(("steer_beyond_pio4", st, tg, sw, OM.mptg_params(max_iter=5)))
    # a sweep of distances whose float `i += horizon / n` loops take a step count other than ceil(distance / ds)
    m = 160
    s2, t2, p2 = demo(m)
    p2[0] = np.linspace(0.35, 12.0, m, dtype=np.float32)
    sets.append(("distance_sweep", s2, t2, p2, OM.mptg_params(max_iter=1)))
    return sets


def stopping_sets():
    """Problems the reference does not define (or this library cannot reproduce): checked against the checker's
    statuses only."""
    st, tg, pa = demo(5)
    pa[0, 0] = -1.0          # empty roll-out
    pa[0, 1] = 5000.0        # 50000 steps > CRB_MPTG_MAX_STEPS
    pa[1, 2] = 150.0         # tanf beyond the exact range
    st[2, 3] = 200.0         # sinf / cosf beyond the exact range
    pa[0, 4] = np.float32(np.nan)
    return ("stopping", st, tg, pa, OM.mptg_params()), [OM.EMPTY_TRAJ, OM.STEP_CAP, OM.OUT_OF_RANGE,
                                                        OM.OUT_OF_RANGE, OM.EMPTY_TRAJ]


# ---- away from the demo's start, speed and parameters (tests/test_mptg_params.py) ------------------------------
def relative(n, seed, yaw=(0.0, 0.0), xy=0.0, v=(3.0, 3.0), reach=1.0):
    """n problems, problem i a function of (seed, i) only: a start at (x, y) in [-xy, xy]^2 with yaw in `yaw` and
    speed log-uniform in `v`; a target placed in the start's own frame the way synth.mptg_inputs places it around the
    origin (ahead by [3, 8] * reach, aside by [-3, 3] * reach, turned by [-0.6, 0.6] from the start yaw, unwrapped),
    so that most problems converge; initial parameter (|target - start| + reach, 0, 0, 0)."""
    idx = np.arange(n, dtype=np.uint64)
    st = np.empty((4, n), f32)
    st[0] = synth.uniform(seed, 1, idx, -xy, xy)
    st[1] = synth.uniform(seed, 2, idx, -xy, xy)
    st[2] = synth.uniform(seed, 3, idx, *yaw)
    st[3] = np.exp(synth.uniform(seed, 4, idx, np.log(v[0]), np.log(v[1])))
    lx = synth.uniform(seed, 5, idx, 3.0, 8.0) * reach
    ly = synth.uniform(seed, 6, idx, -3.0, 3.0) * reach
    c, s = np.cos(st[2].astype(np.float64)), np.sin(st[2].astype(np.float64))
    tg = np.empty((3, n), f32)
    tg[0] = st[0] + c * lx - s * ly
    tg[1] = st[1] + s * lx + c * ly
    tg[2] = st[2] + f32(synth.uniform(seed, 7, idx, -0.6, 0.6))
    pa = np.zeros((4, n), f32)
    pa[0] = np.hypot(lx, ly) + reach
    return st, tg, pa


def _cols(*sets):
    return tuple(np.ascontiguousarray(np.concatenate(a, axis=1)) for a in zip(*sets))


def _target_yaws():
    """Target yaws at 2 pi k +- 1 ulp, +-4 pi, 1e6 and 1e30 (both signs), for the demo's start and target x, y."""
    ys = []
    for k in (1, 2, 3, 7, 100):
        for sg in (1.0, -1.0):
            c = f32(sg * 2.0 * np.pi * k)
            ys += [np.nextafter(c, f32(-np.inf)), c, np.nextafter(c, f32(np.inf))]
    ys += [f32(4.0 * np.pi), f32(-4.0 * np.pi), f32(1e6), f32(-1e6), f32(1e30), f32(-1e30)]
    st, tg, pa = demo(len(ys))
    tg[2] = np.float32(ys)
    return st, tg, pa


@functools.lru_cache(maxsize=None)
def _param_sets():
    P = OM.mptg_params
    sets = []
    # start yaws across (-120, 120): beyond 3 pi the first step's YAW_P2P and calc_diff take the general fmod
    st, tg, pa = relative(94, 0x51, yaw=(-119.5, 119.5))
    s2, t2, p2 = relative(2, 0x52)
    s2[2] = (BELOW_120, -BELOW_120)
    t2[2] = s2[2] + f32(0.25)
    sets.append(("start_yaw", *_cols((st, tg, pa), (s2, t2, p2)), P()))
    sets.append(("far_start", *relative(64, 0x53, yaw=(-3.1, 3.1), xy=1e4), P()))
    sets.append(("speed", *relative(64, 0x54, yaw=(-1.0, 1.0), v=(0.1, 20.0)), P()))
    sets.append(("base_l_0.3", *relative(64, 0x55, yaw=(-2.0, 2.0), v=(1.0, 6.0)), P(base_l=0.3, ds=0.05)))
    sets.append(("base_l_2.7", *relative(64, 0x56, v=(0.5, 10.0), reach=2.0),
                 P(base_l=2.7, ds=0.5, h_step=(0.5, 0.02, 0.02))))
    sets.append(("base_l_-1", *relative(64, 0x57, yaw=(-3.0, 3.0)), P(base_l=-1.0)))
    # one step turns the yaw by v / base_l * tan(kp) * dt = 100 tan(kp): YAW_P2P's general fmod on every step
    sets.append(("base_l_1e-3", *relative(48, 0x58), P(base_l=1e-3, max_iter=10)))
    # v / base_l overflows to +inf for v above 3.41: the yaw becomes NaN (tan(kp) = 0 then) or +-inf after a step
    sets.append(("base_l_overflow", *relative(32, 0x59, v=(0.1, 20.0)), P(base_l=1e-38, max_iter=3)))
    sets.append(("ds_0.01", *relative(48, 0x5A, yaw=(-1.0, 1.0), reach=0.5), P(ds=0.01)))
    sets.append(("ds_1", *relative(48, 0x5B, yaw=(-1.0, 1.0), reach=4.0), P(ds=1.0, h_step=(1.0, 0.005, 0.005))))
    # ds beyond every distance: one step of v * dt = ds whatever the distance
    sets.append(("ds_beyond_distance", *relative(32, 0x5C), P(ds=50.0, max_iter=1)))
    # the six Jacobian roll-outs of one iteration differ by up to 60 steps (distance +- 3 at ds 0.1)
    sets.append(("h_step_large", *relative(64, 0x5D, yaw=(-1.0, 1.0), reach=2.0),
                 P(h_step=(3.0, 0.4, 0.7))))
    sets.append(("cost_th_negative", *relative(24, 0x5E), P(cost_th=-1.0, max_iter=30)))
    sets.append(("cost_th_0", *relative(24, 0x5F), P(cost_th=0.0, max_iter=30)))
    sets.append(("cost_th_large", *relative(32, 0x60, yaw=(-6.0, 6.0)), P(cost_th=1e30)))
    # max_iter = CRB_MPTG_MAX_ITER: targets 6 aside and barely ahead (some iterate to the limit, some leave the tanf
    # range or empty the roll-out) and problems that never meet a negative cost_th (every iteration runs)
    st, tg, pa = relative(10, 0x61)
    tg[0] *= f32(0.2)
    tg[1] = st[1] + f32(6.0)
    sets.append(("diverge_1000", st, tg, pa, P(max_iter=OM.MAX_ITER)))
    sets.append(("fixed_point_1000", *relative(8, 0x62), P(max_iter=OM.MAX_ITER, cost_th=-1.0)))
    sets.append(("target_yaw", *_target_yaws(), P(max_iter=3)))
    return sets


def param_sets():
    """Seeded problems away from the demo's start (yaw across (-120, 120), far from the origin), speed (0.1 to 20)
    and parameters (base_l, ds, h_step, cost_th, max_iter up to CRB_MPTG_MAX_ITER), and target yaws far from any
    reachable one.  Every set is (name, state, target, param, params)."""
    return list(_param_sets())


# ---- at the limits (built from the checker, not from constants) ------------------------------------------------
def flip(pred, lo, hi):
    """Adjacent positive floats (a, b) in [lo, hi] with pred(a) false and pred(b) true, by bisection on the bit
    pattern (pred(lo) must be false, pred(hi) true)."""
    ia, ib = int(f32(lo).view(np.int32)), int(f32(hi).view(np.int32))
    assert 0 < ia < ib and not pred(f32(lo)) and pred(f32(hi)), (lo, hi)
    while ib - ia > 1:
        m = (ia + ib) // 2
        if pred(np.int32(m).view(f32)):
            ib = m
        else:
            ia = m
    return np.int32(ia).view(f32), np.int32(ib).view(f32)


def _one(st, q):
    return (np.float32(st).reshape(4, 1), np.float32(q).reshape(4, 1))


def gen_status(st, q, prm):
    s, p = _one(st, q)
    return int(OM.generate(s, p, prm)["status"][0])


def opt_status(st, tg, q, prm):
    s, p = _one(st, q)
    return int(OM.optimize(s, np.float32(tg).reshape(3, 1), p, prm)["status"][0])


DEMO_ST = (0.0, 0.0, 0.0, 3.0)


def _cap_distances(prm):
    """(last distance of 16384 steps, first distance of 16385) at v = 3 for the nominal roll-out."""
    return flip(lambda d: gen_status(DEMO_ST, (d, 0, 0, 0), prm) == OM.STEP_CAP, 1630.0, 1650.0)


def jacobian_cap_distances(prm, tg):
    """Distances whose nominal roll-out completes while distance + h_step[0] crosses the step cap, as the pair where
    one Newton iteration towards tg starts to stop with CRB_MPTG_STEP_CAP."""
    return flip(lambda d: opt_status(DEMO_ST, tg, (d, 0, 0, 0), prm) == OM.STEP_CAP, 1630.0, 1638.2)


@functools.lru_cache(maxsize=None)
def _limit_sets():
    P = OM.mptg_params
    C, MI, E, CAP, OOR = OM.CONVERGED, OM.MAX_ITER_REACHED, OM.EMPTY_TRAJ, OM.STEP_CAP, OM.OUT_OF_RANGE
    sets = []
    conv0 = P(cost_th=1e30, max_iter=1)   # the nominal roll-out alone decides
    # the nominal roll-out: 16384 steps, then 16385
    a, b = _cap_distances(conv0)
    st, tg, pa = demo(2)
    pa[0] = (a, b)
    sets.append(("cap_nominal", st, tg, pa, conv0, (C, CAP)))
    # a Jacobian roll-out (distance + h_step[0]): towards a target 1500 ahead the line search shortens the distance
    one = P(max_iter=1)
    tj = (1500.0, 0.0, 0.0)
    a, b = jacobian_cap_distances(one, tj)
    st, tg, pa = demo(2)
    tg[:] = np.float32(tj)[:, None]
    pa[0] = (a, b)
    sets.append(("cap_jacobian", st, tg, pa, one, (MI, CAP)))
    # a line-search candidate (distance + 1.5 dp): the Jacobian roll-outs are the same on both sides, the target x
    # differs by one ulp
    a, b = flip(lambda x: opt_status(DEMO_ST, (x, 0, 0), (1000, 0, 0, 0), one) == CAP, 1300.0, 1600.0)
    st, tg, pa = demo(2)
    tg[0], tg[1:] = (a, b), 0.0
    pa[0] = 1000.0
    sets.append(("cap_line_search", st, tg, pa, one, (MI, CAP)))
    # the steering: at horizon 4 (distance 4, v = 1) the interpolation is exact and the first kp is steering[0]
    sv = (0.0, 0.0, 0.0, 1.0)
    a, b = flip(lambda k: gen_status(sv, (4.0, k, 0, 0), conv0) == OOR, 100.0, 130.0)
    st = np.tile(np.float32(sv)[:, None], (1, 4))
    tg = np.zeros((3, 4), f32)
    pa = np.zeros((4, 4), f32)
    pa[0], pa[1] = 4.0, (a, b, -a, -b)
    sets.append(("steer_120", st, tg, pa, conv0, (C, OOR, C, OOR)))
    # the start yaw
    a, b = flip(lambda y: opt_status((0, 0, y, 3), (5, 2, 0), (6, 0, 0, 0), conv0) == OOR, 100.0, 130.0)
    st, tg, pa = demo(4)
    st[2] = (a, b, -a, -b)
    sets.append(("start_yaw_120", st, tg, pa, conv0, (C, OOR, C, OOR)))
    # one Jacobian roll-out stops at the step cap (distance + h_step[0]) and another leaves the tanf range
    # (steering[2] + h_step[2] = 121): CRB_MPTG_OUT_OF_RANGE whatever order the six run in
    d = jacobian_cap_distances(one, tj)[1]
    st, tg, pa = demo(1)
    tg[:] = np.float32([[0.0], [500.0], [0.0]])
    pa[:, 0] = (d, 0.0, 0.0, 118.0)
    sets.append(("cap_and_out_of_range", st, tg, pa, P(max_iter=1, h_step=(0.2, 0.005, 3.0)), (OOR,)))
    # non-finite starts: v = 0 (dt = inf: one step to NaN, then a NaN parameter rolls out nothing), v < 0 and
    # v = inf (horizon <= 0: nothing), x or y NaN (NaN costs, NaN parameter)
    st, tg, pa = demo(5)
    st[3, :3] = (0.0, -3.0, np.inf)
    st[0, 3] = st[1, 4] = np.nan
    sets.append(("non_finite_start", st, tg, pa, P(), (E, E, E, E, E)))
    # a denormal ds: n = distance / ds = inf, dt = 0, the time never advances
    st, tg, pa = demo(1)
    sets.append(("denormal_ds", st, tg, pa, P(ds=1e-45), (CAP,)))
    return sets


def limit_sets():
    """Problems at the limits of include/crb.h: (name, state, target, param, params, statuses) with the status each
    column is built to end with.  Pairs of columns are the two sides of one limit: 16384 / 16385 steps (nominal,
    Jacobian and line-search roll-outs), |kp| = nextafter(120, 0) / 120, start yaw nextafter(120, 0) / 120."""
    return list(_limit_sets())
