"""Problem sets for tests/test_mptg.py and tests/golden/make_mptg_golden.py: seeded problems around the demo and
the reference's corner cases, each with the parameters it needs.  Every set is (name, state, target, param, params)."""
import numpy as np

from cpprobotics_b200 import synth
from oracle import mptg as OM


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
