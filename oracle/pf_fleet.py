"""The particle-filter checker (oracle/oracle.py) composed robot by robot, for crb_pf_step_many_batched: each robot's
filter is one call of the unchanged single-filter checker, pf_predict_weight_batched with the robot's u and its
observation list, then pf_estimate and pf_resample on its np particles.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import numpy as np

from . import oracle as OO

# include/crb.h
RESULT_LEN = 24
MAX_LANDMARKS = 64
FLEET_OK, FLEET_BAD_OBSERVATIONS = 0, 1


def list_ok(z_off, z_of, n_rows, r):
    """Whether robot r's list reference is valid (crb.h): index, offsets and at most MAX_LANDMARKS rows."""
    s = int(z_of[r])
    if not 0 <= s < len(z_off) - 1:
        return False
    lo, hi = int(z_off[s]), int(z_off[s + 1])
    return 0 <= lo <= hi <= n_rows and hi - lo <= MAX_LANDMARKS


def step_one(px, pw, u, rows, noise, uniforms, nth=None, consts=None):
    """One robot's pf_localization + resampling with the single-filter checker.  Returns (px predicted, pw, px_next,
    result [RESULT_LEN]) laid out as crb_pf_step's."""
    c = dict(consts or OO.pf_constants())
    c["u"] = np.asarray(u, np.float32)
    pxp, pwr = OO.pf_predict_weight_batched(px, pw, noise, rows, consts=c)
    pwn, xe, pe, sw = OO.pf_estimate(pxp, pwr)
    npr = pxp.shape[1]
    pxn, pwo, did, neff = OO.pf_resample(pxp, pwn, np.asarray(uniforms, np.float64), npr // 2 if nth is None else nth)
    res = np.empty(RESULT_LEN)
    res[0:4] = xe
    res[4:20] = np.asarray(pe, np.float32).T.reshape(-1)   # column-major
    res[20] = sw
    res[21] = neff
    res[22] = 1.0 if did else 0.0
    res[23] = float(np.sum(pwn.astype(np.float64) ** 2))
    return pxp, (pwo if did else pwn), (pxn if did else pxp.copy()), res


def step_many(np_per_robot, px, pw, u, z, z_off, z_of, noise, uniforms, nth=None, consts=None, robots=None):
    """crb_pf_step_many_batched's outputs from the checker: (px, pw, px_next, result [RESULT_LEN, n_robots], status).
    Robots outside `robots` (all when None) and robots with a bad list keep px / pw, get px_next = px and NaN results.
    noise [2, n] and uniforms [n] are explicit."""
    npr = int(np_per_robot)
    nr = int(np.asarray(u).shape[-1])
    z = np.asarray(z, np.float32).reshape(-1, 3)
    px_o, pw_o = np.array(px, np.float32), np.array(pw, np.float32)
    px_n = px_o.copy()
    res = np.full((RESULT_LEN, nr), np.nan)
    status = np.full(nr, FLEET_BAD_OBSERVATIONS, np.int32)
    for r in (range(nr) if robots is None else robots):
        if not list_ok(z_off, z_of, len(z), r):
            continue
        s = int(z_of[r])
        cols = slice(r * npr, (r + 1) * npr)
        a, b, c, d = step_one(px_o[:, cols], pw_o[cols], np.asarray(u)[:, r], z[int(z_off[s]):int(z_off[s + 1])],
                              np.asarray(noise)[:, cols], np.asarray(uniforms)[cols], nth, consts)
        px_o[:, cols], pw_o[cols], px_n[:, cols], res[:, r] = a, b, c, d
        status[r] = FLEET_OK
    return px_o, pw_o, px_n, res, status
