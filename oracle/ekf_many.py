"""The EKF checker (oracle/oracle.py) composed model by model, for crb_ekf_step_many_batched: the agents that name
model m are one call of the unchanged batched checker, ekf_step_batched with model m's dt, Q and R (it takes them per
call, as the reference's ekf_estimation does).  An index outside [0, n_models) gives that agent NaN and BAD_MODEL.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: tests/, __graft_entry__.smoke() and scripts may import it, the product
package (cpprobotics_b200/) never does.
"""
from __future__ import annotations

import numpy as np

from . import oracle as OO

# include/crb.h
EKF_OK, EKF_BAD_MODEL = 0, 1


def step_many(x, P, z, u, dt, Q, R, model_of, n_steps=1, agents=None):
    """x [4, n], P [16, n], z, u [2 * n_steps, n]; the model table as dt [m], Q [m, 16], R [m, 4]; model_of [n].
    Returns new (x, P, status [n]).  agents (indices) restricts the work to those agents; the others keep their
    inputs and status EKF_OK."""
    x = np.array(x, np.float32)
    P = np.array(P, np.float32)
    z, u = np.asarray(z, np.float32), np.asarray(u, np.float32)
    dt = np.asarray(dt, np.float64).reshape(-1)
    Q = np.asarray(Q, np.float32).reshape(dt.size, 16)
    R = np.asarray(R, np.float32).reshape(dt.size, 4)
    mof = np.asarray(model_of).astype(np.int64)
    st = np.full(mof.size, EKF_OK, np.int32)
    sel = np.arange(mof.size) if agents is None else np.unique(np.asarray(agents, np.int64))
    ms = mof[sel]
    bad = sel[(ms < 0) | (ms >= dt.size)]
    x[:, bad] = np.nan
    P[:, bad] = np.nan
    st[bad] = EKF_BAD_MODEL
    good = sel[(ms >= 0) & (ms < dt.size)]
    order = good[np.argsort(mof[good], kind="stable")]
    models, starts = np.unique(mof[order], return_index=True)
    for m, cols in zip(models, np.split(order, starts[1:])):
        xo, Po = OO.ekf_step_batched(x[:, cols], P[:, cols], z[:, cols], u[:, cols], Q=Q[m], R=R[m], dt=float(dt[m]),
                                     n_steps=n_steps)
        x[:, cols], P[:, cols] = xo, Po
    return x, P, st
