"""One small invocation of each hot path on cuda:0, checked against the CPU oracle.

Called by __graft_entry__.smoke().  The oracle is imported here as the CHECKER only.
"""
from __future__ import annotations

import os
import sys

import numpy as np


def run() -> None:
    import torch

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    from oracle import dwa as OD  # checker only
    from oracle import mptg as OM  # checker only
    from oracle import oracle as O  # checker only

    from . import synth
    from .engine import Engine, mpc_default_params

    if not torch.cuda.is_available():
        raise RuntimeError("smoke() needs a CUDA device: cpprobotics_b200 has no CPU fallback")
    dev = torch.device("cuda:0")
    eng = Engine(0)

    # EKF: 4097 agents (ragged tail), 2 steps
    n = 4097
    x, P, z, u = synth.ekf_inputs(n, n_steps=2)
    xd, Pd, zd, ud = (torch.from_numpy(a).to(dev) for a in (x, P, z, u))
    eng.ekf_estimation(xd, Pd, zd, ud, n_steps=2)
    torch.cuda.synchronize()
    xo, Po = O.ekf_step_batched(x, P, z, u, n_steps=2)
    ex = np.abs(xd.cpu().numpy() - xo).max(axis=0) / np.abs(xo).max(axis=0)
    eP = np.abs(Pd.cpu().numpy() - Po).max(axis=0) / np.abs(Po).max(axis=0)
    assert ex.max() <= 1e-5 and eP.max() <= 1e-5, (ex.max(), eP.max())
    print(f"smoke EKF   n={n}: max field-normalised err x {ex.max():.2e} P {eP.max():.2e}")

    # PF: 4097 particles, 8 landmarks
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = (torch.from_numpy(a).to(dev) for a in (px, pw, noise))
    eng.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    ew = np.abs(pwd.cpu().numpy() - pwo).max() / np.abs(pwo).max()
    epx = np.abs(pxd.cpu().numpy() - pxo).max()
    assert ew <= 1e-5 and epx <= 1e-5, (ew, epx)
    print(f"smoke PF    n={n}: max err px {epx:.2e}  w (normalised) {ew:.2e}")

    # MPC: 1025 agents, T = 20, bit-exact against the oracle
    T, nm = 20, 1025
    course = synth.mpc_course()
    st, pind = synth.mpc_states(nm, course=course)
    xref, _ = synth.mpc_xref_numpy(st, pind, T, course=course)
    prm = mpc_default_params()
    prm.max_iter, prm.du_th, prm.max_ls = 50, 1e-4, 8
    std, xrd = torch.from_numpy(st).to(dev), torch.from_numpy(xref).to(dev)
    sol = torch.empty((4 * T + 2 * (T - 1), nm), dtype=torch.float32, device=dev)
    u0 = torch.empty((2, nm), dtype=torch.float32, device=dev)
    cost = torch.empty(nm, dtype=torch.float32, device=dev)
    status = torch.empty(nm, dtype=torch.int32, device=dev)
    iters = torch.empty(nm, dtype=torch.int32, device=dev)
    eng.mpc_solve(std, xrd, T, prm, sol=sol, u0=u0, cost=cost, status=status, iters=iters)
    torch.cuda.synchronize()
    ro = O.mpc_solve_batched(st, xref, T, O.mpc_params(max_iter=50, du_th=1e-4, max_ls=8))
    same = (np.array_equal(sol.cpu().numpy(), ro["sol"]) and np.array_equal(u0.cpu().numpy(), ro["u0"])
            and np.array_equal(cost.cpu().numpy(), ro["cost"])
            and np.array_equal(status.cpu().numpy(), ro["status"])
            and np.array_equal(iters.cpu().numpy(), ro["iters"]))
    assert same, "MPC GPU result is not bit-identical to the oracle"
    print(f"smoke MPC   n={nm} T={T}: bit-identical to the oracle; mean iters "
          f"{iters.float().mean().item():.2f}, converged+stationary "
          f"{int(((status == 0) | (status == 2)).sum().item())}/{nm}")
    # the same solve started in hinted order (the previous solve's iteration counts): the same bits
    sol2, u02, cost2 = torch.empty_like(sol), torch.empty_like(u0), torch.empty_like(cost)
    status2, iters2 = torch.empty_like(status), torch.empty_like(iters)
    eng.mpc_solve_hinted(std, xrd, T, iters, prm, sol=sol2, u0=u02, cost=cost2, status=status2, iters=iters2)
    torch.cuda.synchronize()
    assert (torch.equal(sol2, sol) and torch.equal(u02, u0) and torch.equal(cost2, cost)
            and torch.equal(status2, status) and torch.equal(iters2, iters)), "hinted MPC solve changed the result"
    print("smoke MPC   hinted order: bit-identical to the index-order solve")

    # one whole particle-filter iteration on the device (crb_pf_step) against the oracle's stages
    npf = 8192
    px, pw, noise = synth.pf_inputs(npf)
    uni = (1.0 + np.random.default_rng(7).random(npf)).astype(np.float32)
    pxd, pwd, nd, ud2 = (torch.from_numpy(a).to(dev) for a in (px, pw, noise, uni))
    nxt = torch.empty_like(pxd)
    res_d = eng.pf_step(pxd, pwd, nxt, nd, lm, uniforms=ud2, nth=float(npf))
    torch.cuda.synchronize()
    res = res_d.cpu().numpy()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pwn, xeo, Peo, swo = O.pf_estimate(pxo, pwo)
    assert res[22] == 1.0 and abs(res[20] - swo) <= 1e-5 * abs(swo), (res[20], swo)
    assert np.allclose(res[0:4], xeo, rtol=1e-5, atol=1e-5), (res[0:4], xeo)
    w_out = pwd.cpu().numpy()
    assert np.all(w_out == np.float32(1.0 / npf)), "resampled weights are not uniform"
    src = pxd.cpu().numpy()
    got = nxt.cpu().numpy()
    keys = {tuple(c) for c in src.T}
    assert all(tuple(c) in keys for c in got.T[:: max(1, npf // 256)]), "a resampled particle is not a copy of an input"
    print(f"smoke PF    full iteration n={npf}: sum_w / xEst match the oracle, particles resampled on the device")
    # DWA: 4097 robots against the demo's 10 obstacles, bit-identical to the oracle
    nd = 4097
    xw, uw, gw = synth.dwa_inputs(nd)
    ob = synth.DWA_DEMO_OBSTACLES
    n_pts = eng.dwa_rollout_points()
    xwd, uwd, gwd, obd = (torch.from_numpy(a).to(dev) for a in (xw, uw, gw, ob))
    cw = torch.empty(nd, dtype=torch.float32, device=dev)
    bw = torch.empty(nd, dtype=torch.int32, device=dev)
    tw = torch.empty((5 * n_pts, nd), dtype=torch.float32, device=dev)
    eng.dwa_control(xwd, uwd, gwd, obd, cost=cw, best=bw, traj=tw)
    torch.cuda.synchronize()
    rw = OD.dwa_control(xw, uw, gw, ob)
    same = all(np.array_equal(a.cpu().numpy().view(np.uint32), b.view(np.uint32))
               for a, b in ((uwd, rw["u"]), (cw, rw["cost"]), (bw, rw["best"]), (tw, rw["traj"])))
    assert same, "DWA GPU result is not bit-identical to the oracle"
    print(f"smoke DWA   n={nd} obstacles={len(ob)}: bit-identical to the oracle; "
          f"{int((bw >= 0).sum().item())}/{nd} robots with an admissible sample")
    # MPTG: 4097 trajectory optimisations around the demo's target, the same as the checker (any NaN equals any NaN)
    nm, mp = 4097, 64
    sm, tm, pm = synth.mptg_inputs(nm)
    smd, tmd, pmd = (torch.from_numpy(a).to(dev) for a in (sm, tm, pm))
    trm = torch.zeros((3 * mp, nm), dtype=torch.float32, device=dev)
    i32 = [torch.empty(nm, dtype=torch.int32, device=dev) for _ in range(3)]
    cm = torch.empty(nm, dtype=torch.float32, device=dev)
    eng.mptg_optimize(smd, tmd, pmd, traj=trm, traj_len=i32[0], cost=cm, status=i32[1], iters=i32[2])
    torch.cuda.synchronize()
    rm = OM.optimize(sm, tm, pm, max_pts=mp, traj_fill=0.0)

    def same_nan(a, b):
        a, b = a.cpu().numpy(), np.asarray(b)
        if a.dtype.kind != "f":
            return np.array_equal(a, b)
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    ok = all(same_nan(g, rm[k]) for g, k in ((pmd, "param"), (trm, "traj"), (i32[0], "traj_len"), (cm, "cost"),
                                            (i32[1], "status"), (i32[2], "iters")))
    assert ok, "MPTG GPU result is not bit-identical to the checker"
    print(f"smoke MPTG  n={nm}: bit-identical to the checker; "
          f"{int((i32[1] == 0).sum().item())}/{nm} converged")
    print(f"smoke ok: {eng.launches} kernel launches through libcrb.so")
    eng.close()
