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
    # SLP: the biased sampler for 33 queries, the search in a synthetic 64-row table and the optimizer, as the checker
    from oracle import slp as OS  # checker only
    from ._lib import SlpSampler
    fs, qs = synth.slp_inputs(33, 1)
    ss = SlpSampler(fs["kind"], fs["nxy"], fs["nh"], fs["ns"], fs["d"])
    tbs = synth.slp_table(64)
    tsd, nsd, std_ = eng.slp_sample_states(ss, torch.from_numpy(qs).to(dev))
    gs = eng.slp_generate_path(tsd, torch.from_numpy(tbs).to(dev), max_pts=32)
    torch.cuda.synchronize()
    os_ = OS.sample(OS.sampler(fs["kind"], fs["nxy"], fs["nh"], fs["ns"], fs["d"]), qs)
    og = OS.generate_path(os_["target"], tbs, max_pts=32)
    ok = same_nan(tsd, os_["target"]) and same_nan(nsd, os_["n_states"]) and same_nan(std_, os_["status"])
    ok = ok and all(same_nan(gs[k], og[k]) for k in ("param", "traj", "traj_len", "cost", "status", "iters", "row"))
    assert ok, "SLP GPU result is not bit-identical to the checker"
    print(f"smoke SLP   {qs.shape[1]} queries, {int(nsd.sum().item())} states: bit-identical to the checker; "
          f"{int((gs['status'] == 0).sum().item())} converged")
    # grid A* / Dijkstra: the demo's map and 65 queries on it per planner, as the checker
    from oracle import grid as OG  # checker only
    from ._lib import GridBox
    gox, goy = synth.grid_demo_obstacles()
    gd = synth.GRID_DEMO
    gb = OG.box_of_obstacles(gox, goy, gd["reso"])
    gm = OG.obstacle_map(gox, goy, gd["reso"], gd["rr"], gb)
    gsg = synth.grid_inputs(65, gb, gm, gd["reso"])
    box = GridBox(*[int(v) for v in gb])
    gmd = eng.grid_obstacle_map(torch.from_numpy(gox).to(dev), torch.from_numpy(goy).to(dev), gd["reso"], gd["rr"], box)
    for algo in (OG.ASTAR, OG.DIJKSTRA):
        gr = eng.grid_plan(algo, box, gmd, gd["reso"], torch.from_numpy(gsg).to(dev), max_pts=128)
        torch.cuda.synchronize()
        go = OG.plan(algo, gb, gm, gd["reso"], gsg, max_pts=128)
        ok = same_nan(gmd, gm) and all(same_nan(gr[k], go[k]) for k in ("path", "path_len", "cost", "n_visited",
                                                                          "status"))
        assert ok, "grid planner GPU result is not bit-identical to the checker"
        print(f"smoke GRID  {'A*' if algo == OG.ASTAR else 'Dijkstra'} 65 queries on the demo map: bit-identical to "
              f"the checker; {int((gr['status'] == 0).sum().item())} found")
    # RRT: the demo's obstacles and 65 seeded queries on them, every output as the checker
    from oracle import rrt as OR  # checker only
    rd = synth.RRT_DEMO
    rob = synth.rrt_demo_obstacles()
    rse, rseed = synth.rrt_inputs(65, rob, rd["rand_min"], rd["rand_max"])
    rp = eng.rrt_default_params()
    rp.expand_dis, rp.max_iter = rd["expand_dis"], 4096
    rr = eng.rrt_plan(torch.from_numpy(rob).to(dev), torch.from_numpy(rse).to(dev),
                      torch.from_numpy(rseed.view(np.int32)).to(dev), rp, max_pts=64, max_nodes=512)
    torch.cuda.synchronize()
    ro = OR.plan(dict(rand_min=rp.rand_min, rand_max=rp.rand_max, expand_dis=rp.expand_dis,
                      goal_sample_rate=rp.goal_sample_rate, max_iter=rp.max_iter), rob, rse, rseed, max_pts=64,
                 max_nodes=512)
    ok = all(same_nan(rr[k], ro[k]) for k in ("path", "path_len", "tree", "parent", "n_nodes", "n_iter", "status"))
    assert ok, "RRT GPU result is not bit-identical to the checker"
    print(f"smoke RRT   65 queries on the demo map: bit-identical to the checker; "
          f"{int((rr['status'] == 0).sum().item())} found")
    # LQR path tracking: 4- and 5-state control, then update, for 257 vehicles on the demo-shaped course, every output as
    # the checker
    from oracle import lqrt as OL  # checker only
    lcourse = synth.lqr_course("demo")
    lst, lind, lpe, lpth = synth.lqr_track_inputs(257, lcourse, seed=0x5A0)
    dcourse = [torch.from_numpy(a).to(dev) for a in lcourse]
    for nx in (4, 5):
        dst = torch.from_numpy(lst).to(dev)
        dind, dpe, dpth = (torch.from_numpy(a.copy()).to(dev) for a in (lind, lpe, lpth))
        lr = eng.lqr_steering_control(nx, dst, dcourse[: 4 if nx == 4 else 5], dind, dpe, dpth)
        nu = 1 if nx == 4 else 2
        eng.lqr_update(dst, lr["u"][0].contiguous() if nx == 5 else torch.zeros_like(dpe), lr["u"][nu - 1].contiguous())
        torch.cuda.synchronize()
        lo = OL.control(nx, lst, lcourse, lind, lpe, lpth)
        lnew = OL.update(lst, lo["u"][0] if nx == 5 else np.zeros(257, np.float32), lo["u"][nu - 1])
        ok = all(same_nan(g, w) for g, w in ((lr["u"], lo["u"]), (dind, lo["ind"]), (dpe, lo["pe"]), (dpth, lo["pth_e"]),
                                             (lr["iters"], lo["iters"]), (lr["status"], lo["status"]), (dst, lnew)))
        assert ok, f"LQR tracking (nx {nx}) GPU result is not bit-identical to the checker"
    print("smoke LQRT  257 vehicles, 4- and 5-state control and update on the demo course: bit-identical to the checker")
    # a course per vehicle: 257 vehicles in random order over 8 fleet courses, 4- and 5-state control and the MPC
    # lookup, every output as the checker run course by course
    mcourses = synth.fleet_courses(8, seed=0x5A1)
    packed = synth.pack_courses(mcourses)
    mof = np.random.default_rng(0x5A2).integers(0, 8, 257).astype(np.int32)
    mst = np.zeros((4, 257), np.float32)
    mind = np.zeros(257, np.int32)
    for c in range(8):
        sel = np.nonzero(mof == c)[0]
        mst[:, sel], mind[sel] = synth.lqr_track_inputs(sel.size, mcourses[c], seed=c)[:2]
    dpk = [torch.from_numpy(a).to(dev) for a in packed]
    for nx in (4, 5):
        dind = torch.from_numpy(mind.copy()).to(dev)
        dz = torch.zeros(257, dtype=torch.float32, device=dev)
        dz2 = torch.zeros(257, dtype=torch.float32, device=dev)
        mr = eng.lqr_steering_control_many(nx, torch.from_numpy(mst).to(dev), dpk[:4] + dpk[5:] if nx == 4 else dpk,
                                           torch.from_numpy(mof).to(dev), dind, dz, dz2)
        torch.cuda.synchronize()
        ok = True
        for c in range(8):
            sel = np.nonzero(mof == c)[0]
            z = np.zeros(sel.size, np.float32)
            mo = OL.control(nx, mst[:, sel], mcourses[c], mind[sel], z, z)
            sel_t = torch.from_numpy(sel)
            ok = ok and all(same_nan(g[..., sel_t], w) for g, w in ((mr["u"].cpu(), mo["u"]), (dind.cpu(), mo["ind"]),
                                                                    (mr["status"].cpu(), mo["status"])))
        assert ok, f"many-course LQR tracking (nx {nx}) GPU result is not bit-identical to the checker"
    T = 8
    dti = torch.from_numpy(mind.copy()).to(dev)
    xr = torch.empty((4 * T, 257), dtype=torch.float32, device=dev)
    eng.calc_ref_trajectory_many(torch.from_numpy(mst).to(dev), (dpk[0], dpk[1], dpk[2], dpk[4], dpk[5]),
                                 torch.from_numpy(mof).to(dev), 1.0, dti, xr, T)
    torch.cuda.synchronize()
    xh, th = xr.cpu(), dti.cpu().numpy()
    for i in range(257):
        cx, cy, cyaw, _, sp = mcourses[mof[i]]
        wx, wt = O.calc_ref_trajectory(mst[:, i], cx, cy, cyaw, sp, 1.0, T, int(mind[i]))
        assert wt == th[i] and same_nan(xh[:, i], wx.reshape(-1)), "many-course MPC lookup is not the checker"
    print("smoke MANY  257 vehicles on 8 courses, LQR control (4 and 5 states) and the MPC lookup: bit-identical to "
          "the checker")
    # an obstacle list per robot: 257 DWA robots and 65 RRT queries in random order over 8 lists each (empty, 1-row
    # and 256-row lists among the DWA ones), every output as the checker run list by list
    dls = synth.dwa_fleet_obstacles(8, seed=0x5A3)
    dob, doff = synth.pack_obstacles(dls, 2)
    dof = np.random.default_rng(0x5A4).integers(0, 8, 257).astype(np.int32)
    xw, uw, gw = synth.dwa_inputs(257, seed=0x5A5)
    uwd = torch.from_numpy(uw).to(dev)
    cw = torch.empty(257, dtype=torch.float32, device=dev)
    bw = torch.empty(257, dtype=torch.int32, device=dev)
    tw = torch.empty((5 * n_pts, 257), dtype=torch.float32, device=dev)
    sw = eng.dwa_control_many(torch.from_numpy(xw).to(dev), uwd, torch.from_numpy(gw).to(dev),
                              (torch.from_numpy(dob).to(dev), torch.from_numpy(doff).to(dev)),
                              torch.from_numpy(dof).to(dev), cost=cw, best=bw, traj=tw)
    torch.cuda.synchronize()
    ok = bool((sw == 0).all().item())
    for s in range(8):
        sel = np.nonzero(dof == s)[0]
        rw = OD.dwa_control(xw[:, sel], uw[:, sel], gw[:, sel], dls[s])
        sel_t = torch.from_numpy(sel)
        ok = ok and all(same_nan(g[..., sel_t], rw[k]) for g, k in ((uwd.cpu(), "u"), (cw.cpu(), "cost"),
                                                                    (bw.cpu(), "best"), (tw.cpu(), "traj")))
    assert ok, "many-list DWA GPU result is not bit-identical to the checker"
    rls = synth.rrt_fleet_obstacles(8, seed=0x5A6, lo=rd["rand_min"], hi=rd["rand_max"])
    rob_, roff = synth.pack_obstacles(rls, 3)
    rof = np.random.default_rng(0x5A7).integers(0, 8, 65).astype(np.int32)
    rse = np.zeros((4, 65), np.float32)
    rseed = np.zeros(65, np.uint32)
    for s in range(8):
        sel = np.nonzero(rof == s)[0]
        rse[:, sel], rseed[sel] = synth.rrt_inputs(sel.size, rls[s], rd["rand_min"], rd["rand_max"], seed=s)
    rr = eng.rrt_plan_many((torch.from_numpy(rob_).to(dev), torch.from_numpy(roff).to(dev)),
                           torch.from_numpy(rof).to(dev), torch.from_numpy(rse).to(dev),
                           torch.from_numpy(rseed.view(np.int32)).to(dev), rp, max_pts=64, max_nodes=512)
    torch.cuda.synchronize()
    ok = True
    for s in range(8):
        sel = np.nonzero(rof == s)[0]
        ro = OR.plan(dict(rand_min=rp.rand_min, rand_max=rp.rand_max, expand_dis=rp.expand_dis,
                          goal_sample_rate=rp.goal_sample_rate, max_iter=rp.max_iter), rls[s], rse[:, sel], rseed[sel],
                     max_pts=64, max_nodes=512)
        sel_t = torch.from_numpy(sel)
        ok = ok and all(same_nan(rr[k].cpu()[..., sel_t], ro[k]) for k in ("path", "path_len", "tree", "parent",
                                                                          "n_nodes", "n_iter", "status"))
    assert ok, "many-list RRT GPU result is not bit-identical to the checker"
    print("smoke OBST  257 DWA robots and 65 RRT queries, each among its own obstacles (8 lists each): bit-identical "
          "to the checker")
    # a map per query: 8 small fleet maps built in one launch, then 129 queries in random order over them per planner,
    # every map and output as the checker run map by map
    from oracle import grid_many as OGM  # checker only
    from .engine import grid_map_table
    gf = synth.grid_fleet_maps(8, seed=0x5A8)
    gt = grid_map_table(gf["boxes"], gf["reso"])
    gob, goff = synth.pack_obstacles(gf["lists"], 2)
    gdt = tuple(torch.from_numpy(a).to(dev) for a in gt[:3]) + (gt[3],)
    gmaps, gst = eng.grid_obstacle_map_many((torch.from_numpy(gob).to(dev), torch.from_numpy(goff).to(dev)),
                                            torch.from_numpy(gf["ob_of"]).to(dev), torch.from_numpy(gf["rr"]).to(dev),
                                            gdt)
    gwant, _ = OGM.obstacle_map_many(gob, goff, gf["ob_of"], gf["rr"], *gt[:3], int(gt[2][-1]), gt[3])
    assert bool((gst == 0).all().item()) and same_nan(gmaps, gwant), "many-map grid build is not the checker"
    gmof, gmsg = synth.grid_fleet_inputs(129, gt[0], gt[1], gwant, gt[2], seed=0x5A9)
    for algo in (OG.ASTAR, OG.DIJKSTRA):
        gr = eng.grid_plan_many(algo, gdt, gmaps, torch.from_numpy(gmof).to(dev), torch.from_numpy(gmsg).to(dev),
                                max_pts=32)
        torch.cuda.synchronize()
        go = OGM.plan_many(algo, *gt[:3], gwant, gt[3], gmof, gmsg, max_pts=32)
        ok = all(same_nan(gr[k], go[k]) for k in ("path", "path_len", "cost", "n_visited", "status"))
        assert ok, "many-map grid planner GPU result is not bit-identical to the checker"
    print("smoke MAPS  8 grid maps in one build, 129 queries over them per planner: bit-identical to the checker")

    # ---- a particle filter per robot: one fleet step against the checker composed robot by robot ----
    from oracle import pf_fleet as PFF  # checker only
    nfr, nfp = 33, 100
    ff = synth.pf_fleet_inputs(nfr, nfp, seed=0x5F)
    fx, fw = torch.from_numpy(ff["px"]).to(dev), torch.from_numpy(ff["pw"]).to(dev)
    fxn = torch.zeros_like(fx)
    fst = torch.empty(nfr, dtype=torch.int32, device=dev)
    fres = eng.pf_step_many(nfp, fx, fw, fxn, torch.from_numpy(ff["u"]).to(dev),
                            (torch.from_numpy(ff["z"]).to(dev), torch.from_numpy(ff["z_off"]).to(dev)),
                            torch.from_numpy(ff["z_of"]).to(dev), noise=torch.from_numpy(ff["noise"]).to(dev),
                            uniforms=torch.from_numpy(ff["uniforms"]).to(dev), status=fst)
    torch.cuda.synchronize()
    cx, cw, cxn, cres, cst = PFF.step_many(nfp, ff["px"], ff["pw"], ff["u"], ff["z"], ff["z_off"], ff["z_of"],
                                           ff["noise"], ff["uniforms"])
    gres = fres.cpu().numpy()
    assert (fst.cpu().numpy() == cst).all(), "fleet PF status differs from the checker"
    assert np.abs(fx.cpu().numpy() - cx).max() <= 1e-5, "fleet PF particles differ from the checker"
    assert np.abs(gres[:4] - cres[:4]).max() <= 1e-4, "fleet PF estimate differs from the checker"
    print(f"smoke FLEET PF {nfr} robots x {nfp} particles, each with its own u and observations: particles and xEst "
          f"match the checker, {int(gres[22].sum())} robots resampled")

    # ---- an EKF noise model per agent: one mixed-model launch against the checker composed model by model ----
    from oracle import ekf_many as OEM  # checker only
    from .engine import ekf_models
    ef = synth.ekf_fleet_inputs(4097, 8, seed=0xE4, n_steps=2)
    ef["model_of"][[7, 4000]] = [-1, 8]   # two bad indices
    ed = [torch.from_numpy(ef[k]).to(dev) for k in ("x", "P", "z", "u")]
    est = torch.full((4097,), -1, dtype=torch.int32, device=dev)
    eng.ekf_estimation_many(*ed, torch.from_numpy(ekf_models(ef["dt"], ef["Q"], ef["R"])).to(dev),
                            torch.from_numpy(ef["model_of"]).to(dev), n_steps=2, status=est)
    torch.cuda.synchronize()
    cx, cP, cst = OEM.step_many(ef["x"], ef["P"], ef["z"], ef["u"], ef["dt"], ef["Q"], ef["R"], ef["model_of"],
                                n_steps=2)
    gx, gP = ed[0].cpu().numpy(), ed[1].cpu().numpy()
    assert (est.cpu().numpy() == cst).all(), "model-table EKF status differs from the checker"
    assert np.array_equal(np.isnan(gx), np.isnan(cx)) and np.array_equal(np.isnan(gP), np.isnan(cP))
    ok = ~np.isnan(cx).any(axis=0)
    ex = (np.abs(gx[:, ok] - cx[:, ok]).max(axis=0) / np.abs(cx[:, ok]).max(axis=0)).max()
    eP = (np.abs(gP[:, ok] - cP[:, ok]).max(axis=0) / np.abs(cP[:, ok]).max(axis=0)).max()
    assert ex <= 1e-5 and eP <= 1e-5, (ex, eP)
    print(f"smoke EKF MODELS 4097 agents over 8 noise models, 2 bad indices: max field-normalised err x {ex:.2e} "
          f"P {eP:.2e}")
    print(f"smoke ok: {eng.launches} kernel launches through libcrb.so")
    eng.close()
