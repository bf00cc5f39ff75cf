"""Writes tests/golden/ref_golden.npz: inputs and the outputs of the REFERENCE'S OWN SOURCE TEXT
(oracle/_ref/libref_*.so = the unmodified files of /root/reference/src compiled against the header shims
of oracle/shim, see oracle/shim/README.md) on seeded inputs.  tests/test_oracle_ref_golden.py checks the
CPU oracle against this file bit for bit, so the pin also holds where neither /root/reference nor
oracle/_ref exists (a fresh clone, the GPU box).

    make -C oracle && python tests/golden/make_ref_golden.py        (needs /root/reference)
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from cpprobotics_b200 import synth  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle._load import reference  # noqa: E402

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def main():
    L = reference("ekf")
    if L is None:
        raise SystemExit("oracle/_ref not built: needs the reference tree (make -C oracle)")
    out = {}
    # ---- EKF: ekf_estimation (src/extended_kalman_filter.cpp:64-78), 512 agents x 1 step ------------------
    L.ref_ekf_estimation.argtypes = [f32p] * 6
    n = 512
    x, P, z, u = synth.ekf_inputs(n, seed=0xBEEF)
    _, Q, R = O.ekf_constants()
    xo, Po = np.zeros_like(x), np.zeros_like(P)
    for i in range(n):
        xi, Pi = np.ascontiguousarray(x[:, i]).copy(), np.ascontiguousarray(P[:, i]).copy()
        L.ref_ekf_estimation(xi, Pi, np.ascontiguousarray(z[:, i]), np.ascontiguousarray(u[:, i]), Q, R)
        xo[:, i], Po[:, i] = xi, Pi
    out.update(ekf_x=x, ekf_P=P, ekf_z=z, ekf_u=u, ekf_x_out=xo, ekf_P_out=Po)

    # ---- PF: pf_localization (:73-109) and resampling (:111-148), NP = 100 ---------------------------------
    L = reference("pf")
    L.ref_pf_np.restype = C.c_int
    L.ref_pf_localization.argtypes = [f32p, f32p, f32p, f32p, f32p, C.c_int, f32p, f32p, C.c_float, C.c_uint, f64p]
    L.ref_resampling.restype = C.c_int
    L.ref_resampling.argtypes = [f32p, f32p, C.c_uint, f64p]
    NP = L.ref_pf_np()
    c = O.pf_constants()
    for case, seed in enumerate((9, 10, 11)):
        px, pw, _ = synth.pf_inputs(NP, seed=seed)
        lm = synth.pf_landmarks(4, seed=seed)
        pxr, pwr = np.ascontiguousarray(px.T.reshape(-1)).copy(), pw.copy()
        xe, Pe, draws = np.zeros(4, np.float32), np.zeros(16, np.float32), np.zeros(2 * NP)
        L.ref_pf_localization(pxr, pwr, xe, Pe, np.ascontiguousarray(lm.reshape(-1)), len(lm), c["u"],
                              c["rsim_diag"], float(c["Q"]), 4242 + seed, draws)
        out.update({f"pf{case}_px": px, f"pf{case}_pw": pw, f"pf{case}_lm": lm, f"pf{case}_draws": draws,
                    f"pf{case}_px_out": pxr.reshape(NP, 4).T.copy(), f"pf{case}_pw_out": pwr,
                    f"pf{case}_xEst": xe, f"pf{case}_PEst": Pe})
        # resampling on the weighted set the reference just produced
        rx, rw, rdraws = pxr.copy(), pwr.copy(), np.zeros(NP)
        did = L.ref_resampling(rx, rw, 99 + seed, rdraws)
        out.update({f"rs{case}_draws": rdraws, f"rs{case}_did": np.int32(did),
                    f"rs{case}_px_out": rx.reshape(NP, 4).T.copy(), f"rs{case}_pw_out": rw})

    # ---- MPC helpers: update (:69-81), calc_nearest_index / calc_ref_trajectory (:107-170), FG_EVAL (:199-252)
    L = reference("mpc")
    L.ref_mpc_T.restype = C.c_int
    L.ref_update.argtypes = [f32p, C.c_float, C.c_float]
    L.ref_calc_ref_trajectory.argtypes = [f32p, f32p, f32p, f32p, f32p, C.c_int, C.c_float, C.POINTER(C.c_int), f32p]
    L.ref_fg_eval.argtypes = [f32p, f64p, f64p]
    T = L.ref_mpc_T()
    rng = np.random.default_rng(2)
    m = 300
    st = np.stack([rng.uniform(-50, 50, m), rng.uniform(-50, 50, m), rng.uniform(-3, 3, m),
                   rng.uniform(-6, 15.4, m)]).astype(np.float32)
    acc, dl = rng.uniform(-1.5, 1.5, m).astype(np.float32), rng.uniform(-1, 1, m).astype(np.float32)
    upd = np.zeros_like(st)
    for i in range(m):
        r = np.ascontiguousarray(st[:, i]).copy()
        L.ref_update(r, acc[i], dl[i])
        upd[:, i] = r
    out.update(upd_state=st, upd_a=acc, upd_delta=dl, upd_out=upd)
    course = synth.mpc_course()
    cx, cy, cyaw, sp = course
    cst, pind = synth.mpc_states(300, seed=3, course=course)
    xr_out, ti_out = np.zeros((4 * T, 300), np.float32), np.zeros(300, np.int32)
    for i in range(300):
        ti = C.c_int(int(pind[i])); xr = np.zeros(4 * T, np.float32)
        L.ref_calc_ref_trajectory(np.ascontiguousarray(cst[:, i]), cx, cy, cyaw, sp, len(cx), 1.0, C.byref(ti), xr)
        xr_out[:, i], ti_out[i] = xr, ti.value
    out.update(crt_state=cst, crt_pind=pind.astype(np.int32), crt_T=np.int32(T), crt_xref=xr_out, crt_tind=ti_out)
    nv = 4 * T + 2 * (T - 1)
    v = rng.normal(size=(20, nv))
    fg = np.zeros((20, 1 + 4 * T))
    for i in range(20):
        L.ref_fg_eval(np.ascontiguousarray(xr_out[:, i]), np.ascontiguousarray(v[i]), fg[i])
    out.update(fg_vars=v, fg_out=fg)

    # ---- LQR: solve_DARE + dlqr of both demos (lqr_steer_control.cpp:75-96, lqr_speed_steer_control.cpp:85-106)
    for nx, nu in ((4, 1), (5, 2)):
        L = reference(f"lqr{nx}")
        A, B, Qm, Rm = synth.lqr_inputs(64, nx, seed=77)
        K, X = np.zeros((nu * nx, 64), np.float32), np.zeros((nx * nx, 64), np.float32)
        for i in range(64):
            k, xx = np.zeros(nu * nx, np.float32), np.zeros(nx * nx, np.float32)
            a, b = np.ascontiguousarray(A[:, i]), np.ascontiguousarray(B[:, i])
            if nx == 4:
                L.ref_dlqr4.argtypes = [f32p, f32p, f32p, C.c_float, f32p, f32p]
                L.ref_dlqr4(a, b, Qm, float(Rm[0]), k, xx)
            else:
                L.ref_dlqr5.argtypes = [f32p] * 6
                L.ref_dlqr5(a, b, Qm, Rm, k, xx)
            K[:, i], X[:, i] = k, xx
        out.update({f"lqr{nx}_A": A, f"lqr{nx}_B": B, f"lqr{nx}_Q": Qm, f"lqr{nx}_R": Rm, f"lqr{nx}_K": K,
                    f"lqr{nx}_X": X})
    np.savez_compressed(os.path.join(HERE, "ref_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "ref_golden.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
