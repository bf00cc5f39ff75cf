"""GPU parity tests proper: the CUDA path, called through the C ABI (libcrb.so), against the CPU
oracle on the same seeded inputs.  Run with `-m gpu` on an H100."""
import os

import numpy as np
import pytest

from cpprobotics_b200 import mpc_default_params, synth
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _dev(*arrs):
    import torch
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs)


def field_err(got, want):
    """SURVEY §8 d-8 primary gate: per agent, max|gpu-cpu| / max|cpu| over the field."""
    return (np.abs(got - want).max(axis=0) / np.abs(want).max(axis=0)).max()


# ---- EKF ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,steps", [(1, 1), (33, 1), (4097, 1), (100_000, 1), (1000, 7), (1, 1000)])
def test_ekf_device_matches_oracle(engine, n, steps):
    import torch
    x, P, z, u = synth.ekf_inputs(n, n_steps=steps)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud, n_steps=steps)
    torch.cuda.synchronize()
    xo, Po = O.ekf_step_batched(x, P, z, u, n_steps=steps)
    tol = 1e-5 if steps < 100 else 1e-4   # a 1-ulp sin/cos difference (glibc's FMA build) compounds over 1000 steps
    assert field_err(xd.cpu().numpy(), xo) <= tol
    assert field_err(Pd.cpu().numpy(), Po) <= tol
    # sin/cos carry the host libm's bits (crb_sincosf_libm) and every other operation follows the oracle's
    # order: a one-step update is IDENTICAL to the oracle for all but a handful of agents
    if steps == 1:
        same = (xd.cpu().numpy() == xo).all(axis=0) & (Pd.cpu().numpy() == Po).all(axis=0)
        assert (~same).sum() <= max(1, int(4e-6 * n)), int((~same).sum())


def test_ekf_host_entry_matches_device_entry_bitwise(engine):
    import torch
    n = 300_001   # > 2 chunks, ragged tail
    x, P, z, u = synth.ekf_inputs(n)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud)
    torch.cuda.synchronize()
    xh, Ph = x.copy(), P.copy()
    engine.ekf_estimation_host(xh, Ph, z, u)
    assert np.array_equal(xh, xd.cpu().numpy()) and np.array_equal(Ph, Pd.cpu().numpy())


def test_ekf_empty_batch_is_a_noop(engine):
    import torch
    e = torch.empty((4, 0), device="cuda"), torch.empty((16, 0), device="cuda")
    zu = torch.empty((2, 0), device="cuda")
    engine.ekf_estimation(e[0], e[1], zu, zu)


def test_ekf_known_answer(engine):
    """Hand-derivable step from the reference's main() constants (SURVEY Appendix A.1)."""
    import torch
    x = np.zeros((4, 1), np.float32)
    P = np.eye(4, dtype=np.float32).T.reshape(16, 1).copy()
    z = np.array([[0.1], [0.0]], np.float32)
    u = np.array([[1.0], [0.1]], np.float32)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud)
    torch.cuda.synchronize()
    got = xd.cpu().numpy()[:, 0]
    np.testing.assert_allclose(got, [0.1, 0.0, 0.010000001, 1.0], rtol=0, atol=1e-7)
    Pg = Pd.cpu().numpy()[:, 0].reshape(4, 4).T
    assert abs(Pg[0, 0] - 0.50495052) < 1e-6 and abs(Pg[3, 3] - 1.0050495) < 1e-6


# ---- PF ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,n_lm", [(1, 4), (4097, 8), (200_000, 8), (1000, 0), (1000, 64)])
def test_pf_device_matches_oracle(engine, n, n_lm):
    import torch
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(n_lm) if n_lm else np.zeros((0, 3), np.float32)
    pxd, pwd, nd = _dev(px, pw, noise)
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    _assert_pf_parity(pxd.cpu().numpy(), pwd.cpu().numpy(), pxo, pwo, lm)


def _assert_pf_parity(px_got, pw_got, px_want, pw_want, lm, sigma2=0.01):
    """SURVEY §8 d-8 for the particle filter, as written: per-particle relative 1e-5 on w.

    The kernels evaluate sin/cos with glibc's own binary64 algorithm (crb_sincosf_libm), so the predicted
    positions carry the HOST libm's bits: they must be IDENTICAL to the oracle's, except on the ~2e-8 of the
    arguments where glibc's FMA build rounds an intermediate differently (then 1 ulp).  On every particle with
    identical positions the weight must agree to 1e-5 RELATIVE (w > 1e-30; the kernel's single fused
    exponential differs from the reference's eight rounded factors by <= ~1e-6).  The few particles whose
    position is an ulp off get the condition-number gate (one ulp of position is 3e-5 of w per landmark)."""
    same = (px_got == px_want).all(axis=0)
    n = same.size
    n_off = int((~same).sum())
    assert n_off <= max(2, int(4e-6 * n)), f"{n_off} of {n} predicted positions differ from the host libm path"
    assert np.abs(px_got - px_want).max() <= 1e-6 * max(1.0, np.abs(px_want).max())
    big = same & (pw_want > 1e-30)
    rel = np.abs(pw_got[big].astype(np.float64) - pw_want[big]) / pw_want[big]
    assert rel.size == 0 or rel.max() <= 1e-5, float(rel.max())
    # underflow region: the reference's running product goes denormal / 0, the kernel floors exp at 2^-126
    small = same & ~(pw_want > 1e-30)
    assert np.abs(pw_got[small].astype(np.float64) - pw_want[small]).max(initial=0.0) <= 1e-29
    if n_off:
        off = ~same
        cond = np.zeros(n_off)
        ulp = 0.0
        for r, lx, ly in lm:
            prez = np.hypot(px_want[0, off].astype(np.float64) - lx, px_want[1, off].astype(np.float64) - ly)
            cond += np.abs(prez - r) / sigma2
            ulp = max(ulp, float(np.spacing(np.float32(prez.max()))))
        tol = 1e-5 * np.abs(pw_want).max() + np.abs(pw_want[off]) * (cond * 4 * ulp + 32 * 2.0 ** -23)
        assert (np.abs(pw_got[off].astype(np.float64) - pw_want[off]) <= tol).all()


def test_pf_bitwise_when_trig_is_exact(engine):
    """yaw = 0 makes sinf/cosf exact on both sides: positions must then agree bit for bit, and the
    weights within the 2 ulp of expf per landmark."""
    import torch
    n = 10_000
    px, pw, noise = synth.pf_inputs(n)
    px[2] = 0.0
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = _dev(px, pw, noise)
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    assert np.array_equal(pxd.cpu().numpy(), pxo)
    rel = np.abs(pwd.cpu().numpy() - pwo) / np.maximum(pwo, 1e-37)
    assert rel[pwo > 1e-30].max() <= 1e-5


def test_pf_fused_exponent_weights_are_within_3_ulp_of_exact(engine):
    """The default PF kernels take one exponential of a float-float sum instead of the reference's eight
    rounded factors.  With yaw = 0 the positions are bit-exact, so every q_l = dz_l^2 / (2 sigma^2) can be
    restated in numpy binary32 and the weight evaluated exactly in binary64: the GPU must be within 5e-7
    of it (and is at least as close to it as the reference-order oracle is)."""
    import torch
    n = 20_000
    px, pw, noise = synth.pf_inputs(n)
    px[2] = 0.0
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = _dev(px, pw, noise)
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    assert np.array_equal(pxd.cpu().numpy(), pxo)
    f32 = np.float32
    sigma = np.sqrt(f32(0.01))
    two_s2 = f32(2) * sigma * sigma
    pre = 1.0 / np.sqrt(2.0 * 3.141592653 * float(sigma) * float(sigma))
    expo = np.full(n, len(lm) * np.log(pre), np.float64)
    for r, lx, ly in lm.astype(f32):
        dx, dy = pxo[0] - lx, pxo[1] - ly
        prez = np.sqrt(dx * dx + dy * dy)           # binary32 throughout, like the kernel and the reference
        dz = prez - r
        q = (dz * dz) / two_s2
        assert q.dtype == np.float32
        expo -= q.astype(np.float64)
    exact = pw.astype(np.float64) * np.exp(expo)
    ok = exact > 1e-30
    got = pwd.cpu().numpy().astype(np.float64)
    err_gpu = np.abs(got - exact)[ok] / exact[ok]
    err_ref = np.abs(pwo.astype(np.float64) - exact)[ok] / exact[ok]
    assert err_gpu.max() <= 5e-7, err_gpu.max()
    assert err_gpu.mean() <= err_ref.mean()


def test_pf_philox_mode_matches_oracle(engine):
    import torch
    n = 50_000
    px, pw, _ = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxd, pwd = _dev(px, pw)
    engine.pf_predict_weight(pxd, pwd, None, lm, seed=0x1234_5678_9ABC)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, None, lm, seed=0x1234_5678_9ABC)
    # Box-Muller: sin/cos of the angle carry the host libm's bits, logf is CUDA's (<= 1 ulp from glibc's), so
    # the noise and with it the predicted positions agree to an ulp or two: gated at 1e-5 on the POSITIONS.
    # (The weights are exp(-dz^2 / 2 sigma^2) of those positions, 3e-5 per ulp and landmark: their gate with
    # identical noise is test_pf_device_matches_oracle.)
    got_x = pxd.cpu().numpy()
    assert (np.abs(got_x - pxo).max(axis=1) <= 1e-5 * np.maximum(1.0, np.abs(pxo).max(axis=1))).all()
    assert np.mean(got_x == pxo) > 0.9           # most coordinates are in fact identical
    got, want = pwd.cpu().numpy(), pwo
    lw = np.abs(np.log(np.maximum(got, 1e-37)) - np.log(np.maximum(want, 1e-37)))[want > 1e-30]
    assert lw.max() < 0.02 and np.median(lw) < 1e-4


def test_pf_host_entry_matches_device_entry_bitwise(engine):
    import torch
    n = 600_001
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = _dev(px, pw, noise)
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxh, pwh = px.copy(), pw.copy()
    engine.pf_predict_weight_host(pxh, pwh, noise, lm)
    assert np.array_equal(pxh, pxd.cpu().numpy()) and np.array_equal(pwh, pwd.cpu().numpy())


def test_pf_estimate_matches_oracle(engine):
    import torch
    n = 100_003
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pxd, pwd = _dev(pxo, pwo)
    xe, Pe, sw = engine.pf_estimate(pxd, pwd)
    torch.cuda.synchronize()
    pwn, xeo, Peo, swo = O.pf_estimate(pxo, pwo)
    assert abs(sw - swo) <= 1e-12 * abs(swo) + 1e-30
    np.testing.assert_allclose(xe, xeo, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(Pe, Peo, rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(pwd.cpu().numpy(), pwn, rtol=1e-6, atol=0)
    assert abs(float(pwd.sum().item()) - 1.0) < 1e-3


# ---- MPC ---------------------------------------------------------------------------------------------
def _mpc_case(n, T, seed=0xC0FFEE):
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, seed=seed, course=course)
    xref, _ = synth.mpc_xref_numpy(st, pind, T, course=course)
    return st, xref


def _mpc_gpu(engine, st, xref, T, prm, u_init=None, host=False):
    import torch
    n = st.shape[1]
    nsol = 4 * T + 2 * (T - 1)
    if host:
        out = dict(sol=np.empty((nsol, n), np.float32), u0=np.empty((2, n), np.float32),
                   cost=np.empty(n, np.float32), status=np.empty(n, np.int32),
                   iters=np.empty(n, np.int32))
        engine.mpc_solve_host(st, xref, T, prm, u_init=u_init, **out)
        return out
    std, xrd = _dev(st, xref)
    uid = _dev(u_init)[0] if u_init is not None else None
    out = dict(sol=torch.empty((nsol, n), dtype=torch.float32, device="cuda"),
               u0=torch.empty((2, n), dtype=torch.float32, device="cuda"),
               cost=torch.empty(n, dtype=torch.float32, device="cuda"),
               status=torch.empty(n, dtype=torch.int32, device="cuda"),
               iters=torch.empty(n, dtype=torch.int32, device="cuda"))
    engine.mpc_solve(std, xrd, T, prm, u_init=uid, **out)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _params(**kw):
    p = mpc_default_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("n,T,max_iter,du_th", [(1, 20, 50, 1e-4), (257, 20, 50, 1e-4), (4096, 20, 50, 1e-4),
                                                (513, 6, 50, 1e-4), (513, 20, 3, 0.1), (129, 32, 20, 1e-3),
                                                (65, 2, 10, 1e-4)])
def test_mpc_device_bit_exact_vs_oracle(engine, n, T, max_iter, du_th):
    st, xref = _mpc_case(n, T)
    got = _mpc_gpu(engine, st, xref, T, _params(max_iter=max_iter, du_th=du_th, max_ls=8))
    want = O.mpc_solve_batched(st, xref, T, O.mpc_params(max_iter=max_iter, du_th=du_th, max_ls=8))
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(got[k], want[k]), k


def test_mpc_warm_start_and_speed_limits_bit_exact(engine):
    """u_init given; reference speed above MAX_SPEED so the speed bound (:298-301) is active."""
    n, T = 300, 20
    st, xref = _mpc_case(n, T, seed=7)
    xref = xref.copy()
    xref[3::4] = 20.0                       # ask for 20 m/s > 55/3.6
    st = st.copy(); st[3] = 14.9 + 0.3 * (np.arange(n) % 3)   # near / above the limit
    rng = np.random.default_rng(0)
    u_init = rng.uniform(-1.2, 1.2, size=(2 * (T - 1), n)).astype(np.float32)  # partly infeasible
    got = _mpc_gpu(engine, st, xref, T, _params(max_iter=30, du_th=1e-4, max_ls=8), u_init=u_init)
    want = O.mpc_solve_batched(st, xref, T, O.mpc_params(max_iter=30, du_th=1e-4, max_ls=8), u_init=u_init)
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(got[k], want[k]), k
    v = got["sol"][3 * T:4 * T]
    vmax = np.float32(55.0 / 3.6)
    feas = st[3] <= vmax                       # agents that start inside the speed limit stay inside
    assert v[1:, feas].max() <= vmax * (1 + 1e-6)
    assert v[2:, ~feas].max() <= vmax * (1 + 1e-6)        # the others are back inside after 2 steps of a=-1


def test_mpc_nonfinite_inputs_flagged(engine):
    n, T = 64, 20
    st, xref = _mpc_case(n, T)
    st = st.copy(); st[2, 5] = np.nan; xref = xref.copy(); xref[8, 9] = np.inf
    got = _mpc_gpu(engine, st, xref, T, _params(max_iter=10, du_th=1e-4, max_ls=8))
    want = O.mpc_solve_batched(st, xref, T, O.mpc_params(max_iter=10, du_th=1e-4, max_ls=8))
    assert got["status"][5] == 3 and got["status"][9] == 3
    assert np.array_equal(got["status"], want["status"])
    ok = got["status"] != 3
    assert np.array_equal(got["u0"][:, ok], want["u0"][:, ok])


def test_mpc_host_entry_matches_device_entry_bitwise(engine):
    n, T = 70_001, 20     # > 2 chunks, ragged
    st, xref = _mpc_case(n, T)
    prm = _params(max_iter=50, du_th=1e-4, max_ls=8)
    a = _mpc_gpu(engine, st, xref, T, prm)
    b = _mpc_gpu(engine, st, xref, T, prm, host=True)
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(a[k], b[k]), k


def test_mpc_straight_line_is_stationary(engine):
    """Known answer (SURVEY §8 c-6): on a straight reference at constant speed, starting on it,
    delta = 0, a = 0 and the cost is (numerically) zero."""
    T, n = 20, 4
    v = np.float32(10.0 / 3.6)
    st = np.zeros((4, n), np.float32); st[3] = v
    xref = np.zeros((4 * T, n), np.float32)
    for t in range(T):
        xref[4 * t + 0] = v * np.float32(0.2) * t
        xref[4 * t + 3] = v
    got = _mpc_gpu(engine, st, xref, T, _params(max_iter=50, du_th=1e-4, max_ls=8))
    assert np.abs(got["u0"]).max() < 1e-4 and got["cost"].max() < 1e-6


def test_plant_update_matches_oracle(engine):
    import torch
    n = 5000
    st, _ = synth.mpc_states(n)
    rng = np.random.default_rng(3)
    u0 = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.0, 1.0, n)]).astype(np.float32)
    st[3, :100] = 15.2   # exercise the speed clamp
    std, u0d = _dev(st, u0)
    engine.mpc_plant_update(std, u0d)
    torch.cuda.synchronize()
    want = np.stack([O.plant_update(st[:, i], u0[0, i], u0[1, i]) for i in range(n)], axis=1)
    got = std.cpu().numpy()
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def test_calc_ref_trajectory_bit_exact(engine):
    """Integer index work must be bit-exact (SURVEY §8 d-8), including near the end of the course."""
    import torch
    n, T = 20_000, 20
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, course=course)
    pind = pind.copy(); pind[:50] = len(course[0]) - 1 - np.arange(50) % 12   # window runs off the end
    st[3, 50:100] = -3.0                                                        # negative speed: |v|
    cd = _dev(*course)
    std = _dev(st)[0]
    tid = torch.from_numpy(pind.copy()).cuda()
    xr = torch.empty((4 * T, n), dtype=torch.float32, device="cuda")
    engine.calc_ref_trajectory(std, *cd, 1.0, tid, xr, T)
    torch.cuda.synchronize()
    got_x, got_t = xr.cpu().numpy(), tid.cpu().numpy()
    for i in list(range(200)) + list(range(n - 200, n)):
        wx, wt = O.calc_ref_trajectory(st[:, i], *course, 1.0, T, int(pind[i]))
        assert wt == got_t[i]
        assert np.array_equal(wx.reshape(-1), got_x[:, i])
    # and the vectorised numpy restatement used by the synthetic generator agrees on the whole batch
    xn, tn = synth.mpc_xref_numpy(st, pind, T, course=course)
    assert np.array_equal(tn, got_t) and np.array_equal(xn, got_x)


# ---- stats ------------------------------------------------------------------------------------------
def test_stats_reduce(engine):
    import torch
    n = 100_001
    rng = np.random.default_rng(1)
    v = rng.normal(size=n).astype(np.float32); v[17] = np.nan
    status = (rng.integers(0, 3, n)).astype(np.int32)
    iters = rng.integers(1, 20, n).astype(np.int32)
    vd, sd, it = _dev(v, status, iters)
    out = engine.stats_reduce(vd, sd, it, i0=1000).cpu().numpy()
    ok = np.isfinite(v)
    assert abs(out[0] - v[ok].astype(np.float64).sum()) < 1e-9 * n
    assert out[1] == v[ok].min() and out[2] == v[ok].max() and out[3] == 1
    assert out[4] == (status == 0).sum() and out[5] == iters.sum() and out[7] == n
    chk = (v[ok].astype(np.float64) * (((1000 + np.arange(n))[ok] % 251) + 1)).sum()
    assert abs(out[6] - chk) < 1e-7 * n


def test_ekf_tma_staged_variant_is_bitwise_the_direct_kernel(engine, tmp_path):
    """CRB_EKF_VARIANT=4 selects the cp.async.bulk + mbarrier pipelined kernel (same ekf_step code): the
    results must be bit-identical to the default kernel.  The variant is latched per process, so the
    staged kernel runs in a child process."""
    import subprocess
    import sys
    import torch
    n = 300_004          # many tiles per CTA, ragged last tile (multiple of 4)
    x, P, z, u = synth.ekf_inputs(n)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud)
    torch.cuda.synchronize()
    code = ("import sys, numpy as np, torch; sys.path.insert(0, %r)\n"
            "from cpprobotics_b200 import Engine, synth\n"
            "x, P, z, u = synth.ekf_inputs(%d)\n"
            "e = Engine(0); t = [torch.from_numpy(a).cuda() for a in (x, P, z, u)]\n"
            "e.ekf_estimation(*t); torch.cuda.synchronize()\n"
            "np.savez(%r, x=t[0].cpu().numpy(), P=t[1].cpu().numpy())\n") % (
                os.path.dirname(os.path.dirname(os.path.abspath(__file__))), n, str(tmp_path / "o.npz"))
    env = dict(os.environ, CRB_EKF_VARIANT="4")
    subprocess.check_call([sys.executable, "-c", code], env=env)
    o = np.load(tmp_path / "o.npz")
    assert np.array_equal(o["x"], xd.cpu().numpy()) and np.array_equal(o["P"], Pd.cpu().numpy())


def test_closed_loop_on_device_matches_oracle_step_by_step(engine):
    """mpc_simulation's loop body (:372-376) entirely on the device: calc_ref_trajectory -> mpc_solve ->
    update, several steps without a host round trip.  Each step is checked against the oracle fed with
    the GPU's own state (update() goes through libm, so states drift apart by ulps otherwise): index work
    and the solve bit-exact, the plant step to 1e-5."""
    import torch
    n, T, steps = 2000, 20, 6
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, seed=21, course=course)
    cd = _dev(*course)
    state = _dev(st)[0]
    tind = torch.from_numpy(pind.copy()).cuda()
    xref = torch.empty((4 * T, n), dtype=torch.float32, device="cuda")
    u0 = torch.empty((2, n), dtype=torch.float32, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    prm = _params()
    for k in range(steps):
        s_in, t_in = state.cpu().numpy().copy(), tind.cpu().numpy().copy()
        engine.calc_ref_trajectory(state, *cd, 1.0, tind, xref, T)
        engine.mpc_solve(state, xref, T, prm, u0=u0, status=status)
        engine.mpc_plant_update(state, u0)
        torch.cuda.synchronize()
        xr_o, t_o = synth.mpc_xref_numpy(s_in, t_in, T, course=course)
        assert np.array_equal(t_o, tind.cpu().numpy()) and np.array_equal(xr_o, xref.cpu().numpy())
        ro = O.mpc_solve_batched(s_in, xr_o, T)
        assert np.array_equal(ro["u0"], u0.cpu().numpy()) and np.array_equal(ro["status"], status.cpu().numpy())
        s_o = np.stack([O.plant_update(s_in[:, i], ro["u0"][0, i], ro["u0"][1, i]) for i in range(0, n, 20)], axis=1)
        assert np.abs(state.cpu().numpy()[:, ::20] - s_o).max() <= 1e-5 * np.abs(s_o).max()
    # the fleet actually drives: mean speed moved towards the 10/3.6 m/s reference, indices advanced
    assert (tind.cpu().numpy() >= pind).all() and (tind.cpu().numpy() > pind).mean() > 0.5


def test_pf_resample_matches_oracle(engine):
    """resampling() (:120-148), batched statement: index work (which particle survives where) bit-exact."""
    import torch
    n = 200_003
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pwn = O.pf_estimate(pxo, pwo)[0]
    rng = np.random.default_rng(4)
    u = (1.0 + rng.random(n)).astype(np.float32)
    pxd, pwd, ud = _dev(pxo, pwn, u)
    did, neff = engine.pf_resample(pxd, pwd, uniforms=ud)
    torch.cuda.synchronize()
    px2, pw2, did_o, neff_o = O.pf_resample(pxo, pwn, u.astype(np.float64))
    assert did and did_o and abs(neff - neff_o) <= 1e-6 * neff_o
    assert np.array_equal(pxd.cpu().numpy(), px2) and np.array_equal(pwd.cpu().numpy(), pw2)
    # Philox mode draws the same uniforms as the oracle's generator
    pxd, pwd = _dev(pxo, pwn)
    engine.pf_resample(pxd, pwd, uniforms=None, seed=77)
    torch.cuda.synchronize()
    up = np.array([O.philox_uniform12(77, j) for j in range(0, n, 1)])
    px3, _, _, _ = O.pf_resample(pxo, pwn, up)
    assert np.array_equal(pxd.cpu().numpy(), px3)
    # flat weights: Neff = n >= n/2 -> untouched
    pxd, pwd = _dev(px, pw)
    did, neff = engine.pf_resample(pxd, pwd, uniforms=None)
    assert not did and abs(neff - n) < 1e-3 * n and np.array_equal(pxd.cpu().numpy(), px)


@pytest.mark.parametrize("nx,nu,n", [(4, 1, 1), (4, 1, 50_001), (5, 2, 20_003)])
def test_dlqr_bit_exact_vs_oracle(engine, nx, nu, n):
    """solve_DARE + dlqr (row f-4): no transcendental, so the GPU must match the oracle bit for bit,
    iteration counts included."""
    import torch
    A, B, Q, R = synth.lqr_inputs(n, nx)
    Ad, Bd, Qd, Rd = _dev(A, B, Q, R)
    X = torch.empty((nx * nx, n), dtype=torch.float32, device="cuda")
    it = torch.empty(n, dtype=torch.int32, device="cuda")
    K = engine.dlqr(Ad, Bd, Qd, Rd, nx, nu, X=X, iters=it)
    torch.cuda.synchronize()
    r = O.dlqr_batched(A, B, Q, R, nx, nu)
    assert np.array_equal(it.cpu().numpy(), r["iters"])
    assert np.array_equal(K.cpu().numpy(), r["K"]) and np.array_equal(X.cpu().numpy(), r["X"])


# ---- *_host entries on pinned, device-mapped buffers (zero-copy path) ---------------------------------------
def _pin(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


def test_host_entries_on_pinned_buffers_match_the_staged_pipeline_bitwise(engine):
    """The *_host entries launch the resident kernels straight on pinned + mapped host memory (EKF, PF) or
    let the solver store its results there (MPC); pageable numpy arrays take the staged pipeline.  Both
    must give the same bits, including a ragged tail and odd leading dimensions."""
    import torch
    l0 = engine.launches
    n = 300_001
    x, P, z, u = synth.ekf_inputs(n, n_steps=2)
    xs, Ps = x.copy(), P.copy()
    engine.ekf_estimation_host(xs, Ps, z, u, n_steps=2)                 # pageable -> staged
    staged_launches = engine.launches - l0
    xp, Pp, zp, up = _pin(x), _pin(P), _pin(z), _pin(u)
    l0 = engine.launches
    engine.ekf_estimation_host(xp, Pp, zp, up, n_steps=2)               # pinned -> one direct launch
    assert engine.launches - l0 == 1 and staged_launches >= 3
    assert np.array_equal(xp.numpy(), xs) and np.array_equal(Pp.numpy(), Ps)

    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxs, pws = px.copy(), pw.copy()
    engine.pf_predict_weight_host(pxs, pws, noise, lm)
    pxp, pwp, nop = _pin(px), _pin(pw), _pin(noise)
    l0 = engine.launches
    engine.pf_predict_weight_host(pxp, pwp, nop, lm)
    assert engine.launches - l0 == 1                # odd leading dimension -> the scalar kernel, one launch
    assert np.array_equal(pxp.numpy(), pxs) and np.array_equal(pwp.numpy(), pws)
    # Philox mode (no noise array) through the same path
    pxs2, pws2 = px.copy(), pw.copy()
    engine.pf_predict_weight_host(pxs2, pws2, None, lm, seed=99)
    pxp2, pwp2 = _pin(px), _pin(pw)
    engine.pf_predict_weight_host(pxp2, pwp2, None, lm, seed=99)
    assert np.array_equal(pxp2.numpy(), pxs2) and np.array_equal(pwp2.numpy(), pws2)

    m, T = 70_001, 20
    st, xref = _mpc_case(m, T)
    prm = _params(max_iter=50, du_th=1e-4, max_ls=8)
    a = _mpc_gpu(engine, st, xref, T, prm, host=True)                   # pageable outputs -> D2H copies
    nsol = 4 * T + 2 * (T - 1)
    out = dict(sol=torch.empty((nsol, m), dtype=torch.float32).pin_memory(),
               u0=torch.empty((2, m), dtype=torch.float32).pin_memory(),
               cost=torch.empty(m, dtype=torch.float32).pin_memory(),
               status=torch.empty(m, dtype=torch.int32).pin_memory(),
               iters=torch.empty(m, dtype=torch.int32).pin_memory())
    engine.mpc_solve_host(_pin(st), _pin(xref), T, prm, **out)          # kernel stores into pinned memory
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(a[k], out[k].numpy()), k


def test_host_zero_copy_can_be_switched_off(tmp_path):
    """CRB_HOST_ZEROCOPY=0 forces the staged pipeline even for pinned buffers (fresh process: the switch
    is read once)."""
    import subprocess
    import sys
    code = (
        "import numpy as np, torch\n"
        "from cpprobotics_b200 import synth\n"
        "from cpprobotics_b200.engine import Engine\n"
        "e = Engine(); n = 300001\n"
        "x, P, z, u = (torch.from_numpy(a).pin_memory() for a in synth.ekf_inputs(n))\n"
        "l0 = e.launches; e.ekf_estimation_host(x, P, z, u); print('LAUNCHES', e.launches - l0)\n"
        "print('SUM', float(x.double().sum()))\n")
    res = {}
    for flag in ("0", "1"):
        env = dict(os.environ, CRB_HOST_ZEROCOPY=flag,
                   PYTHONPATH=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        res[flag] = dict(l.split() for l in r.stdout.strip().splitlines() if l.split()[0] in ("LAUNCHES", "SUM"))
    assert int(res["1"]["LAUNCHES"]) == 1 and int(res["0"]["LAUNCHES"]) == 3
    assert res["0"]["SUM"] == res["1"]["SUM"]


# ---- BASELINE.json full sizes ----------------------------------------------------------------------------
def test_full_size_ekf_2pow20_matches_oracle_and_is_shard_invariant(engine):
    """configs[1] at full size: every agent against the oracle (field-normalised 1e-5), and the same bits
    whether the batch runs as one launch or as two shards with an odd split (what a 2-GPU run does)."""
    import torch
    n = 1 << 20
    x, P, z, u = synth.ekf_inputs(n)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud)
    torch.cuda.synchronize()
    xo, Po = O.ekf_step_batched(x, P, z, u)
    assert field_err(xd.cpu().numpy(), xo) <= 1e-5 and field_err(Pd.cpu().numpy(), Po) <= 1e-5
    same = (xd.cpu().numpy() == xo).all(axis=0) & (Pd.cpu().numpy() == Po).all(axis=0)
    assert (~same).sum() <= 8, int((~same).sum())      # bit-identical but for glibc-FMA rounding cases (2e-8 / call)
    k = 524_289
    parts = []
    for sl in (slice(0, k), slice(k, n)):
        a = _dev(*(np.ascontiguousarray(t[:, sl]) for t in (x, P, z, u)))
        engine.ekf_estimation(*a)
        torch.cuda.synchronize()
        parts.append((a[0].cpu().numpy(), a[1].cpu().numpy()))
    assert np.array_equal(np.concatenate([p[0] for p in parts], axis=1), xd.cpu().numpy())
    assert np.array_equal(np.concatenate([p[1] for p in parts], axis=1), Pd.cpu().numpy())


def test_full_size_pf_2pow20_matches_oracle_and_is_shard_invariant(engine):
    """configs[2] at full size (2^20 particles, 8 landmarks): positions and weights against the oracle, same
    bits in two shards (even split: packed kernel; the shards' Philox/noise indices are absolute)."""
    import torch
    n = 1 << 20
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = _dev(px, pw, noise)
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    _assert_pf_parity(pxd.cpu().numpy(), pwd.cpu().numpy(), pxo, pwo, lm)   # per-particle 1e-5 on w at 2^20
    k = 1 << 19
    outs = []
    for sl in (slice(0, k), slice(k, n)):
        a = _dev(np.ascontiguousarray(px[:, sl]), np.ascontiguousarray(pw[sl]), np.ascontiguousarray(noise[:, sl]))
        engine.pf_predict_weight(a[0], a[1], a[2], lm)
        torch.cuda.synchronize()
        outs.append((a[0].cpu().numpy(), a[1].cpu().numpy()))
    assert np.array_equal(np.concatenate([o[0] for o in outs], axis=1), pxd.cpu().numpy())
    assert np.array_equal(np.concatenate([o[1] for o in outs]), pwd.cpu().numpy())
    # the normalised weights still sum to one and the estimate is finite (size-independent property)
    xe, Pe, sw = engine.pf_estimate(pxd, pwd)
    assert np.isfinite(xe).all() and np.isfinite(Pe).all() and abs(float(pwd.double().sum().item()) - 1.0) < 1e-6


def test_full_size_mpc_65536_bit_exact_vs_oracle(engine):
    """configs[3] at full size: all 65 536 problems, every output word identical to the oracle."""
    n, T = 1 << 16, 20
    st, xref = _mpc_case(n, T)
    prm = _params()
    got = _mpc_gpu(engine, st, xref, T, prm)
    want = O.mpc_solve_batched(st, xref, T, O.mpc_params())
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(got[k], want[k]), k
    assert (got["status"] == 0).mean() > 0.999


@pytest.mark.gpu
@pytest.mark.parametrize("n,kind", [(65536, "iters"), (65536, "random"), (5000, "constant"), (40_000, "one_long"),
                                    (70_001, "negative_and_huge")])
def test_mpc_hinted_order_gives_the_same_bits(engine, n, kind):
    """crb_mpc_solve_batched_hinted changes the order in which problems start (largest hints first, four passes over
    the index space) and nothing else: every output word equals the un-hinted solve for any hint array, including
    useless ones.  Outputs are pre-filled with a pattern, so a skipped problem would show."""
    import torch
    T = 20
    st, xref = _mpc_case(n, T)
    prm = _params()
    want = _mpc_gpu(engine, st, xref, T, prm)
    rng = np.random.default_rng(3)
    hint = {"iters": want["iters"], "random": rng.integers(0, 40, n), "constant": np.full(n, 7),
            "one_long": np.where(np.arange(n) == n // 2, 50, 3),
            "negative_and_huge": rng.integers(-5, 10_000, n)}[kind].astype(np.int32)
    std, xrd, hd = _dev(st, xref, hint)
    nsol = 4 * T + 2 * (T - 1)
    out = dict(sol=torch.full((nsol, n), float("nan"), dtype=torch.float32, device="cuda"),
               u0=torch.full((2, n), float("nan"), dtype=torch.float32, device="cuda"),
               cost=torch.full((n,), float("nan"), dtype=torch.float32, device="cuda"),
               status=torch.full((n,), -7, dtype=torch.int32, device="cuda"),
               iters=torch.full((n,), -7, dtype=torch.int32, device="cuda"))
    engine.mpc_solve_hinted(std, xrd, T, hd, prm, **out)
    torch.cuda.synchronize()
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(out[k].cpu().numpy(), want[k], equal_nan=True), k
    with pytest.raises(Exception):     # the hint is read while iters is written: aliasing is refused
        engine.mpc_solve_hinted(std, xrd, T, out["iters"], prm, iters=out["iters"])


def test_full_size_resample_properties_2pow20(engine):
    """Size-independent properties of resampling() at 2^20 particles (no oracle needed): the surviving source
    indices are non-decreasing in j (both resampleid and the cumulative weights are monotone), every output
    particle is a copy of an input particle, particle i survives within +-2 of n*w_i times (systematic
    resampling with one jittered draw per slot), and the weights come back uniform."""
    import torch
    n = 1 << 20
    rng = np.random.default_rng(11)
    w = rng.gamma(0.3, 1.0, n).astype(np.float64)            # heavy-tailed weights
    w[rng.integers(0, n, n // 4)] = 0.0                      # a quarter of the particles are dead
    w = (w / w.sum()).astype(np.float32)
    px = np.stack([np.arange(n, dtype=np.float32),           # field 0 = the particle's own index (exact < 2^24)
                   rng.standard_normal(n).astype(np.float32),
                   rng.standard_normal(n).astype(np.float32),
                   rng.standard_normal(n).astype(np.float32)])
    pxd, pwd = _dev(px, w)
    did, neff = engine.pf_resample(pxd, pwd, seed=5, nth=float(n))
    torch.cuda.synchronize()
    assert did
    out = pxd.cpu().numpy()
    src = out[0].astype(np.int64)
    assert (np.diff(src) >= 0).all()
    assert np.array_equal(out[1:], px[1:, src])
    counts = np.bincount(src, minlength=n)
    assert np.abs(counts - n * w.astype(np.float64)).max() <= 2.0 + 1e-3 * n * w.max()
    dead = w == 0
    assert counts[:-1][dead[:-1]].sum() == 0           # dead particles never survive ...
    assert not dead[-1] or counts[-1] <= 2             # ... except slot NP-1 catching the reference's cap (:139)
    assert np.array_equal(pwd.cpu().numpy(), np.full(n, np.float32(1.0 / n)))


def test_ekf_n_steps_is_the_composition_of_single_steps_bitwise(engine):
    """n_steps = k in one launch (state kept in registers) must equal k launches of one step, bit for bit,
    at the full 2^20-agent size."""
    import torch
    n, k = 1 << 20, 5
    x, P, z, u = synth.ekf_inputs(n, n_steps=k)
    a = _dev(x, P, z, u)
    engine.ekf_estimation(*a, n_steps=k)
    xb, Pb = _dev(x, P)
    for s in range(k):
        zs, us = _dev(z[2 * s:2 * s + 2], u[2 * s:2 * s + 2])
        engine.ekf_estimation(xb, Pb, zs, us)
    torch.cuda.synchronize()
    assert torch.equal(a[0], xb) and torch.equal(a[1], Pb)


# ---- the CUDA path against outputs of the reference's own source text (tests/golden/ref_golden.npz) ------------
def test_cuda_path_against_reference_text_outputs(engine):
    """No oracle in between: EKF within the float tolerance (CUDA vs glibc sinf/cosf), DARE/LQR gains and the
    reference-trajectory index work bit for bit, the plant update to 1e-5."""
    import torch
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_golden.npz"))
    xd, Pd, zd, ud = _dev(G["ekf_x"], G["ekf_P"], G["ekf_z"], G["ekf_u"])
    engine.ekf_estimation(xd, Pd, zd, ud)
    torch.cuda.synchronize()
    assert field_err(xd.cpu().numpy(), G["ekf_x_out"]) <= 1e-5
    assert field_err(Pd.cpu().numpy(), G["ekf_P_out"]) <= 1e-5
    for nx, nu in ((4, 1), (5, 2)):
        Ad, Bd, Qd, Rd = _dev(G[f"lqr{nx}_A"], G[f"lqr{nx}_B"], G[f"lqr{nx}_Q"], G[f"lqr{nx}_R"])
        X = torch.empty((nx * nx, Ad.shape[1]), dtype=torch.float32, device="cuda")
        K = engine.dlqr(Ad, Bd, Qd, Rd, nx, nu, X=X)
        torch.cuda.synchronize()
        assert np.array_equal(K.cpu().numpy(), G[f"lqr{nx}_K"]) and np.array_equal(X.cpu().numpy(), G[f"lqr{nx}_X"])
    T = int(G["crt_T"])
    course = synth.mpc_course()
    std = _dev(G["crt_state"])[0]
    tid = torch.from_numpy(G["crt_pind"].astype(np.int32)).cuda()
    xr = torch.empty((4 * T, std.shape[1]), dtype=torch.float32, device="cuda")
    engine.calc_ref_trajectory(std, *_dev(*course), 1.0, tid, xr, T)
    torch.cuda.synchronize()
    assert np.array_equal(tid.cpu().numpy(), G["crt_tind"]) and np.array_equal(xr.cpu().numpy(), G["crt_xref"])
    sd, u0d = _dev(G["upd_state"], np.stack([G["upd_a"], G["upd_delta"]]))
    engine.mpc_plant_update(sd, u0d)
    torch.cuda.synchronize()
    assert np.abs(sd.cpu().numpy() - G["upd_out"]).max() <= 1e-5 * np.abs(G["upd_out"]).max()


# ---- resident-state EKF tracking (the reference's time loop, :171-183) -------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
def test_ekf_track_matches_the_multi_step_launch_bitwise(engine, pinned):
    """K single steps through crb_ekf_track_step (x, P resident on the device, 16 B in / 16 B out per update)
    must give the bits of ONE launch with n_steps = K on the same observations, synchronous and pipelined."""
    import torch
    n, K = 70_001, 6
    x, P, z, u = synth.ekf_inputs(n, n_steps=K)
    xd, Pd, zd, ud = _dev(x, P, z, u)
    engine.ekf_estimation(xd, Pd, zd, ud, n_steps=K)
    torch.cuda.synchronize()
    want_x, want_P = xd.cpu().numpy(), Pd.cpu().numpy()

    def host(a):
        t = torch.from_numpy(np.ascontiguousarray(a))
        return t.pin_memory() if pinned else t
    for async_ in (False, True):
        trk = engine.ekf_track_open(x, P)
        zs = [host(z[2 * k:2 * k + 2]) for k in range(K)]
        us = [host(u[2 * k:2 * k + 2]) for k in range(K)]
        outs = [host(np.zeros((4, n), np.float32)) for _ in range(K)]
        for k in range(K):
            engine.ekf_track_step(trk, zs[k], us[k], x_out=outs[k], async_=async_)
        engine.ekf_track_sync(trk)
        gx, gP = np.empty_like(x), np.empty_like(P)
        engine.ekf_track_read(trk, gx, gP)
        engine.ekf_track_close(trk)
        assert np.array_equal(gx, want_x) and np.array_equal(gP, want_P)
        assert np.array_equal(outs[-1].numpy(), want_x)
        # every intermediate x is what a (k+1)-step launch gives
        xk, Pk = _dev(x, P)
        engine.ekf_estimation(xk, Pk, _dev(z[:6])[0], _dev(u[:6])[0], n_steps=3)
        torch.cuda.synchronize()
        assert np.array_equal(outs[2].numpy(), xk.cpu().numpy())


# ---- one complete PF iteration on the device (crb_pf_step) ------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [300_001, 1_000_000])
def test_pf_step_is_the_composition_of_the_reference_stages(engine, n):
    """predict+weight (:81-102) -> normalise, estimate, covariance (:104-107) -> Neff, resampling (:120-148) in ONE
    call without a host round trip, against the oracle's stages.  n = 10^6 is not a power of two: j/NP is then
    inexact in binary32 and adjacent resampleids can be inverted; the reference's monotone search index makes
    that a running maximum, which the gather kernel reproduces (round 1 did not)."""
    import torch
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    rng = np.random.default_rng(4)
    u = (1.0 + rng.random(n)).astype(np.float32)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pwn, xeo, Peo, swo = O.pf_estimate(pxo, pwo)
    # (a) nth = 0: never resample -> px_next is a copy, pw the normalised weights
    pxd, pwd, nd, ud = _dev(px, pw, noise, u)
    nxt = torch.empty_like(pxd)
    res = engine.pf_step(pxd, pwd, nxt, nd, lm, uniforms=ud, nth=0.0)
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    gx, gw = pxd.cpu().numpy(), pwd.cpu().numpy()
    assert r[22] == 0.0 and np.array_equal(nxt.cpu().numpy(), gx)
    assert (gx == pxo).all(axis=0).mean() > 1 - 1e-5
    np.testing.assert_allclose(gw, pwn, rtol=2e-5, atol=1e-30)
    assert abs(r[20] - swo) <= 1e-5 * abs(swo)
    np.testing.assert_allclose(r[0:4], xeo, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(r[4:20].reshape(4, 4).T, Peo, rtol=1e-4, atol=1e-6)
    neff_o = 1.0 / float(np.float32(np.sum(gw.astype(np.float64) ** 2)))
    assert abs(r[21] - neff_o) <= 1e-5 * neff_o
    # (b) nth = n: always resample -> the index work is bit-exact against the oracle run on the GPU's own weights
    pxd2, pwd2 = _dev(px, pw)
    nxt2 = torch.empty_like(pxd2)
    res2 = engine.pf_step(pxd2, pwd2, nxt2, nd, lm, uniforms=ud, nth=float(n))
    torch.cuda.synchronize()
    px2, pw2, did_o, _ = O.pf_resample(gx, gw, u.astype(np.float64), nth=float(n))
    assert res2.cpu().numpy()[22] == 1.0 and did_o
    assert np.array_equal(nxt2.cpu().numpy(), px2) and np.array_equal(pwd2.cpu().numpy(), pw2)
    # the stand-alone entry gives the same particles (its cumulative weights are materialised, not fused)
    pxd3, pwd3 = _dev(gx, gw)
    engine.pf_resample(pxd3, pwd3, uniforms=ud, nth=float(n))
    torch.cuda.synchronize()
    assert np.array_equal(pxd3.cpu().numpy(), px2)


def _pf_inputs_at(n, centre):
    """synth.pf_inputs and its landmarks; with a centre, moved rigidly there and shrunk to a 5 cm cloud."""
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    if centre is not None:
        lm = lm.astype(np.float64)
        for f in (0, 1):
            px[f] = (centre[f] + (px[f].astype(np.float64) - synth.PF_TRUTH[f]) * 0.25).astype(np.float32)
            lm[:, 1 + f] += centre[f] - synth.PF_TRUTH[f]
        lm = lm.astype(np.float32)
    return px, pw, noise, lm


def _pf_shard_worker(rank, world, port, n, q, centre=None):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from cpprobotics_b200 import Engine, _lib as L
    eng = Engine(rank)
    buf = torch.zeros(L.CRB_COMM_ID_BYTES, dtype=torch.uint8, device="cuda")
    if rank == 0:
        buf.copy_(torch.frombuffer(bytearray(eng.comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(buf, 0)
    eng.comm_init(world, rank, bytes(buf.cpu().numpy().tobytes()))
    px, pw, noise, lm = _pf_inputs_at(n, centre)
    k = n // world
    sl = slice(rank * k, (rank + 1) * k)
    pxd, pwd, nd = (torch.from_numpy(np.ascontiguousarray(a[..., sl])).cuda() for a in (px, pw, noise))
    # index-addressed noise: shard r applies the noise of particles [r k, (r+1) k)
    nxt = torch.empty_like(pxd)
    res = eng.pf_step(pxd, pwd, nxt, nd, lm, nth=0.0)
    torch.cuda.synchronize()
    q.put((rank, res.cpu().numpy().copy(), pwd.cpu().numpy().copy()))
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_pf_sharded_over_two_gpus_equals_the_single_gpu_estimate(engine):
    """SURVEY f-2: pw / pw.sum() (:104) across shards is one small all-reduce inside libcrb; every rank must get the
    single-GPU estimate and globally normalised weights.  NCCL takes one rank per GPU, so on a machine with a single
    GPU the batch is ONE shard behind a one-rank communicator: the same sharded code path (partials, all-reduce,
    finalize) against the unsharded one."""
    import socket
    import torch
    import torch.multiprocessing as mp
    n, world = 400_000, min(2, torch.cuda.device_count())
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = _dev(px, pw, noise)
    nxt = torch.empty_like(pxd)
    want = engine.pf_step(pxd, pwd, nxt, nd, lm, nth=0.0).cpu().numpy()
    want_w = pwd.cpu().numpy()
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_pf_shard_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = sorted([q.get(timeout=240) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, w in got:
        # the same sums in another association: the sharded form divides sum(w x) by sum(w), the single-GPU form sums
        # the normalised weights; narrowed to the reference's float they may differ by one float ulp (xEst) and by
        # the cancellation in the covariance
        np.testing.assert_allclose(res[0:4], want[0:4], rtol=2e-7, atol=1e-7)
        np.testing.assert_allclose(res[4:20], want[4:20], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(res[20], want[20], rtol=1e-9)
        k = n // world
        np.testing.assert_allclose(w, want_w[rank * k:(rank + 1) * k], rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_pf_sharded_covariance_far_from_the_origin(engine):
    """The sharded moments are centred on rank 0's particle 0, broadcast to every rank: a 5 cm cloud 10^5 m from the
    origin keeps PEst at float accuracy, entry by entry within 1e-6 sqrt(P_rr P_cc) of the float64 two-pass
    covariance around the single-GPU xEst, and xEst within one float ulp of the single-GPU one."""
    import socket
    import torch
    import torch.multiprocessing as mp
    n, world, centre = 400_000, min(2, torch.cuda.device_count()), (1e5, 1e5)
    px, pw, noise, lm = _pf_inputs_at(n, centre)
    pxd, pwd, nd = _dev(px, pw, noise)
    nxt = torch.empty_like(pxd)
    want = engine.pf_step(pxd, pwd, nxt, nd, lm, nth=0.0).cpu().numpy()
    gx = pxd.cpu().numpy()
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_pf_shard_worker, args=(r, world, port, n, q, centre)) for r in range(world)]
    for p in procs:
        p.start()
    got = sorted([q.get(timeout=240) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    gw = np.concatenate([w for _, _, w in got]).astype(np.float64)   # the globally normalised weights
    for rank, res, w in got:
        assert (np.abs(res[0:4] - want[0:4]) <= np.spacing(np.abs(want[0:4]).astype(np.float32))).all()
        d = (gx - res[0:4].astype(np.float32)[:, None]).astype(np.float64)   # around this rank's xEst
        C = (d * gw) @ d.T
        P = res[4:20].reshape(4, 4).T
        assert np.array_equal(P, P.T)
        err = np.abs(P - C) / np.sqrt(np.outer(np.diag(C), np.diag(C)))
        assert err.max() <= 1e-6, err.max()
