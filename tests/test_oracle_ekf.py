"""CPU: the EKF restatement (oracle/crb_oracle.c) against hand-derived known answers, an independent
float64 numpy statement of src/extended_kalman_filter.cpp:22-78, and the committed golden vectors."""
import os

import numpy as np
import pytest

from cpprobotics_b200 import synth
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def ekf_numpy_f64(x, P, z, u, Q, R, dt=0.1):
    """Independent statement with numpy matrices (row/column conventions of the reference text)."""
    def motion_model(x, u):
        F = np.eye(4)
        B = np.array([[dt * np.cos(x[2]), 0], [dt * np.sin(x[2]), 0], [0, dt], [1.0, 0]])
        return F @ x + B @ u

    def jacobF(x, u):
        jF = np.eye(4)
        yaw, v = x[2], u[0]
        jF[0, 2] = -dt * v * np.sin(yaw); jF[0, 3] = dt * np.cos(yaw)
        jF[1, 2] = dt * v * np.cos(yaw); jF[1, 3] = dt * np.sin(yaw)
        return jF
    H = np.array([[1.0, 0, 0, 0], [0, 1.0, 0, 0]])
    xp = motion_model(x, u)
    jF = jacobF(xp, u)
    PP = jF @ P @ jF.T + Q
    y = z - H @ xp
    S = H @ PP @ H.T + R
    K = PP @ H.T @ np.linalg.inv(S)
    return xp + K @ y, (np.eye(4) - K @ H) @ PP


def test_known_answer_from_main_constants():
    """xEst=0, PEst=I, u=(1,0.1), z=(0.1,0) with Q,R of main() :139-151 (SURVEY Appendix A.1)."""
    x, P = O.ekf_estimation(np.zeros(4), np.eye(4).reshape(-1), [0.1, 0.0], [1.0, 0.1])
    np.testing.assert_allclose(x, [0.1, 0.0, 0.010000001, 1.0], rtol=0, atol=1e-8)
    Pm = P.reshape(4, 4).T
    want = np.array([[0.50495052, 0, -4.9504131e-04, 4.9502481e-02],
                     [0, 0.50495052, 4.9502481e-02, 4.9504131e-04],
                     [-4.9504125e-04, 4.9502477e-02, 0.99535406, 0],
                     [4.9502477e-02, 4.9504125e-04, 0, 1.0050495]])
    np.testing.assert_allclose(Pm, want, rtol=2e-7, atol=1e-10)
    # hand derivation of the easy entries: xPred = (0.1, 0, 0.01, 1); S = P00+Q00+R = 2.02 -> K00 = 1.02/2.02
    assert abs(Pm[0, 0] - (1.0 - 1.02 / 2.02) * 1.02) < 5e-7


def test_f32_matches_independent_f64_numpy():
    n = 500
    x, P, z, u = synth.ekf_inputs(n)
    dt, Q, R = O.ekf_constants()
    xo, Po = O.ekf_step_batched(x, P, z, u)
    Qm, Rm = Q.reshape(4, 4).T.astype(float), R.reshape(2, 2).T.astype(float)
    for i in range(n):
        xe, Pe = ekf_numpy_f64(x[:, i].astype(float), P[:, i].reshape(4, 4).T.astype(float),
                               z[:, i].astype(float), u[:, i].astype(float), Qm, Rm, dt)
        assert np.abs(xo[:, i] - xe).max() <= 1e-5 * np.abs(xe).max()
        assert np.abs(Po[:, i].reshape(4, 4).T - Pe).max() <= 1e-5 * np.abs(Pe).max()


def test_c_f64_variant_agrees_with_numpy():
    x, P, z, u = synth.ekf_inputs(16)
    dt, Q, R = O.ekf_constants()
    for i in range(16):
        xa, Pa = O.ekf_estimation_f64(x[:, i], P[:, i], z[:, i], u[:, i])
        xe, Pe = ekf_numpy_f64(x[:, i].astype(float), P[:, i].reshape(4, 4).T.astype(float),
                               z[:, i].astype(float), u[:, i].astype(float),
                               Q.reshape(4, 4).T.astype(float), R.reshape(2, 2).T.astype(float), dt)
        np.testing.assert_allclose(xa, xe, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(Pa.reshape(4, 4).T, Pe, rtol=1e-10, atol=1e-12)


def test_summation_order_option_stays_within_tolerance():
    """Eigen's inner-product order is unpinned (SURVEY §7.3): sequential vs pairwise must agree to the
    field-normalised 1e-5 gate (they differ only in jF*P*jF^T)."""
    x, P, z, u = synth.ekf_inputs(2000)
    xa, Pa = O.ekf_step_batched(x, P, z, u, order=O.ORDER_SEQ)
    xb, Pb = O.ekf_step_batched(x, P, z, u, order=O.ORDER_PAIRWISE)
    assert (np.abs(Pa - Pb).max(axis=0) / np.abs(Pa).max(axis=0)).max() < 1e-6
    assert np.array_equal(xa, xb) or np.abs(xa - xb).max() < 1e-5


def test_config1_single_agent_1000_steps_tracks_f64():
    """BASELINE config 1: one agent, 1000 steps, the reference's main() loop with a fixed seed."""
    rng = np.random.default_rng(12345)
    dt, Q, R = O.ekf_constants()
    u = np.array([1.0, 0.1])
    x32, P32 = np.zeros(4, np.float32), np.eye(4, dtype=np.float32).reshape(-1)
    x64, P64 = np.zeros(4), np.eye(4).reshape(-1)
    xT = np.zeros(4)
    for k in range(1000):
        ud = u + rng.normal(size=2) * np.array([1.0, np.deg2rad(30.0) ** 2])       # :174-175
        xT = np.array([xT[0] + dt * np.cos(xT[2]) * u[0], xT[1] + dt * np.sin(xT[2]) * u[0],
                       xT[2] + dt * u[1], xT[3] + u[0]])
        z = xT[:2] + rng.normal(size=2) * 0.25                                       # :180-181
        x32, P32 = O.ekf_estimation(x32, P32, z.astype(np.float32), ud.astype(np.float32))
        x64, P64 = O.ekf_estimation_f64(x64, P64, z.astype(np.float32), ud.astype(np.float32))
        assert np.isfinite(x32).all() and np.isfinite(P32).all()
    assert np.abs(x32 - x64).max() <= 1e-4 * np.abs(x64).max()       # v accumulates to ~1000
    assert np.abs(P32 - P64).max() <= 1e-3 * np.abs(P64).max()
    Pm = P32.reshape(4, 4).T
    assert np.linalg.eigvalsh(0.5 * (Pm + Pm.T)).min() > -1e-3


def test_batched_driver_equals_per_agent_calls_and_multistep():
    n, steps = 37, 3
    x, P, z, u = synth.ekf_inputs(n, n_steps=steps)
    xb, Pb = O.ekf_step_batched(x, P, z, u, n_steps=steps, nthreads=3)
    for i in range(n):
        xi, Pi = x[:, i], P[:, i]
        for s in range(steps):
            xi, Pi = O.ekf_estimation(xi, Pi, z[2 * s:2 * s + 2, i], u[2 * s:2 * s + 2, i])
        assert np.array_equal(xi, xb[:, i]) and np.array_equal(Pi, Pb[:, i])


def test_golden_vectors():
    g = np.load(os.path.join(GOLD, "ekf_golden.npz"))
    xo, Po = O.ekf_step_batched(g["x"], g["P"], g["z"], g["u"], n_steps=int(g["n_steps"]))
    # the fixture was produced by this oracle on x86-64/glibc; sinf/cosf of another libm may differ by ulps
    assert (np.abs(xo - g["x_out"]).max(axis=0) / np.abs(g["x_out"]).max(axis=0)).max() <= 1e-6
    assert (np.abs(Po - g["P_out"]).max(axis=0) / np.abs(g["P_out"]).max(axis=0)).max() <= 1e-6
    # and against the float64 numpy statement stored beside it
    assert (np.abs(xo - g["x_f64"]).max(axis=0) / np.abs(g["x_f64"]).max(axis=0)).max() <= 1e-5
    assert (np.abs(Po - g["P_f64"]).max(axis=0) / np.abs(g["P_f64"]).max(axis=0)).max() <= 1e-5


def test_best_effort_build_is_a_timing_arm_that_stays_close():
    """oracle/lib/liboracle_fast.so (-O3 -march=x86-64-v3 -ffp-contract=fast, bench.py's best_effort_value) is the
    same source: results within the float tolerance of the faithful build, and the switch is reversible."""
    x, P, z, u = synth.ekf_inputs(2000, seed=5)
    xa, Pa = O.ekf_step_batched(x, P, z, u, nthreads=1)
    try:
        if not O.use_library("fast"):
            pytest.skip("fast build or AVX2/FMA not available")
        xb, Pb = O.ekf_step_batched(x, P, z, u, nthreads=1)
    finally:
        O.use_library("faithful")
    xc, Pc = O.ekf_step_batched(x, P, z, u, nthreads=1)
    assert np.array_equal(xa, xc) and np.array_equal(Pa, Pc)
    err = lambda g, w: (np.abs(g - w).max(axis=0) / np.abs(w).max(axis=0)).max()  # noqa: E731
    assert err(xb, xa) <= 1e-5 and err(Pb, Pa) <= 1e-5


def test_restated_glibc_sincosf_carries_this_hosts_libm_bits():
    """The CUDA kernels evaluate sin/cos with glibc's binary64 algorithm (crb_sincosf_libm, crb_common.cuh); its C
    restatement in the oracle is pinned here against the libm of THIS host over ~6e7 arguments in |y| < 120:
    on a host with FMA (where glibc's ifunc selects its -mfma build, which is what is restated) sin and cos are
    identical on every argument; on a host without FMA a few in 1e8 differ by one ulp."""
    import ctypes as C
    from oracle import oracle as O
    L = O.lib()
    L.crb_oracle_libm_sincosf_census.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    L.crb_oracle_libm_sincosf.argtypes = [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    out = np.zeros(2, np.int64)
    L.crb_oracle_libm_sincosf_census(0, 0x42F00000, 37, out.ctypes.data)   # every 37th float in [0, 120), both signs
    n = 2 * (0x42F00000 // 37)
    has_fma = " fma " in open("/proc/cpuinfo").read()
    assert (out == 0).all() if has_fma else (out[0] <= 2e-7 * n and out[1] <= 2e-7 * n), out
    # the workloads' range, densely: yaw in [-pi - 1, pi + 1]
    lo = np.float32(0.5).view(np.uint32)
    hi = np.float32(4.2).view(np.uint32)
    L.crb_oracle_libm_sincosf_census(int(lo), int(hi), 1, out.ctypes.data)
    assert out[0] <= 4 and out[1] <= 4, out
    s, c = C.c_float(), C.c_float()
    for y, ws, wc in [(0.0, 0.0, 1.0), (1e-5, 1e-5, 1.0), (np.inf, np.nan, np.nan), (-np.inf, np.nan, np.nan),
                      (np.nan, np.nan, np.nan)]:
        L.crb_oracle_libm_sincosf(C.c_float(y), C.byref(s), C.byref(c))
        assert (np.isnan(s.value) and np.isnan(ws)) or s.value == np.float32(ws)
        assert (np.isnan(c.value) and np.isnan(wc)) or c.value == np.float32(wc)


def test_restated_sincosf_beyond_120_is_this_hosts_libm_on_every_float():
    """From |y| = 120 on, glibc reduces with reduce_large (integer products with a window of 2/pi) instead of the
    binary64 multiply-subtract; the restatement does the same, and must give this host's sinf and cosf on every one
    of the 2,032,140,288 finite floats with |y| >= 120, both signs (about 5 s on 8 threads).  On a host without FMA,
    glibc's plain build of the shared polynomial differs by an ulp on a few arguments in 1e8."""
    import ctypes as C
    L = O.lib()
    L.crb_oracle_libm_sincosf_census.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    out = np.zeros(2, np.int64)
    L.crb_oracle_libm_sincosf_census(0x42F00000, 0x7F800000, 1, out.ctypes.data)
    n = 2 * (0x7F800000 - 0x42F00000)
    assert n == 2_032_140_288
    has_fma = " fma " in open("/proc/cpuinfo").read()
    assert (out == 0).all() if has_fma else (out[0] <= 2e-7 * n and out[1] <= 2e-7 * n), out


def _two_over_pi_words():
    """glibc's __inv_pio4 from first principles: pi by Machin's formula in integers, then word k = the bits
    [8k - 24, 8k + 8) of the binary fraction of 2/pi."""
    prec = 320                                   # bits; the words need 200
    one = 1 << (prec + 16)

    def arctan_inv(q):                           # arctan(1/q) * one
        s, t, k, sign = 0, one // q, 1, 1
        while t:
            s += sign * (t // k)
            t //= q * q
            k += 2
            sign = -sign
        return s
    pi = 16 * arctan_inv(5) - 4 * arctan_inv(239)   # pi * one, good to ~prec bits
    frac = (2 * one << prec) // pi                  # 2/pi * 2^prec
    return [(frac >> (prec - 8 * (k + 1))) & 0xFFFFFFFF for k in range(24)]


def test_reduce_large_table_is_two_over_pi():
    """The 2/pi words of the restated reduce_large, in the checker and in the kernels' header, regenerated here."""
    import ctypes as C
    import re
    want = _two_over_pi_words()
    assert want[:6] == [0xa2, 0xa2f9, 0xa2f983, 0xa2f9836e, 0xf9836e4e, 0x836e4e44]
    assert list((C.c_uint32 * 24).in_dll(O.lib(), "crb_oracle_inv_pio4")) == want
    src = open(os.path.join(os.path.dirname(GOLD), "..", "cpprobotics_b200", "csrc", "crb_common.cuh")).read()
    body = re.search(r"crb_inv_pio4\[24\] = \{([^}]*)\}", src).group(1)
    assert [int(w, 16) for w in re.findall(r"0x[0-9a-f]+", body)] == want
