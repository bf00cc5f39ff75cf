"""CPU: particle-filter restatement against known answers, an independent numpy statement of
src/particle_filter.cpp:26-57,81-107, Philox known-answer vectors, and the arithmetic identities the
CUDA kernel relies on."""
import ctypes as C
import os

import numpy as np

from cpprobotics_b200 import synth
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_gauss_likelihood_known_values():
    # gauss_likelihood(0, 0.1) = 1/sqrt(2*3.141592653*0.01)  (SURVEY §8 c-6); PI is the truncated literal
    s = float(np.sqrt(np.float32(0.01)))
    assert abs(O.gauss_likelihood(0.0, s) - 1.0 / np.sqrt(2 * 3.141592653 * s * s)) < 3e-7
    # one sigma out: factor exp(-1/2)
    assert abs(O.gauss_likelihood(s, s) / O.gauss_likelihood(0.0, s) - np.exp(-0.5)) < 2e-7


def pf_numpy(px, pw, noise, lm, c):
    px = px.astype(np.float64).copy(); pw = pw.astype(np.float64).copy()
    ud0 = c["u"][0] + noise[0].astype(np.float64) * float(c["rsim_diag"][0])
    ud1 = c["u"][1] + noise[1].astype(np.float64) * float(c["rsim_diag"][1])
    ud0, ud1 = ud0.astype(np.float32).astype(np.float64), ud1.astype(np.float32).astype(np.float64)
    yaw = px[2].copy()
    px[0] += c["dt"] * np.cos(yaw) * ud0
    px[1] += c["dt"] * np.sin(yaw) * ud0
    px[2] += c["dt"] * ud1
    px[3] += ud0
    sig = float(np.sqrt(np.float32(c["Q"])))
    for r, lx, ly in lm.astype(np.float64):
        dz = np.hypot(px[0] - lx, px[1] - ly) - r
        pw *= 1.0 / np.sqrt(2.0 * c["pi"] * sig * sig) * np.exp(-dz * dz / (2 * sig * sig))
    return px, pw


def test_matches_independent_numpy():
    n = 4000
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pxe, pwe = pf_numpy(px, pw, noise, lm, O.pf_constants())
    assert np.abs(pxo - pxe).max() < 5e-6
    # the weight is conditioned like sum|dz|/sigma^2 times the float32 position rounding (see the GPU test)
    ok = pwe > 1e-30
    rel = np.abs(pwo[ok] - pwe[ok]) / pwe[ok]
    assert np.median(rel) < 1e-4 and rel.max() < 5e-3


def test_philox_known_answer_vectors():
    """Random123 kat_vectors for philox4x32-10."""
    L = O.lib()
    u32 = C.c_uint32 * 4
    k32 = C.c_uint32 * 2
    L.crb_oracle_philox4x32.argtypes = [u32, k32, u32]
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdccceb & 0xffffffff, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases[:2]:
        out = u32()
        L.crb_oracle_philox4x32(u32(*ctr), k32(*key), out)
        assert tuple(out) == want
    out = u32()
    L.crb_oracle_philox4x32(u32(*cases[2][0]), k32(*cases[2][1]), out)
    assert out[0] == 0xd16cfe09 and out[2] == 0x5001e420 and out[3] == 0x24126ea1


def test_philox_normals_are_standard_normal():
    g = np.array([O.philox_normal2(42, i) for i in range(20000)])
    assert abs(g.mean()) < 0.02 and abs(g.std() - 1.0) < 0.02
    assert abs(np.corrcoef(g[:, 0], g[:, 1])[0, 1]) < 0.03


def test_noise_none_uses_philox_per_particle_index():
    n = 64
    px, pw, _ = synth.pf_inputs(n)
    lm = synth.pf_landmarks(4)
    a = O.pf_predict_weight_batched(px, pw, None, lm, seed=7)
    noise = np.stack([[O.philox_normal2(7, i)[k] for i in range(n)] for k in (0, 1)]).astype(np.float32)
    b = O.pf_predict_weight_batched(px, pw, noise, lm)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_kernel_arithmetic_identities():
    """The CUDA kernel replaces x / (2 sigma^2) by an FMA sequence and the double-precision prefactor
    product by a float-float product; both must be value-identical (exhaustive over the relevant range)."""
    L = O.lib()
    L.crb_oracle_check_const_division.restype = C.c_int64
    L.crb_oracle_check_const_division.argtypes = [C.c_float, C.c_uint32, C.c_uint32]
    L.crb_oracle_check_ff_product.restype = C.c_int64
    L.crb_oracle_check_ff_product.argtypes = [C.c_double, C.c_uint32, C.c_uint32]
    bits = lambda v: int(np.float32(v).view(np.uint32))
    sigma = np.sqrt(np.float32(0.01))
    two_s2 = np.float32(2) * sigma * sigma
    assert L.crb_oracle_check_const_division(float(two_s2), bits(-1e-20), bits(-1e4)) == 0
    pre = 1.0 / np.sqrt(2.0 * 3.141592653 * float(sigma) * float(sigma))
    assert L.crb_oracle_check_ff_product(pre, bits(1e-30), bits(1.0)) == 0


def test_resample_id_reciprocal_is_the_correctly_rounded_quotient():
    """crb_pf_step's gather computes resampleid = (float)(base(j) + U / NP), base(j) = (float)(j / NP), with both
    double quotients as Markstein sequences around r = RN(1 / NP) instead of divisions.  Census: every NP <= 2^21 at
    the edge j and 32 hashed j, every j for five NP, and every Philox U in [1, 2) for those NP - the quotients and the
    float result must be the correctly rounded ones, without exception."""
    L = O.lib()
    L.crb_oracle_check_resample_id_rcp.restype = C.c_int64
    L.crb_oracle_check_resample_id_rcp.argtypes = [C.c_int64, C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int64)]
    ns = (C.c_int64 * 5)(3, 1025, 1_000_000, (1 << 21) - 1, 1 << 21)
    evaluated = C.c_int64(0)
    bad = L.crb_oracle_check_resample_id_rcp(1 << 21, ns, len(ns), C.byref(evaluated))
    assert evaluated.value > 5 * (1 << 23) + (1 << 21) * 38 - 16
    assert bad == 0


def test_estimate_tail_matches_numpy():
    n = 5000
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pwn, xe, Pe, sw = O.pf_estimate(pxo, pwo)
    w = pwo.astype(np.float64) / np.float32(pwo.astype(np.float64).sum())
    np.testing.assert_allclose(pwn, w, rtol=2e-7, atol=1e-38)      # denormal weights round coarsely
    m = (pxo.astype(np.float64) * w).sum(axis=1)
    np.testing.assert_allclose(xe, m, rtol=1e-6, atol=1e-6)
    d = pxo.astype(np.float64) - xe[:, None].astype(np.float64)
    np.testing.assert_allclose(Pe, (d * w) @ d.T, rtol=1e-5, atol=1e-9)


def test_golden_vectors():
    g = np.load(os.path.join(GOLD, "pf_golden.npz"))
    pxo, pwo = O.pf_predict_weight_batched(g["px"], g["pw"], g["noise"], g["lm"])
    assert np.abs(pxo - g["px_out"]).max() <= 1e-6
    ok = g["pw_out"] > 1e-30
    assert (np.abs(pwo[ok] - g["pw_out"][ok]) / g["pw_out"][ok]).max() <= 1e-3   # libm-dependent, see above


def test_resample_batched_mode_properties():
    """The batched statement (double cumulative sum, base = j/n): survivors are existing particles, heavy
    particles are duplicated about n*w times, weights reset to 1/n, nothing happens when Neff >= nth."""
    n = 20000
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8)
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm)
    pwn = O.pf_estimate(pxo, pwo)[0]
    u = np.array([O.philox_uniform12(5, j) for j in range(n)])
    assert u.min() >= 1.0 and u.max() < 2.0
    px2, pw2, did, neff = O.pf_resample(pxo, pwn, u)
    assert did and abs(neff - 1.0 / np.sum(pwn.astype(np.float64) ** 2)) < 1e-3 * neff
    assert np.all(pw2 == np.float32(1.0 / n))
    keys = {tuple(c) for c in pxo.T}
    assert all(tuple(c) in keys for c in px2.T[::97])
    top = int(np.argmax(pwn))
    copies = int((px2.T == pxo[:, top]).all(axis=1).sum())
    assert abs(copies - n * pwn[top]) <= 2
    px3, pw3, did3, _ = O.pf_resample(px, np.full(n, 1.0 / n, np.float32), u)
    assert not did3 and np.array_equal(px3, px)
