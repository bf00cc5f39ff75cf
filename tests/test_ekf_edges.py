"""The EKF step (crb_ekf.cu) away from the reference's constants, at special values, at any yaw and past 2^31 element
offsets, against the oracle (oracle/crb_oracle.c, which calls the host libm's sinf / cosf like the reference).

The oracle and the kernel perform the same binary32 operations in the same order and take sin / cos with the host
libm's bits (crb_sincosf_libm, crb_common.cuh), so unless a test says otherwise every agent must be bit-identical to
the oracle on a host whose glibc uses its FMA build (any x86-64 CPU with FMA); elsewhere a few agents in 1e7 may
differ by an ulp of sin / cos.
  - every entry point (both device kernels, the staged and the zero-copy host entries, the resident track) at seven
    parameter sets besides the defaults, and the float64 statement for the well-conditioned ones;
  - NaN, inf, zero signs, subnormals, overflow and a singular innovation covariance in isolated agents;
  - yaw at the branch edges of sinf / cosf, from 120 on (glibc's reduce_large) up to FLT_MAX, and a 3000-step track
    that turns past |yaw| = 3000;
  - batches whose element offsets pass 2^31;
  - crb_sincosf_libm itself on all 2^32 bit patterns, and the PF and MPC plant kernels at |yaw| >= 120."""
import os
import subprocess

import numpy as np
import pytest

from cpprobotics_b200 import EkfParams, synth
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
FMA_HOST = " fma " in open("/proc/cpuinfo").read()
CHUNK = 131072                                   # the staged host entry's chunk (crb_ekf.cu)


def _sets():
    dt, Q, R = O.ekf_constants()
    Qfull = (1e-3 * (1 + np.arange(16))).astype(F32)      # 16 distinct entries, Q[r + 4c] != Q[c + 4r]
    return {
        "default": (dt, Q, R),
        "dt_0.05": (0.05, Q, R),
        "dt_1_30": (1.0 / 30.0, Q, R),                       # not a float: narrowing dt changes the bits
        "dt_1": (1.0, Q, R),
        "Q_full": (dt, Qfull, R),
        "R_asym": (dt, Q, np.array([1.0, 0.3, -0.2, 0.8], F32)),   # R[1] != R[2]
        "Q0": (dt, np.zeros(16, F32), R),
        "R_1e-6": (dt, Q, np.array([1e-6, 0, 0, 1e-6], F32)),       # S = PPred's xy block + 1e-6 I
    }


SETS = _sets()
NAMES = list(SETS)


def _params(dt, Q, R):
    p = EkfParams()
    p.dt = float(dt)
    for k in range(16):
        p.Q[k] = float(Q[k])
    for k in range(4):
        p.R[k] = float(R[k])
    return p


def _oracle(x, P, z, u, name_or_set, n_steps=1):
    dt, Q, R = SETS[name_or_set] if isinstance(name_or_set, str) else name_or_set
    return O.ekf_step_batched(x, P, z, u, Q=Q, R=R, dt=dt, n_steps=n_steps)


def _assert_same(got, want, what="", zero_sign=True, inf_input=None):
    """Bit for bit wherever the oracle is finite (signed zeros included), the same infinity where it is infinite,
    NaN where it is NaN (payloads are not compared).  Without FMA, the host glibc's sinf / cosf round differently from
    its FMA build (which the kernels restate) on ~2e-8 of the arguments: there a few agents in 1e6 may differ.

    The kernel skips the products with the structural zeros of F, B, jF and jH that the reference's dense Eigen
    products evaluate (crb_ekf.cu).  That is exact except in two places, which the callers name: zero_sign=False lets
    an exact zero have the other sign (a dense sum adds +0 terms, which turn -0 into +0), and inf_input marks agents
    with an infinite input, where the dense 0 * inf (F * x, jH * xPred) makes NaN of every entry, also of those the
    kernel computes without the infinite component: there only the oracle's finite and infinite entries bind."""
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    nan = np.isnan(want)
    if zero_sign:
        bad = ~nan & (got.view(np.uint32) != want.view(np.uint32))
    else:   # equal values have equal bits, except +0 and -0
        bad = ~nan & ~(got == want)
    lost_nan = nan & ~np.isnan(got)
    if inf_input is not None:
        lost_nan &= ~inf_input[None, :]
    bad |= lost_nan
    agents = np.flatnonzero(bad.any(axis=0))
    allowed = 0 if FMA_HOST else max(1, int(4e-6 * want.shape[-1]))
    if agents.size > allowed:
        raise AssertionError(f"{what}: {agents.size} agents differ from the oracle, first {agents[:8].tolist()}")


def _dev(a, misaligned=False):
    """A CUDA copy of `a`; misaligned=True makes it a contiguous view at storage offset 1 (4-byte aligned only)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if not misaligned:
        return t.cuda()
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 8 == 4
    return v


def _run_device(engine, x, P, z, u, prm, n_steps=1, misaligned=False):
    import torch
    d = [_dev(a, misaligned) for a in (x, P, z, u)]
    engine.ekf_estimation(*d, params=prm, n_steps=n_steps)
    torch.cuda.synchronize()
    return d[0].cpu().numpy(), d[1].cpu().numpy()


# ---- CPU: the parameter sets tell the constants apart ----------------------------------------------------------
def test_parameter_sets_catch_transposed_or_narrowed_constants():
    """The bitwise tests below would catch a kernel that read Q or R transposed (R[1] and R[2] swapped) or narrowed
    dt to float: the oracle's results with Q^T, R^T or (float)dt differ from those with Q, R, dt on nearly every
    agent (dt over 5 steps: one step changes the float rounding of 58 % of the agents, five steps of 98 %)."""
    n = 4000
    x, P, z, u = synth.ekf_inputs(n, n_steps=5)

    def frac_diff(a, b):
        return float(((a[0] != b[0]).any(axis=0) | (a[1] != b[1]).any(axis=0)).mean())
    dt, Q, R = SETS["Q_full"]
    assert frac_diff(_oracle(x, P, z, u, (dt, Q, R)), _oracle(x, P, z, u, (dt, Q.reshape(4, 4).T.ravel().copy(), R))) > 0.99
    dt, Q, R = SETS["R_asym"]
    assert frac_diff(_oracle(x, P, z, u, (dt, Q, R)), _oracle(x, P, z, u, (dt, Q, R[[0, 2, 1, 3]].copy()))) > 0.99
    dt, Q, R = SETS["dt_1_30"]
    assert frac_diff(_oracle(x, P, z, u, (dt, Q, R), n_steps=5),
                     _oracle(x, P, z, u, (float(F32(dt)), Q, R), n_steps=5)) > 0.95


# ---- every entry point at every parameter set --------------------------------------------------------------------
FORMS = {"two_agent": (4098, False), "one_agent_odd_n": (4097, False), "one_agent_misaligned": (4098, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("n_steps", [1, 5])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("name", NAMES)
def test_device_entry_at_every_parameter_set(engine, name, form, n_steps):
    """The two-agent kernel (even n, 8-byte aligned arrays) and the one-agent kernel (odd n, or arrays at a 4-byte
    offset) against the oracle with the same constants, one and five steps per launch."""
    n, mis = FORMS[form]
    x, P, z, u = synth.ekf_inputs(n, n_steps=n_steps, seed=0xE1 + n_steps)
    gx, gP = _run_device(engine, x, P, z, u, _params(*SETS[name]), n_steps, mis)
    xo, Po = _oracle(x, P, z, u, name, n_steps)
    _assert_same(gx, xo, "x")
    _assert_same(gP, Po, "P")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_host_entries_at_every_parameter_set(engine, name):
    """The staged host entry (pageable arrays, more than two chunks and a ragged tail) at one and five steps, and
    the zero-copy entry (pinned arrays, one launch on mapped memory)."""
    import torch
    n = 2 * CHUNK + 4097
    prm = _params(*SETS[name])
    for n_steps in (1, 5):
        x, P, z, u = synth.ekf_inputs(n, n_steps=n_steps, seed=0xE7 + n_steps)
        xo, Po = _oracle(x, P, z, u, name, n_steps)
        xs, Ps = x.copy(), P.copy()
        l0 = engine.launches
        engine.ekf_estimation_host(xs, Ps, z, u, params=prm, n_steps=n_steps)
        assert engine.launches - l0 == 3
        _assert_same(xs, xo, f"staged x, {n_steps} steps")
        _assert_same(Ps, Po, f"staged P, {n_steps} steps")
        pin = [torch.from_numpy(a.copy()).pin_memory() for a in (x, P, z, u)]
        l0 = engine.launches
        engine.ekf_estimation_host(*pin, params=prm, n_steps=n_steps)
        assert engine.launches - l0 == 1
        _assert_same(pin[0].numpy(), xo, f"zero-copy x, {n_steps} steps")
        _assert_same(pin[1].numpy(), Po, f"zero-copy P, {n_steps} steps")


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
def test_track_with_parameters_changed_between_steps(engine, pinned):
    """The resident track takes its constants per step: one step at each parameter set in turn, x_out after every
    step and x, P at the end against the oracle run with the same sequence."""
    import torch
    n = 4097
    K = len(NAMES)
    x, P, z, u = synth.ekf_inputs(n, n_steps=K, seed=0xE9)

    def host(a):
        t = torch.from_numpy(np.ascontiguousarray(a))
        return t.pin_memory() if pinned else t
    trk = engine.ekf_track_open(x, P)
    xo, Po = x, P
    try:
        for k, name in enumerate(NAMES):
            out = host(np.zeros((4, n), F32))
            engine.ekf_track_step(trk, host(z[2 * k:2 * k + 2]), host(u[2 * k:2 * k + 2]), params=_params(*SETS[name]),
                                  x_out=out)
            xo, Po = _oracle(xo, Po, z[2 * k:2 * k + 2], u[2 * k:2 * k + 2], name)
            _assert_same(out.numpy(), xo, f"x_out after step {k} ({name})")
        gx, gP = np.empty_like(x), np.empty_like(P)
        engine.ekf_track_read(trk, gx, gP)
    finally:
        engine.ekf_track_close(trk)
    _assert_same(gx, xo, "x")
    _assert_same(gP, Po, "P")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [k for k in NAMES if k != "R_1e-6"])
def test_device_entry_tracks_float64_at_every_parameter_set(engine, name):
    """Against the float64 statement of the same step (O.ekf_estimation_f64), field-normalised per agent.  R = 1e-6 I
    is left out: there the update cancels the xy block of PPred down to ~1e-6, the difference of O(1) terms, so float32
    keeps only the leading bits of those entries and how close they come to float64 says nothing about the kernel;
    the bitwise comparison with the oracle above is its test."""
    n = 2000
    dt, Q, R = SETS[name]
    x, P, z, u = synth.ekf_inputs(n, seed=0xEB)
    gx, gP = _run_device(engine, x, P, z, u, _params(dt, Q, R))
    X, PP = np.empty((4, n)), np.empty((16, n))
    for i in range(n):
        X[:, i], PP[:, i] = O.ekf_estimation_f64(x[:, i], P[:, i], z[:, i], u[:, i], Q=Q, R=R, dt=dt)

    def field_err(got, want):
        return (np.abs(got - want).max(axis=0) / np.abs(want).max(axis=0)).max()
    assert field_err(gx, X) <= 1e-5
    assert field_err(gP, PP) <= 1e-5


# ---- special values ------------------------------------------------------------------------------------------------
def _special_batch(n):
    """ekf_inputs with isolated agents poisoned; returns the arrays and the poisoned agent indices.  Pair partners
    (2k, 2k+1) of poisoned agents are left clean on both sides."""
    x, P, z, u = synth.ekf_inputs(n, seed=0xED)
    nan, inf = F32(np.nan), F32(np.inf)
    big = F32(3e38)
    poison = {
        2: lambda: z.__setitem__((0, 2), nan),
        5: lambda: u.__setitem__((1, 5), inf),                # agent 2k+1 poisoned, its partner 4 clean
        8: lambda: x.__setitem__((2, 8), -inf),               # yaw -inf: sin / cos NaN
        11: lambda: P.__setitem__((5, 11), nan),
        14: lambda: x.__setitem__((0, 14), inf),
        17: lambda: u.__setitem__((0, 17), -nan),
        20: lambda: x.__setitem__((2, 20), nan),
        23: lambda: P.__setitem__((10, 23), inf),
        26: lambda: z.__setitem__((1, 26), -inf),
        # finite values whose products or sums overflow
        29: lambda: P.__setitem__((slice(None), 29), big),
        32: lambda: (z.__setitem__((0, 32), big), x.__setitem__((0, 32), -big)),
        35: lambda: u.__setitem__((0, 35), big),
        38: lambda: x.__setitem__((3, 38), big),
    }
    for f in poison.values():
        f()
    # signed zeros everywhere (P = -0 too: the update then runs on exact zeros of both signs)
    for a in (x, z, u):
        a[:, 41] = F32(-0.0)
    P[:, 41] = F32(-0.0)
    P[:, 44] = 0.0
    P[[0, 5, 10, 15], 44] = F32(-0.0)
    # subnormal P: a yaw / speed block of 1e-39 with u0 = 0, so the subnormals reach x and P through jF's products
    P[:, 47] = 0.0
    P[0, 47] = P[5, 47] = 0.5
    P[[10, 11, 14, 15], 47] = F32(1e-39)
    u[0, 47] = 0.0
    P[:, 50] = F32(1e-39)
    P[[0, 5], 50] = F32(0.25)
    return x, P, z, u, sorted(poison) + [41, 44, 47, 50]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 65])
def test_special_values_follow_the_oracle(engine, n):
    """NaN and +-inf in z, u, x and P, signed zeros, subnormal P, and finite inputs that overflow, each in an isolated
    agent, in the two-agent (n = 64) and the one-agent (n = 65) kernel; every other agent keeps its clean bits."""
    x, P, z, u, special = _special_batch(n)
    prm = SETS["default"]
    gx, gP = _run_device(engine, x, P, z, u, _params(*prm))
    xo, Po = _oracle(x, P, z, u, prm)
    # agent 41 (all inputs -0) may return +0 for -0, agent 14 (x = +inf) numbers where the reference's 0 * inf gives
    # NaN (see _assert_same); every other agent bit for bit, and x of agent 14 must not come back finite
    strict = np.setdiff1d(np.arange(n), [14, 41])
    _assert_same(gx[:, strict], xo[:, strict], "x")
    _assert_same(gP[:, strict], Po[:, strict], "P")
    inf_input = np.zeros(2, bool)
    inf_input[0] = True
    _assert_same(gx[:, [14, 41]], xo[:, [14, 41]], "x of agents 14, 41", zero_sign=False, inf_input=inf_input)
    _assert_same(gP[:, [14, 41]], Po[:, [14, 41]], "P of agents 14, 41", zero_sign=False, inf_input=inf_input)
    assert not np.isfinite(gx[:, 14]).any()
    assert np.isnan(xo[:, 2]).all() and np.isnan(Po[:, 29]).all()           # the poison did reach the outputs
    assert np.isinf(xo[:, 26]).all() and np.isinf(xo[:, 32]).all()           # z = -inf; z - x overflows to inf
    clean = np.setdiff1d(np.arange(n), special)
    xc, Pc = _oracle(*(np.ascontiguousarray(a[:, clean]) for a in (x, P, z, u)), prm)
    assert np.array_equal(gx[:, clean], xc) and np.array_equal(gP[:, clean], Pc)
    assert ((np.abs(Po[:, 47]) < 2.0 ** -126) & (Po[:, 47] != 0)).any()        # subnormal results to compare


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 65])
def test_subnormal_constants_and_a_singular_innovation_covariance(engine, n):
    """Q and R with subnormal entries (a flush-to-zero or fast-math build changes these bits); then Q = R = 0 with
    agents whose P is zero, so S = 0, det = 0 and S^-1 is inf * 0 = NaN, beside agents with a regular S."""
    x, P, z, u = synth.ekf_inputs(n, seed=0xEF)
    dt, Q, R = SETS["default"]
    Qs, Rs = Q.copy(), R.copy()
    Qs[[1, 4, 14]] = F32(1e-40)
    Rs[[1, 2]] = (F32(3e-42), F32(-2e-41))
    P[:, 3::4] = 0.0
    P[[0, 5, 10, 15], 3::4] = 0.5
    P[[10, 11, 14, 15], 7::8] = F32(1e-39)
    u[0, 7::8] = 0.0
    gx, gP = _run_device(engine, x, P, z, u, _params(dt, Qs, Rs))
    xo, Po = _oracle(x, P, z, u, (dt, Qs, Rs))
    _assert_same(gx, xo, "x (subnormal Q, R)")
    _assert_same(gP, Po, "P (subnormal Q, R)")
    assert ((np.abs(Po) < 2.0 ** -126) & (Po != 0)).any()
    Z = np.zeros(16, F32)
    P[:, ::3] = 0.0
    gx, gP = _run_device(engine, x, P, z, u, _params(dt, Z, Z[:4]))
    xo, Po = _oracle(x, P, z, u, (dt, Z, Z[:4]))
    _assert_same(gx, xo, "x (S = 0)")
    # with Q = R = 0 the update cancels the xy rows of P to exact zeros, whose sign the dense evaluation can flip
    _assert_same(gP, Po, "P (S = 0)", zero_sign=False)
    assert np.isnan(xo[:, ::3]).any() and np.isfinite(xo[:, 1::3]).all()


# ---- yaw: the branch edges of sinf / cosf and the whole range beyond 120 -----------------------------------------
def _yaw_cases():
    def around(v, k=3):
        b = int(np.float32(v).view(np.uint32))
        return [np.uint32(b + d).view(F32) for d in range(-k, k + 1) if 0 <= b + d < 0x7F800000]
    ys = [F32(0.0)]
    ys += around(2.0 ** -12)                                   # the |y| < 2^-12 shortcut
    ys += around(0.75) + around(np.pi / 4)                     # abstop12 = 0x3f4 starts reduce_fast; pi/4 itself
    for k in range(1, 77):                                     # multiples of pi/2 below 120
        ys += around(k * np.pi / 2, 2)
    ys += around(119.99999) + around(120.0)                    # 0x42f00000: reduce_large from here on
    for k in range(7, 128):
        ys += around(2.0 ** k, 1)
    for v in (1e3, 1e6, 2.0 ** 23, 2.0 ** 24):
        ys += around(v)
    ys += around(np.finfo(F32).max, 2)
    rng = np.random.default_rng(120)
    ys += list(rng.integers(0x42F00000, 0x7F800000, 100_000, dtype=np.uint64).astype(np.uint32).view(F32))
    ys = np.asarray(ys, F32)
    return np.concatenate([ys, -ys])


@pytest.mark.gpu
@pytest.mark.parametrize("odd", [False, True])
def test_any_yaw_matches_the_host_libm(engine, odd):
    """EKF at yaw around every branch edge of glibc's sinf / cosf, at 120 (where glibc switches to reduce_large), at
    the powers of two up to 2^127, at FLT_MAX and at 1e5 random floats with |yaw| >= 120, both signs: every agent
    bit for bit.  The predicted yaw xp[2] = yaw + dt * u1 feeds jacobF's sin / cos: u1 = 0 keeps it at yaw, and a
    second batch with u1 = +-1 and yaw just inside +-120 puts only xp[2] past 120."""
    ys = _yaw_cases()
    n = ys.size + ys.size % 2 + int(odd)                      # even: the two-agent kernel, odd: the one-agent one
    x, P, z, u = synth.ekf_inputs(n, seed=0xF1)
    x[2, :ys.size] = ys
    u[1] = 0.0
    prm = SETS["default"]
    gx, gP = _run_device(engine, x, P, z, u, _params(*prm))
    xo, Po = _oracle(x, P, z, u, prm)
    _assert_same(gx, xo, "x")
    _assert_same(gP, Po, "P")
    # only the predicted yaw crosses 120
    m = 4096 + int(odd)
    x, P, z, u = synth.ekf_inputs(m, seed=0xF3)
    inside = np.array([119.99, 119.95, 119.9000015, np.nextafter(F32(120), F32(0))], F32)
    x[2] = np.resize(np.concatenate([inside, -inside]), m)
    u[1] = np.sign(x[2]) * np.resize(np.array([1.0, 0.75, 1.0, 0.5], F32), m)
    xp2 = x[2] + F32(0.1) * u[1]
    assert (np.abs(xp2) >= 120).all() and (np.abs(x[2]) < 120).all()
    gx, gP = _run_device(engine, x, P, z, u, _params(*prm))
    xo, Po = _oracle(x, P, z, u, prm)
    _assert_same(gx, xo, "x (xp[2] past 120)")
    _assert_same(gP, Po, "P (xp[2] past 120)")


@pytest.mark.gpu
def test_long_track_turns_past_3000_rad(engine):
    """The reference's open-ended loop never wraps yaw.  4096 agents at yaw rates up to +-10 rad/s for 3000 steps of
    0.1 s (|yaw| up to ~3000): x_out after every step, and x, P at the end, bit for bit."""
    n, K = 4096, 3000
    x, P, _, _ = synth.ekf_inputs(n, seed=0xF5)
    rng = np.random.default_rng(3000)
    rate = rng.uniform(-10.0, 10.0, n).astype(F32)
    speed = rng.uniform(0.0, 2.0, n).astype(F32)
    trk = engine.ekf_track_open(x, P)
    xo, Po = x, P
    out = np.zeros((4, n), F32)
    try:
        for k in range(K):
            u = np.stack([speed, rate]).astype(F32)
            z = (xo[:2] + rng.normal(0.0, 0.25, (2, n))).astype(F32)
            engine.ekf_track_step(trk, z, u, x_out=out)
            xo, Po = O.ekf_step_batched(xo, Po, z, u)
            if not np.array_equal(out, xo):
                _assert_same(out, xo, f"x_out after step {k}")
        gx, gP = np.empty_like(x), np.empty_like(P)
        engine.ekf_track_read(trk, gx, gP)
    finally:
        engine.ekf_track_close(trk)
    assert np.abs(xo[2]).max() > 2500
    assert np.array_equal(gx, xo) and np.array_equal(gP, Po)


# ---- element offsets past 2^31 -------------------------------------------------------------------------------------
BLOCK = 65_521   # prime: an offset wrapped by a multiple of 2^31 lands on an agent of another residue


@pytest.mark.gpu
@pytest.mark.parametrize("n,n_steps", [((1 << 28) + 3, 1), ((1 << 28) + 2, 1), ((1 << 27) + 1, 4)],
                         ids=["one_agent_2^28+3", "two_agent_2^28+2", "steps4_2^27+1"])
def test_offsets_past_2_31(engine, n, n_steps):
    """19 * n + i passes 2^31 from n ~ 1.1e8; with 4 steps at 2^27 the z / u rows reach 7 * n + i, 2^32 bytes.
    Agent i gets the inputs of agent i mod L of one block of L = 65521 (prime) agents, so it must produce exactly the
    block's result for agent i mod L; an offset computed in 32 bits would be off by a multiple of 2^31 elements, not
    a multiple of L, and bring another agent's numbers (or none)."""
    import torch
    fields = 20 + 4 * n_steps
    need = 4 * n * fields + (3 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    x, P, z, u = synth.ekf_inputs(BLOCK, n_steps=n_steps, seed=0xF7)
    xo, Po = O.ekf_step_batched(x, P, z, u, n_steps=n_steps)
    reps = -(-n // BLOCK)

    def tile(a):
        src = torch.from_numpy(a).cuda()
        out = torch.empty((a.shape[0], n), dtype=torch.float32, device="cuda")
        for f in range(a.shape[0]):
            out[f].copy_(src[f].repeat(reps)[:n])
        return out
    d = [tile(a) for a in (x, P, z, u)]
    try:
        engine.ekf_estimation(*d, n_steps=n_steps)
        torch.cuda.synchronize()
        want = [torch.from_numpy(a).cuda() for a in (xo, Po)]
        step = 1 << 24
        for a0 in range(0, n, step):
            a1 = min(n, a0 + step)
            idx = torch.arange(a0, a1, device="cuda") % BLOCK
            for got, w, what in ((d[0], want[0], "x"), (d[1], want[1], "P")):
                assert torch.equal(got[:, a0:a1], w[:, idx]), f"{what}: agents [{a0}, {a1}) differ"
    finally:
        del d
        torch.cuda.empty_cache()


# ---- crb_sincosf_libm itself ---------------------------------------------------------------------------------------
SINCOSF_CENSUS_CU = r"""
// crb_sincosf_libm on the device for every float of [lo, hi) (both signs, in chunks), checked on the host by the
// checker's crb_oracle_libm_sincosf_check (argv[3] = liboracle.so).  Prints the number of mismatching arguments.
#include <dlfcn.h>

#include "crb_common.cuh"
__global__ void census(unsigned lo, unsigned long long count, float* out) {
  for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned b = (lo + (unsigned)(k >> 1)) | ((k & 1) ? 0x80000000u : 0u);
    float s, c;
    crb_sincosf_libm(__uint_as_float(b), s, c);
    out[2 * k] = s;
    out[2 * k + 1] = c;
  }
}
int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const unsigned lo = (unsigned)strtoul(argv[1], 0, 0), hi = (unsigned)strtoul(argv[2], 0, 0);
  void* so = dlopen(argv[3], RTLD_NOW);
  if (!so) return 2;
  typedef long long (*check_fn)(unsigned, unsigned, const float*);
  check_fn check = (check_fn)dlsym(so, "crb_oracle_libm_sincosf_check");
  if (!check) return 2;
  const unsigned chunk = 1u << 26;
  float *d, *h;
  if (cudaMalloc(&d, 4ull * chunk * 4) != cudaSuccess || cudaMallocHost(&h, 4ull * chunk * 4) != cudaSuccess) return 3;
  long long bad = 0;
  for (unsigned a = lo; a < hi; a = (hi - a > chunk) ? a + chunk : hi) {
    const unsigned b = (hi - a > chunk) ? a + chunk : hi;
    census<<<2048, 256>>>(a, 2ull * (b - a), d);
    if (cudaMemcpy(h, d, 4ull * (b - a) * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
    bad += check(a, b, h);
  }
  printf("%lld\n", bad);
  cudaFreeHost(h);
  cudaFree(d);
  return 0;
}
"""


@pytest.mark.gpu
def test_gpu_sincosf_census_against_the_checker(engine, tmp_path):
    """crb_sincosf_libm on the device against the checker's C restatement (itself pinned to the host libm by
    tests/test_oracle_ekf.py) on all 2^32 bit patterns: sin and cos, NaN matching NaN."""
    import __graft_entry__ as G
    src = tmp_path / "census.cu"
    src.write_text(SINCOSF_CENSUS_CU)
    exe = tmp_path / "census"
    subprocess.check_call([G.NVCC] + G.GENCODE + ["-O3", "-std=c++17", "-fmad=false",
                           "-I", os.path.join(ROOT, "cpprobotics_b200", "csrc"), str(src), "-o", str(exe), "-ldl"])
    out = subprocess.check_output([str(exe), "0x0", "0x80000000", O.LIB_PATH], text=True)
    assert int(out.strip()) == 0


# ---- the other crb_sincosf_libm callers beyond 120 -----------------------------------------------------------------
@pytest.mark.gpu
def test_pf_predicted_positions_at_large_yaw(engine):
    import torch
    n = 4097
    px, pw, noise = synth.pf_inputs(n)
    rng = np.random.default_rng(121)
    yaw = np.concatenate([rng.uniform(120.0, 1e4, n // 2), rng.integers(0x42F00000, 0x7F800000, n - n // 2)
                          .astype(np.uint32).view(F32)]).astype(F32)
    px[2] = yaw * np.where(rng.random(n) < 0.5, F32(-1), F32(1))
    lm = synth.pf_landmarks(8)
    pxd, pwd, nd = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (px, pw, noise))
    engine.pf_predict_weight(pxd, pwd, nd, lm)
    torch.cuda.synchronize()
    pxo, _ = O.pf_predict_weight_batched(px, pw, noise, lm)
    _assert_same(pxd.cpu().numpy(), pxo, "predicted positions")


@pytest.mark.gpu
def test_mpc_plant_update_at_large_yaw(engine):
    import torch
    n = 2000
    st, _ = synth.mpc_states(n)
    rng = np.random.default_rng(122)
    st[2] = rng.uniform(120.0, 1e5, n).astype(F32) * np.where(rng.random(n) < 0.5, F32(-1), F32(1))
    u0 = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-0.5, 0.5, n)]).astype(F32)
    std, u0d = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (st, u0))
    engine.mpc_plant_update(std, u0d)
    torch.cuda.synchronize()
    want = np.stack([O.plant_update(st[:, i], u0[0, i], u0[1, i]) for i in range(n)], axis=1)
    _assert_same(std.cpu().numpy(), want, "state")
