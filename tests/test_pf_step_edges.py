"""crb_pf_step, one complete particle-filter iteration, at the edges of its launch forms, layouts and weight shapes.

crb_pf_step runs three launches for n <= 2^21 (PF2_MAX_CHUNKS * 2048) and seven above.  Every case here checks the
GPU against float64 / oracle restatements of the same operations, fed with the GPU's own intermediate state:
  - predict + weight against the oracle's stages (positions bit-exact except glibc's FMA-build cases);
  - the normalised weights as float(w / float(sum w)) with the GPU's own weight sum;
  - Neff within one float ulp of the oracle's from the same weights, and the decision exactly `Neff < nth`;
  - px_next and pw against oracle resampling on the GPU's weights, bit for bit except at cumulative-weight ties of
    the two summation orders (or a bit copy without resampling);
  - xEst within one float ulp of the float64 weighted mean, and PEst entry by entry against the float64 two-pass
    covariance around that xEst (calc_covariance, src/particle_filter.cpp:59-71):
    |dP_rc| <= 1e-6 sqrt(P_rr P_cc), PEst exactly symmetric with a non-negative diagonal."""
import numpy as np
import pytest

from cpprobotics_b200 import Engine, synth
from oracle import oracle as O

F32 = np.float32
CHUNK = 2048                # weights per scan block
FORM_SIZES = (1 << 20, (1 << 21) + 1)   # the three-launch and the seven-launch form


# ---- helpers ----------------------------------------------------------------------------------------------------
def _assert_pf_parity(px_got, pw_got, px_want, pw_want, lm, sigma2=0.01):
    """Per-particle relative 1e-5 on w.

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


def _philox_u12(seed, n):
    """crb_oracle_philox_uniform12(seed, j) for j = 0 .. n-1, vectorised: the uniforms in [1, 2) the resampling
    draws when no uniforms are given."""
    m32 = np.uint64(0xFFFFFFFF)
    idx = np.arange(n, dtype=np.uint64)
    c0, c1 = idx & m32, idx >> np.uint64(32)
    c2 = np.full(n, 0x5EED5EED, np.uint64)
    c3 = np.zeros(n, np.uint64)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m32
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return F32(1.0) + (c0 >> np.uint64(9)).astype(F32) * F32(1.1920928955078125e-07)


def test_vectorised_philox_uniforms_match_the_oracle():
    seed = 0x9_8765_4321
    idx = [0, 1, 2, 1023, 1024, 999_999, (1 << 21) + 1]
    u = _philox_u12(seed, idx[-1] + 1)
    assert [float(u[j]) for j in idx] == [O.philox_uniform12(seed, j) for j in idx]


def _to_dev(a, offset=False):
    """A CUDA copy of `a`; with offset=True a view one float into a larger buffer (4-byte aligned only), which
    makes the packed predict kernel and the 16-byte staging of the scan inapplicable."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if not offset:
        return t.cuda()
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 8 == 4
    return v


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def _check_estimate(gx, gw, xe_got, P_got):
    """xEst within one float ulp of the float64 weighted mean; PEst against the float64 two-pass covariance around
    that xEst with d = float32(px - xEst), as calc_covariance.  Returns max |dP_rc| / sqrt(P_rr P_cc)."""
    if not np.isfinite(gw).all():
        assert np.isnan(xe_got).all() and np.isnan(P_got).all()
        return 0.0
    w = gw.astype(np.float64)
    m = gx.astype(np.float64) @ w
    xe = xe_got.astype(F32)
    assert np.array_equal(xe.astype(np.float64), xe_got)
    assert (np.abs(xe_got - m) <= np.spacing(np.abs(m).astype(F32)).astype(np.float64)).all(), (xe_got, m)
    d = (gx - xe[:, None]).astype(np.float64)
    C = (d * w) @ d.T
    assert np.array_equal(P_got, P_got.T)
    assert (np.diag(P_got) >= 0).all()
    scale = np.sqrt(np.outer(np.diag(C), np.diag(C)))
    err = np.abs(P_got - C)
    ratio = float(np.max(np.where(scale > 0, err / np.where(scale > 0, scale, 1.0), np.where(err > 0, np.inf, 0.0))))
    assert ratio <= 1e-6, f"max |dP| / sqrt(P_rr P_cc) = {ratio:.3g}\nGPU\n{P_got}\ntwo-pass\n{C}"
    return ratio


def _assert_same_survivors(nxt, px2, gx, gw, U):
    """Resampled particles against the oracle, bit for bit, except at ties of the cumulative weight.

    The GPU sums the weights in blocks, the oracle in sequence; both round the double sums to the float wcum.  Where a
    double prefix sum lies within its rounding error of a float rounding boundary the two wcum can differ by one float
    ulp, and a resampleid equal to one of them then picks a neighbouring particle (a few per 10^6 particles with
    synthetic weights).  Every differing slot j must be such a tie: the GPU's particle is one within 64 of the
    oracle's, and every cumulative weight between the two lies within one float ulp of resampleid_j."""
    n = gx.shape[1]
    bad = np.flatnonzero(~(nxt == px2).all(axis=0))
    if bad.size == 0:
        return
    assert bad.size <= max(2, n >> 16), f"{bad.size} resampled particles differ, first at j = {bad[:8]}"
    w64 = np.cumsum(gw.astype(np.float64))
    wcum = w64.astype(F32)
    j = np.arange(n)
    rid = ((j / n).astype(F32).astype(np.float64) + U / n).astype(F32)
    rid[1:] = np.maximum(rid[1:], rid[:-1])          # the reference's search index never moves back
    for jb in bad:
        i_o = min(int(np.searchsorted(wcum, rid[jb], "left")), n - 1)
        assert (px2[:, jb] == gx[:, i_o]).all()
        lo, hi = max(0, i_o - 64), min(n, i_o + 65)
        ks = lo + np.flatnonzero((gx[:, lo:hi] == nxt[:, [jb]]).all(axis=0))
        assert ks.size, f"slot {jb}: the GPU's particle is not within 64 of the oracle's {i_o}"
        tie = lambda k: (np.abs(w64[min(k, i_o):max(k, i_o)] - rid[jb]) <= np.spacing(rid[jb])).all()
        assert any(tie(int(k)) for k in ks), f"slot {jb}: a different particle without a cumulative-weight tie"


def _step(engine, px, pw, noise, lm, nth, uniforms, resample_seed, seed, offset):
    import torch
    a, b = _to_dev(px, offset), _to_dev(pw, offset)
    nd = None if noise is None else _to_dev(noise, offset)
    ud = None if uniforms is None else _to_dev(uniforms)
    nxt = _to_dev(np.full_like(px, np.nan), offset)
    r = engine.pf_step(a, b, nxt, nd, lm, seed=seed, uniforms=ud, resample_seed=resample_seed, nth=nth)
    torch.cuda.synchronize()
    return a.cpu().numpy(), b.cpu().numpy(), nxt.cpu().numpy(), r.cpu().numpy()


def _check_step(engine, px, pw, noise, lm, *, nth, uniforms=None, resample_seed=0, seed=0, offset=False,
                weights_unchanged=False):
    """One crb_pf_step case checked end to end (see the module docstring).  Returns the GPU's state."""
    import torch
    n = px.shape[1]
    lm = np.asarray(lm, F32).reshape(-1, 3)
    # predict + weight on their own, against the oracle's stages
    a, b = _to_dev(px, offset), _to_dev(pw, offset)
    engine.pf_predict_weight(a, b, None if noise is None else _to_dev(noise, offset), lm, seed=seed)
    torch.cuda.synchronize()
    rx, rw = a.cpu().numpy(), b.cpu().numpy()
    pxo, pwo = O.pf_predict_weight_batched(px, pw, noise, lm, seed=seed)
    if noise is not None:
        _assert_pf_parity(rx, rw, pxo, pwo, lm)
    else:   # Philox normals: logf is CUDA's (<= 1 ulp from glibc's), positions agree to an ulp or two
        assert (np.abs(rx - pxo).max(axis=1) <= 1e-5 * np.maximum(1.0, np.abs(pxo).max(axis=1))).all()
    if weights_unchanged:   # n_lm = 0: the weight update is W * exp(0)
        assert np.array_equal(rw, pw)
    # never resample: px_next is a bit copy, pw the normalised weights
    gx, gw, n0, r0 = _step(engine, px, pw, noise, lm, 0.0, uniforms, resample_seed, seed, offset)
    assert np.array_equal(gx, rx), "crb_pf_step predicts other positions than crb_pf_predict_weight_batched"
    assert r0[22] == 0.0 and np.array_equal(n0, gx)
    s = np.sum(rw, dtype=np.float64)
    assert abs(r0[20] - s) <= 1e-12 * abs(s), (r0[20], s)
    with np.errstate(invalid="ignore"):   # all-zero weights: 0 / 0
        assert _same(gw, rw / F32(r0[20])), "weights are not float(w / float(sum w))"
    # the requested threshold: the same estimate, Neff, the decision and the index work
    x1, w1, nxt, r = _step(engine, px, pw, noise, lm, nth, uniforms, resample_seed, seed, offset)
    assert np.array_equal(x1, gx) and _same(r[:22], r0[:22]) and _same(r[23], r0[23])
    U = (uniforms if uniforms is not None else _philox_u12(resample_seed, n)).astype(np.float64)
    neff_o = O.pf_resample(gx, gw, U, nth=0.0)[3]
    neff = F32(r[21])
    assert (np.isnan(neff) and np.isnan(neff_o)) or abs(neff - F32(neff_o)) <= np.spacing(F32(neff_o)), (neff, neff_o)
    assert r[22] == (1.0 if neff < F32(nth) else 0.0)
    if r[22]:
        px2, pw2, did, _ = O.pf_resample(gx, gw, U, nth=np.inf)
        assert did
        _assert_same_survivors(nxt, px2, gx, gw, U)
        assert np.array_equal(w1, pw2)
    else:
        assert np.array_equal(nxt, gx) and _same(w1, gw)
    ratio = _check_estimate(gx, gw, r0[0:4], r0[4:20].reshape(4, 4).T)
    return dict(x=gx, w=gw, r=r, nxt=nxt, w_out=w1, ratio=ratio)


def _inputs(n, n_lm=8, seed=0xC0FFEE):
    px, pw, noise = synth.pf_inputs(n, seed=seed)
    lm = synth.pf_landmarks(n_lm) if n_lm else np.zeros((0, 3), F32)
    return px, pw, noise, lm


# ---- shapes x layouts -------------------------------------------------------------------------------------------
SHAPES = [1, 2, 3, 255, 1023, 1024, 1025, 2047, 2048, 2049, 4097, 1 << 20, 1_000_002, (1 << 21) - 1, 1 << 21,
          (1 << 21) + 1, (1 << 21) + 2, 3 * (1 << 20) + 7]
OFFSET_SHAPES = [2, 1024, 2048, 1 << 20, 1_000_002, 1 << 21, (1 << 21) + 2]


@pytest.mark.gpu
@pytest.mark.parametrize("n,offset", [(n, False) for n in SHAPES] + [(n, True) for n in OFFSET_SHAPES])
def test_pf_step_shapes_and_layouts(engine, n, offset):
    """Ragged tails, n at the 2048-weight chunk and 1024-output tile boundaries, n = 2^21 (all 1024 chunk offsets
    of the three-launch form in use) and the seven-launch form above it.  Arrays one float into a larger buffer take
    the general predict kernel plus a separate weight-sum pass and the 4-byte staging of the scan."""
    px, pw, noise, lm = _inputs(n)
    u = (1.0 + np.random.default_rng(n).random(n)).astype(F32)
    _check_step(engine, px, pw, noise, lm, nth=float(n), uniforms=u, offset=offset)


# ---- Philox noise and Philox resampling -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1025, 1 << 20, 1_000_000, 1 << 21, (1 << 21) + 1])
def test_pf_step_philox_resampling(engine, n):
    """noise = None and uniforms = None with seeds above 2^32 (the seed's high word keys Philox): the three-launch
    form computes these resampleids before its dependency wait, with reciprocal quotients (their census is in
    tests/test_oracle_pf.py).  This is the path bench.py's pf_full_iteration runs."""
    px, pw, _, lm = _inputs(n)
    _check_step(engine, px, pw, None, lm, nth=float(n), seed=0x1_2345_6789, resample_seed=0x9_8765_4321 + n)


# ---- landmark counts --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_lm", [0, 1, 64])
@pytest.mark.parametrize("n", [4097, (1 << 21) + 1])
def test_pf_step_landmark_counts(engine, n, n_lm):
    px, pw, noise, lm = _inputs(n, n_lm)
    u = (1.0 + np.random.default_rng(7).random(n)).astype(F32)
    _check_step(engine, px, pw, noise, lm, nth=float(n), uniforms=u, weights_unchanged=n_lm == 0)


# ---- controlled weights -----------------------------------------------------------------------------------------
def _weights(kind, n):
    """Weight families that synthetic likelihoods never produce: one-hot, the NP-1 cap, long zero runs, two levels
    2^20 apart, and heavy-tailed gamma(0.1) weights clipped to a narrow exponent span with a quarter of them dead."""
    rng = np.random.default_rng(WEIGHT_KINDS.index(kind))
    w = np.zeros(n, np.float64)
    if kind.startswith("onehot"):
        w[{"onehot_first": 0, "onehot_last": n - 1, "onehot_chunk_end": 100 * CHUNK - 1,
           "onehot_chunk_start": 100 * CHUNK}[kind]] = 1.0
    elif kind == "cap":             # all mass on NP-1, tiny weights elsewhere: the reference's cap (:139)
        w[:] = 2.0 ** -40
        w[-1] = 1.0
    elif kind == "zero_run":        # > 4096 zeros between normal weights: both non-staged window searches
        w[:] = 1.0 + np.floor(rng.random(n) * 64)
        a = n // 3
        w[a:a + 5000] = 0.0
        w[2 * a:2 * a + 9000] = 0.0
    elif kind == "two_levels":
        w[:] = np.where(rng.random(n) < 0.5, 1.0, 2.0 ** -20)
    elif kind == "gamma":           # heavy-tailed, a quarter dead, clipped to a span of 2^(29 - log2 n)
        g = rng.gamma(0.1, 1.0, n)
        span = 2.0 ** (29 - int(np.ceil(np.log2(n))))
        g = np.clip(g, g.max() / span, None)
        w = g.astype(F32).astype(np.float64)
        w[rng.integers(0, n, n // 4)] = 0.0
    elif kind == "all_zero":
        pass
    return w.astype(F32)


WEIGHT_KINDS = ["onehot_first", "onehot_last", "onehot_chunk_end", "onehot_chunk_start", "cap", "zero_run",
                "two_levels", "gamma", "all_zero"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", WEIGHT_KINDS)
@pytest.mark.parametrize("n", FORM_SIZES)
def test_pf_step_controlled_weights(engine, n, kind):
    """With no landmarks the weight update is W * exp(0): the weights are what the test sets.  All-zero weights are
    0 / 0 in the reference (:104): NaN weights and estimate, Neff NaN, no resampling, px_next a copy.  The same
    weights then go through crb_pf_resample, whose gather reads materialised cumulative weights."""
    import torch
    px, _, noise, lm = _inputs(n, 0)
    pw = _weights(kind, n)
    u = (1.0 + np.random.default_rng(3).random(n)).astype(F32)
    st = _check_step(engine, px, pw, noise, lm, nth=float(n), uniforms=u, weights_unchanged=True)
    if kind == "all_zero":
        assert np.isnan(st["r"][0:20]).all() and np.isnan(st["w"]).all() and st["r"][22] == 0.0
    elif kind.startswith("onehot"):   # every slot takes the hot particle, or NP-1 where resampleid passes 1 (:139)
        hot, last = st["x"][:, [int(np.argmax(pw))]], st["x"][:, [-1]]
        assert st["r"][22] == 1.0 and ((st["nxt"] == hot).all(axis=0) | (st["nxt"] == last).all(axis=0)).all()
    elif kind == "cap":
        assert st["r"][22] == 1.0 and (st["nxt"][:, -2:] == st["x"][:, [-1]]).all()
    # the stand-alone resampling entry on the same particles and normalised weights
    gx, gw = st["x"], st["w"]
    a, b, ud = _to_dev(gx), _to_dev(gw), _to_dev(u)
    did, neff = engine.pf_resample(a, b, uniforms=ud, nth=float("inf"))
    torch.cuda.synchronize()
    px2, pw2, did_o, neff_o = O.pf_resample(gx, gw, u.astype(np.float64), nth=np.inf)
    assert did == did_o
    assert (np.isnan(neff) and np.isnan(neff_o)) or abs(F32(neff) - F32(neff_o)) <= np.spacing(F32(neff_o))
    if did:
        _assert_same_survivors(a.cpu().numpy(), px2, gx, gw, u.astype(np.float64))
    else:
        assert _same(a.cpu().numpy(), px2)
    assert _same(b.cpu().numpy(), pw2)


# ---- the decision boundary --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", FORM_SIZES)
def test_pf_step_decision_boundary(engine, n):
    """Neff < nth (:127) is strict: nth = Neff keeps the particles, the next float above resamples."""
    px, pw, noise, lm = _inputs(n)
    _, _, _, r = _step(engine, px, pw, noise, lm, 0.0, None, 5, 0, False)
    neff = F32(r[21])
    st = _check_step(engine, px, pw, noise, lm, nth=float(neff), resample_seed=5)
    assert st["r"][22] == 0.0
    st = _check_step(engine, px, pw, noise, lm, nth=float(np.nextafter(neff, F32(np.inf))), resample_seed=5)
    assert st["r"][22] == 1.0


# ---- closed loop and context reuse ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", FORM_SIZES)
def test_pf_step_closed_loop_ping_pong(engine, n):
    """Three iterations with px / px_next swapped between calls, as a caller runs the filter.  Each iteration is
    checked against the oracle fed with the GPU's own state, and the ping-pong buffers hold exactly that state."""
    import torch
    px, pw, _, lm = _inputs(n)
    A, W = _to_dev(px), _to_dev(pw)
    B = torch.empty_like(A)
    for it in range(3):
        noise = synth.pf_inputs(n, seed=100 + it)[2]
        u = (1.0 + np.random.default_rng(it).random(n)).astype(F32)
        host_x, host_w = A.cpu().numpy(), W.cpu().numpy()
        st = _check_step(engine, host_x, host_w, noise, lm, nth=n / 2, uniforms=u)
        r = engine.pf_step(A, W, B, _to_dev(noise), lm, uniforms=_to_dev(u), nth=n / 2)
        torch.cuda.synchronize()
        assert _same(r.cpu().numpy(), st["r"])
        assert np.array_equal(B.cpu().numpy(), st["nxt"]) and _same(W.cpu().numpy(), st["w_out"])
        A, B = B, A


@pytest.mark.gpu
def test_pf_step_results_do_not_depend_on_earlier_calls(engine):
    """The scratch space grows and shrinks between forms, and the seven-launch form's ticket counters must be back
    at zero after every call: 2^21+1, 1025, 2^21+1 on one context equal fresh contexts bit for bit."""
    import torch

    def run(eng, n):
        px, pw, noise, lm = _inputs(n)
        a, b, nd = _to_dev(px), _to_dev(pw), _to_dev(noise)
        nxt = torch.empty_like(a)
        r = eng.pf_step(a, b, nxt, nd, lm, resample_seed=9, nth=float(n))
        torch.cuda.synchronize()
        return r.cpu().numpy(), nxt.cpu().numpy(), b.cpu().numpy()

    big, small = (1 << 21) + 1, 1025
    fresh = {}
    for n in (small, big):
        e = Engine(0)
        try:
            fresh[n] = run(e, n)
        finally:
            e.close()
    for n in (big, small, big, small):
        got = run(engine, n)
        assert all(_same(g, f) for g, f in zip(got, fresh[n])), n


# ---- large coordinates ------------------------------------------------------------------------------------------
def _far(n, centre, spread=0.05):
    """synth.pf_inputs moved rigidly to `centre` (with the landmarks) and shrunk to `spread` metres."""
    px, pw, noise = synth.pf_inputs(n)
    lm = synth.pf_landmarks(8).astype(np.float64)
    T = synth.PF_TRUTH
    for f in (0, 1):
        px[f] = (centre[f] + (px[f].astype(np.float64) - T[f]) * (spread / 0.2)).astype(F32)
        lm[:, 1 + f] += centre[f] - T[f]
    return px, pw, noise, lm.astype(F32)


@pytest.mark.gpu
@pytest.mark.parametrize("centre", [(1e4, -3e4), (1e5, 1e5)], ids=["1e4_-3e4", "1e5_1e5"])
@pytest.mark.parametrize("n", FORM_SIZES)
def test_pf_step_covariance_far_from_the_origin(engine, n, centre):
    """A cloud of 5 cm a few km from the origin: PEst must stay at float accuracy.  crb_pf_estimate (two-pass, centred
    on xEst) on the same predicted particles must pass the same gate and agree with crb_pf_step to it."""
    import torch
    px, pw, noise, lm = _far(n, centre)
    st = _check_step(engine, px, pw, noise, lm, nth=float(n), resample_seed=11)
    a, b = _to_dev(px), _to_dev(pw)
    engine.pf_predict_weight(a, b, _to_dev(noise), lm)
    xe, Pe, _ = engine.pf_estimate(a, b)
    torch.cuda.synchronize()
    ex, ew = a.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(ex, st["x"])
    _check_estimate(ex, ew, xe.astype(np.float64), Pe.astype(np.float64))
    P_step = st["r"][4:20].reshape(4, 4).T
    scale = np.sqrt(np.outer(np.diag(P_step), np.diag(P_step)))
    assert (np.abs(P_step - Pe) <= 1e-6 * scale).all()
