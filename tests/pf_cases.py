"""Inputs and float64 checks shared by the particle-filter tests (tests/test_pf_step_edges.py, tests/test_pf_fleet.py,
tests/test_pf_fleet_edges.py): the resampling draws in numpy, the estimate against the two-pass float64 covariance, the
resampled particles against the oracle, weight families, far-off clouds and the grouped fleet."""
import numpy as np

from cpprobotics_b200 import synth

F32 = np.float32
CHUNK = 2048                # weights per scan block of crb_pf_step


def philox_u12(seed, n):
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


def check_estimate(gx, gw, xe_got, P_got):
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


def assert_same_survivors(nxt, px2, gx, gw, U):
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


WEIGHT_KINDS = ["onehot_first", "onehot_last", "onehot_chunk_end", "onehot_chunk_start", "cap", "zero_run",
                "two_levels", "gamma", "all_zero"]


def weights(kind, n, seed=None, zero_runs=(5000, 9000)):
    """Weight families that synthetic likelihoods never produce: one-hot (first, last, middle, either side of crb_pf_step's
    100th scan block), the NP-1 cap, long zero runs, two levels 2^20 apart, heavy-tailed gamma(0.1) weights clipped to a
    narrow exponent span with a quarter of them dead, all zero, and all denormal.  seed defaults to the kind's place in
    WEIGHT_KINDS (0 for the others); zero_runs are the lengths of the two zero runs, at n/3 and 2n/3."""
    if seed is None:
        seed = WEIGHT_KINDS.index(kind) if kind in WEIGHT_KINDS else 0
    rng = np.random.default_rng(seed)
    w = np.zeros(n, np.float64)
    if kind.startswith("onehot"):
        w[{"onehot_first": 0, "onehot_last": n - 1, "onehot_mid": n // 2, "onehot_chunk_end": 100 * CHUNK - 1,
           "onehot_chunk_start": 100 * CHUNK}[kind]] = 1.0
    elif kind == "cap":             # all mass on NP-1, tiny weights elsewhere: the reference's cap (:139)
        w[:] = 2.0 ** -40
        w[-1] = 1.0
    elif kind == "zero_run":        # > 4096 zeros between normal weights: both non-staged window searches
        w[:] = 1.0 + np.floor(rng.random(n) * 64)
        a = n // 3
        w[a:a + zero_runs[0]] = 0.0
        w[2 * a:2 * a + zero_runs[1]] = 0.0
    elif kind == "two_levels":
        w[:] = np.where(rng.random(n) < 0.5, 1.0, 2.0 ** -20)
    elif kind == "gamma":           # heavy-tailed, a quarter dead, clipped to a span of 2^(29 - log2 n)
        g = rng.gamma(0.1, 1.0, n)
        span = 2.0 ** (29 - int(np.ceil(np.log2(n))))
        g = np.clip(g, g.max() / span, None)
        w = g.astype(F32).astype(np.float64)
        w[rng.integers(0, n, n // 4)] = 0.0
    elif kind == "denormal":        # every weight a float denormal (below 2^-126)
        w[:] = rng.integers(1, 1 << 23, n) * 2.0 ** -149
    elif kind == "all_zero":
        pass
    else:
        raise ValueError(kind)
    return w.astype(F32)


def far(n, centre, spread=0.05, seed=0xC0FFEE):
    """synth.pf_inputs moved rigidly to `centre` (with 8 landmarks) and shrunk to `spread` metres."""
    px, pw, noise = synth.pf_inputs(n, seed=seed)
    lm = synth.pf_landmarks(8).astype(np.float64)
    T = synth.PF_TRUTH
    for f in (0, 1):
        px[f] = (centre[f] + (px[f].astype(np.float64) - T[f]) * (spread / 0.2)).astype(F32)
        lm[:, 1 + f] += centre[f] - T[f]
    return px, pw, noise, lm.astype(F32)


def grouped_fleet(nr, npr, seed):
    """A fleet whose robots use one of three lists (0, 1 and 64 rows, shuffled over the robots) and one of two controls,
    so that each of the six (list, u) groups can be checked with ONE crb_pf_predict_weight_batched call."""
    f = synth.pf_fleet_inputs(nr, npr, seed=seed)
    rng = np.random.default_rng(seed)
    lm64 = synth.pf_landmarks(64, seed=seed)
    lists = [np.zeros((0, 3), np.float32), lm64[:1], lm64]
    z, z_off = synth.pack_obstacles(lists, 3)
    f["z"], f["z_off"], f["z_of"] = z, z_off, rng.integers(0, 3, nr).astype(np.int32)
    us = np.array([[1.0, 0.1], [0.7, -0.2]], np.float32)
    g = rng.integers(0, 2, nr)
    f["u"] = np.ascontiguousarray(us[g].T)
    f["ugroup"], f["lists"], f["us"] = g, lists, us
    return f
