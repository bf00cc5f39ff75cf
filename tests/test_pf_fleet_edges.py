"""crb_pf_step_many_batched at the edges of its CTA packing, draws, weight shapes, decision, parameters and poses.

The fleet kernel re-implements crb_pf_step's tail (weight sum, normalisation, moments, Neff, decision, scan and gather)
inside one warp per robot, so every case here holds a sample of robots to crb_pf_step's standard, fed with the GPU's
own state (check_robot):
  - the predicted particles are bitwise crb_pf_predict_weight_batched's with the robot's u, list and parameters;
  - result[20] is within np 2^-52 (relative) of the float64 sum of the raw weights, and the weights are
    float(w / float(result[20])) unless the robot resampled, then exactly float(1/np);
  - Neff is within one float ulp of oracle.pf_resample's from those weights, and result[22] is exactly Neff < nth;
  - px_next is oracle.pf_resample's bit for bit except at cumulative-weight ties, or a bit copy without resampling;
  - xEst is within one float ulp of the float64 weighted mean, PEst within 1e-6 sqrt(P_rr P_cc) of the two-pass
    float64 covariance, exactly symmetric with a non-negative diagonal (pf_cases.check_estimate)."""
import numpy as np
import pytest

import pf_cases as PC
from cpprobotics_b200 import _lib, synth
from oracle import oracle as O

F32 = np.float32
SMEM = 227 * 1024          # a CTA's dynamic shared memory on sm_90


def robots_per_cta(npr):
    """The host's packing: 8 warps per CTA, or as many 1280 + 24 np byte slices as 227 KB holds."""
    return min(8, SMEM // (1280 + 24 * npr))


def sample(nr, npr):
    """Every robot of a small fleet; otherwise the first, the last, each CTA's first and last warp and a stride."""
    if nr <= 64:
        return list(range(nr))
    w = robots_per_cta(npr)
    s = {0, nr - 1} | set(range(0, nr, max(1, nr // 64)))
    for c in range(0, nr, w):
        s |= {c, min(c + w, nr) - 1}
    return sorted(s)


def same(a, b):
    """Bitwise equal, any NaN equal to any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    v = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(v), b[~nb].view(v))


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _params(prm=None, u=None):
    from cpprobotics_b200 import pf_default_params
    p = _lib.PfParams.from_buffer_copy(prm) if prm is not None else pf_default_params()
    if u is not None:
        p.u[0], p.u[1] = float(u[0]), float(u[1])
    return p


def run(engine, f, npr, *, nth, prm=None, noise=True, uniforms=True, seed=11, resample_seed=13):
    import torch
    nr = f["u"].shape[1]
    px, pw = _dev(f["px"]), _dev(f["pw"])
    pxn = torch.full_like(px, 7.0)
    st = torch.full((nr,), -5, dtype=torch.int32, device="cuda:0")
    res = engine.pf_step_many(npr, px, pw, pxn, _dev(f["u"]), (_dev(f["z"]), _dev(f["z_off"])), _dev(f["z_of"]),
                              noise=_dev(f["noise"]) if noise else None, params=prm, seed=seed,
                              uniforms=_dev(f["uniforms"]) if uniforms else None, resample_seed=resample_seed,
                              nth=nth, status=st)
    torch.cuda.synchronize()
    return dict(px=px.cpu().numpy(), pw=pw.cpu().numpy(), pxn=pxn.cpu().numpy(), res=res.cpu().numpy(),
                st=st.cpu().numpy())


def single_filter(engine, f, npr, robots, prm=None, noise=True, seed=11):
    """The raw predicted particles and weights of `robots` from crb_pf_predict_weight_batched, one call per (list, u)
    group: on the group's columns with explicit noise, on the whole array with Philox draws (whose counter is the
    column)."""
    import torch
    gx = np.full_like(f["px"], np.nan)
    gw = np.full_like(f["pw"], np.nan)
    groups = {}
    for r in robots:
        groups.setdefault((int(f["z_of"][r]), F32(f["u"][0, r]).tobytes(), F32(f["u"][1, r]).tobytes()), []).append(r)
    for (ls, _, _), rs in groups.items():
        p = _params(prm, f["u"][:, rs[0]])
        rows = f["z"][f["z_off"][ls]:f["z_off"][ls + 1]]
        cols = np.concatenate([np.arange(r * npr, (r + 1) * npr) for r in rs])
        if noise:
            x, w = _dev(f["px"][:, cols]), _dev(f["pw"][cols])
            engine.pf_predict_weight(x, w, _dev(f["noise"][:, cols]), rows, params=p)
            torch.cuda.synchronize()
            gx[:, cols], gw[cols] = x.cpu().numpy(), w.cpu().numpy()
        else:
            x, w = _dev(f["px"]), _dev(f["pw"])
            engine.pf_predict_weight(x, w, None, rows, params=p, seed=seed)
            torch.cuda.synchronize()
            gx[:, cols], gw[cols] = x.cpu().numpy()[:, cols], w.cpu().numpy()[cols]
    return gx, gw


def check_robot(out, raw, npr, r, nth, U):
    """Robot r of a fleet run (`out`) against crb_pf_step's standard (module docstring), given the single-filter
    kernel's raw predict (`raw`) and the robot's uniforms U.  Returns its normalised weights and PEst ratio."""
    cols = slice(r * npr, (r + 1) * npr)
    res = out["res"][:, r]
    try:
        assert out["st"][r] == _lib.CRB_PF_FLEET_OK
        gx, rw = out["px"][:, cols], raw[1][cols]
        assert same(gx, raw[0][:, cols]), "predicted particles differ from crb_pf_predict_weight_batched"
        s = np.sum(rw, dtype=np.float64)
        assert abs(res[20] - s) <= npr * 2.0 ** -52 * abs(s), (res[20], s)
        with np.errstate(invalid="ignore", divide="ignore"):
            gw = rw / F32(res[20])
        U = np.asarray(U, np.float64)
        neff_o = O.pf_resample(gx, gw, U, nth=0.0)[3]
        neff = F32(res[21])
        assert (np.isnan(neff) and np.isnan(neff_o)) or abs(neff - F32(neff_o)) <= np.spacing(F32(neff_o)), \
            (neff, neff_o)
        assert res[22] == (1.0 if neff < F32(nth) else 0.0), (res[22], neff, nth)
        if res[22]:
            px2, pw2, did, _ = O.pf_resample(gx, gw, U, nth=np.inf)
            assert did
            PC.assert_same_survivors(out["pxn"][:, cols], px2, gx, gw, U)
            assert (out["pw"][cols] == F32(1.0 / npr)).all() and np.array_equal(out["pw"][cols], pw2)
        else:
            assert same(out["pxn"][:, cols], gx), "px_next is not a copy of px"
            assert same(out["pw"][cols], gw), "weights are not float(w / float(sum w))"
        ratio = PC.check_estimate(gx, gw, res[0:4], res[4:20].reshape(4, 4).T)
    except AssertionError as e:
        raise AssertionError(f"robot {r} (np {npr}): {e}") from e
    return gw, ratio


def check_fleet(engine, f, npr, *, nth, prm=None, noise=True, uniforms=True, seed=11, resample_seed=13,
                robots=None):
    """One fleet run with every robot of `robots` (default: sample()) checked; returns the run and the robots' weights."""
    nr = f["u"].shape[1]
    robots = sample(nr, npr) if robots is None else robots
    out = run(engine, f, npr, nth=nth, prm=prm, noise=noise, uniforms=uniforms, seed=seed,
              resample_seed=resample_seed)
    raw = single_filter(engine, f, npr, robots, prm=prm, noise=noise, seed=seed)
    U = f["uniforms"] if uniforms else PC.philox_u12(resample_seed, nr * npr)
    out["w"], out["ratio"], out["raw"] = {}, {}, raw
    for r in robots:
        out["w"][r], out["ratio"][r] = check_robot(out, raw, npr, r, nth, U[r * npr:(r + 1) * npr])
    return out


def empty_lists(f):
    """The fleet with no observations: every weight update is W * exp(0), so the weights are what the test sets."""
    f["z"], f["z_off"] = np.zeros((0, 3), F32), np.zeros(2, np.int64)
    f["z_of"] = np.zeros(f["u"].shape[1], np.int32)
    return f


def ragged(npr):
    """A robot count that leaves the last CTA partial (three robots where a CTA holds one)."""
    w = robots_per_cta(npr)
    return 3 if w == 1 else 3 * w + max(1, w // 2)


def test_helpers():
    assert [robots_per_cta(n) for n in (1, 1157, 1158, 2048, 4789, 4790, 8192)] == [8, 8, 7, 4, 2, 1, 1]
    assert ragged(100) == 28 and ragged(1158) == 24 and ragged(4790) == 3
    s = sample(1000, 100)
    assert {0, 7, 8, 15, 992, 999} <= set(s) and len(s) < 400
    assert sample(20, 8192) == list(range(20))
    w = PC.weights("denormal", 1000, seed=1)
    assert (w > 0).all() and (w < np.finfo(F32).tiny).all()
    assert PC.weights("onehot_mid", 101)[50] == 1.0
    assert same(np.array([np.nan, 1.0], F32), np.array([np.nan, 1.0], F32))
    assert not same(np.array([0.0], F32), np.array([-0.0], F32))


# ---- every np and CTA packing -------------------------------------------------------------------------------------
NPS = [1, 2, 3, 31, 32, 33, 63, 64, 65, 100, 1157, 1158, 2048, 4789, 4790, 8191, 8192]


@pytest.mark.gpu
@pytest.mark.parametrize("npr", NPS)
def test_every_np_and_cta_packing(engine, npr):
    """np on either side of the 32- and 64-particle rounds and of the 8, 7, 2 and 1 robots-per-CTA packings, with a
    partial last CTA, the six (list, u) groups and nth above every Neff: each robot resamples."""
    nr = ragged(npr)
    f = PC.grouped_fleet(nr, npr, seed=npr + 17)
    out = check_fleet(engine, f, npr, nth=2.0 * npr + 1.0)
    assert (out["res"][22] == 1.0).all()


# ---- Philox draws everywhere --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("npr", [33, 100, 1158, 4790])
def test_philox_noise_and_resampling(engine, npr):
    """noise = NULL and uniforms = NULL with seeds above 2^32: particle r*np + j draws Philox(seed, r*np + j) for its
    motion and Philox(resample_seed, r*np + j) for its resampleid, the whole array's draws.  nth is above every Neff,
    so each robot resamples."""
    nr = ragged(npr)
    f = PC.grouped_fleet(nr, npr, seed=npr + 23)
    out = check_fleet(engine, f, npr, nth=2.0 * npr + 1.0, noise=False, uniforms=False, seed=0x1_2345_6789,
                      resample_seed=0x9_8765_4321)
    assert (out["res"][22] == 1.0).all()


# ---- controlled weights -------------------------------------------------------------------------------------------
FLEET_KINDS = ["onehot_first", "onehot_last", "onehot_mid", "cap", "zero_run", "two_levels", "gamma", "all_zero",
               "denormal"]


@pytest.mark.gpu
@pytest.mark.parametrize("npr", [2, 100, 1024, 1158, 8192])
def test_controlled_weights(engine, npr):
    """Without observations each robot's weights are one of FLEET_KINDS, interleaved so that neighbours in a CTA
    differ.  One-hot robots take the hot particle or the np-1 cap in every slot, cap robots end on particle np-1,
    all-zero robots give NaN weights and estimate, no resampling and a bit copy, and leave their neighbours alone."""
    nr = 2 * len(FLEET_KINDS) + 1 if robots_per_cta(npr) > 1 else len(FLEET_KINDS)
    f = empty_lists(synth.pf_fleet_inputs(nr, npr, seed=npr + 5))
    kinds = [FLEET_KINDS[r % len(FLEET_KINDS)] for r in range(nr)]
    for r, k in enumerate(kinds):
        f["pw"][r * npr:(r + 1) * npr] = PC.weights(k, npr, seed=r, zero_runs=(npr // 4, npr // 5))
    out = check_fleet(engine, f, npr, nth=float(npr))
    for r, k in enumerate(kinds):
        cols = slice(r * npr, (r + 1) * npr)
        x, nxt, res = out["px"][:, cols], out["pxn"][:, cols], out["res"][:, r]
        assert same(out["raw"][1][cols], f["pw"][cols]), (r, k)
        if k == "all_zero":
            assert np.isnan(out["w"][r]).all() and np.isnan(res[:20]).all() and res[22] == 0.0
            assert same(nxt, x)
        elif k.startswith("onehot") and npr > 1:
            hot = int(np.argmax(f["pw"][cols]))
            assert res[22] == 1.0
            assert ((nxt == x[:, [hot]]).all(axis=0) | (nxt == x[:, [-1]]).all(axis=0)).all(), (r, k)
        elif k == "cap" and npr > 1:
            assert res[22] == 1.0 and (nxt[:, -2:] == x[:, [-1]]).all(), (r, k)


# ---- the decision boundary ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("npr", [64, 100, 1024])
def test_decision_boundary(engine, npr):
    """Robot m has k = 2^m equal weights and the rest zero, so its Neff is exactly k: with nth = k no robot with that k
    resamples, with nth = nextafter(k, inf) those robots do; robots with fewer (more) particles always (never) do."""
    ks = [1 << m for m in range(int(np.log2(npr)) + 1)]
    nr = len(ks)
    f = empty_lists(synth.pf_fleet_inputs(nr, npr, seed=npr + 3))
    rng = np.random.default_rng(npr)
    for r, k in enumerate(ks):
        w = np.zeros(npr, F32)
        w[np.sort(rng.choice(npr, k, replace=False))] = 1.0
        f["pw"][r * npr:(r + 1) * npr] = w
    for k in ks:
        for nth in (float(k), float(np.nextafter(F32(k), F32(np.inf)))):
            out = check_fleet(engine, f, npr, nth=nth)
            assert out["res"][21].tolist() == [float(k2) for k2 in ks]
            assert out["res"][22].tolist() == [1.0 if k2 < F32(nth) else 0.0 for k2 in ks], (k, nth)


# ---- non-default parameters ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("npr", [100, 1024])
def test_non_default_params(engine, npr):
    """dt, Q, Rsim and pi away from the demo's, with 0-, 1- and 64-row lists (the host rebuilds the -k ln(pre) table
    for every row count from them) and nth = 0.6 np."""
    prm = _params()
    prm.dt, prm.pi, prm.Q = 0.05, 3.14, 0.3 ** 2
    prm.rsim_diag[0], prm.rsim_diag[1] = 0.5, 0.2
    nr = ragged(npr)
    f = PC.grouped_fleet(nr, npr, seed=npr + 29)
    out = check_fleet(engine, f, npr, nth=0.6 * npr, prm=prm)
    dflt = run(engine, f, npr, nth=0.6 * npr)
    assert not np.array_equal(out["px"], dflt["px"])     # the parameters reach the kernel
    assert out["res"][22].any()


# ---- far-off poses ------------------------------------------------------------------------------------------------
FAR_KINDS = ["cloud_1e4_-3e4", "cloud_1e5_1e5", "outlier_w0", "outlier_w2^-40", "two_clusters"]


def far_fleet(nr, npr):
    """Robot r is FAR_KINDS[r % 5]: a 5 cm cloud at (1e4, -3e4) or (1e5, 1e5) with landmarks moved along; a 5 cm cloud
    near the origin whose particle 0 sits 10 km away with raw weight 0 or 2^-40; or two equal-weight 5 cm clusters 1 km
    apart.  The last three see no landmarks, so their weights are what is set here."""
    n = nr * npr
    f = synth.pf_fleet_inputs(nr, npr, seed=npr + 31)
    pa, wa, na, la = PC.far(n, (1e4, -3e4))
    pb, wb, nb, lb = PC.far(n, (1e5, 1e5))
    pc, wc, nc, _ = PC.far(n, synth.PF_TRUTH[:2])
    f["z"], f["z_off"] = synth.pack_obstacles([np.zeros((0, 3), F32), la, lb], 3)
    f["z_of"] = np.zeros(nr, np.int32)
    f["u"][0], f["u"][1] = 1.0, 0.1
    for r in range(nr):
        k, c = FAR_KINDS[r % 5], slice(r * npr, (r + 1) * npr)
        src = {"cloud_1e4_-3e4": (pa, wa, na), "cloud_1e5_1e5": (pb, wb, nb)}.get(k, (pc, wc, nc))
        f["px"][:, c], f["pw"][c], f["noise"][:, c] = src[0][:, c], src[1][c], src[2][:, c]
        if k.startswith("cloud"):
            f["z_of"][r] = 1 + FAR_KINDS.index(k)
        elif k.startswith("outlier"):
            f["px"][0, r * npr] += F32(1e4)
            f["pw"][r * npr] = 0.0 if k == "outlier_w0" else 2.0 ** -40
        else:
            f["px"][0, r * npr + npr // 2:(r + 1) * npr] += F32(1e3)
            f["pw"][c] = 1.0
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("npr", [100, 1024, 8192])
def test_far_off_poses(engine, npr):
    """PEst stays within 1e-6 sqrt(P_rr P_cc) of the two-pass covariance whatever the distance from the origin and from
    particle 0: the moments are centred on the heaviest particle, which lies within sqrt(np) standard deviations of
    the mean."""
    nr = 11 if robots_per_cta(npr) > 1 else 5
    f = far_fleet(nr, npr)
    out = check_fleet(engine, f, npr, nth=float(npr))
    for r in range(nr):
        if FAR_KINDS[r % 5] == "two_clusters":    # the covariance sees both clusters
            P = out["res"][4:20, r].reshape(4, 4).T
            assert 2.4e5 < P[0, 0] < 2.6e5, P[0, 0]


# ---- independence of the launch shape -----------------------------------------------------------------------------
def sub_fleet(f, npr, lo, hi):
    cols = slice(lo * npr, hi * npr)
    g = dict(f)
    g["px"], g["pw"], g["noise"] = f["px"][:, cols], f["pw"][cols], f["noise"][:, cols]
    g["uniforms"], g["u"], g["z_of"] = f["uniforms"][cols], f["u"][:, lo:hi], f["z_of"][lo:hi]
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("npr", [100, 1158])
def test_outputs_do_not_depend_on_the_launch_shape(engine, npr):
    """With explicit noise and uniforms a robot's px, pw, px_next, result column and status are the same bits run alone,
    in a sub-fleet that starts at an odd robot (so at another warp of another CTA), and in the whole fleet."""
    nr = ragged(npr) + robots_per_cta(npr)
    f = PC.grouped_fleet(nr, npr, seed=npr + 37)
    nth = 0.75 * npr
    full = check_fleet(engine, f, npr, nth=nth)
    assert full["res"][22].any()
    lo, hi = 5, nr - 2

    def agrees(got, r_got, r):
        cg, cf = slice(r_got * npr, (r_got + 1) * npr), slice(r * npr, (r + 1) * npr)
        return (same(got["px"][:, cg], full["px"][:, cf]) and same(got["pw"][cg], full["pw"][cf])
                and same(got["pxn"][:, cg], full["pxn"][:, cf]) and same(got["res"][:, r_got], full["res"][:, r])
                and got["st"][r_got] == full["st"][r])

    part = run(engine, sub_fleet(f, npr, lo, hi), npr, nth=nth)
    for r in range(lo, hi):
        assert agrees(part, r - lo, r), r
    for r in (0, 1, lo, robots_per_cta(npr), nr - 1):
        alone = run(engine, sub_fleet(f, npr, r, r + 1), npr, nth=nth)
        assert agrees(alone, 0, r), r


# ---- element offsets past 2^31 ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_offsets_past_2_31(engine):
    """np = 100 and n_robots np just above 2^29: field 3 of px / px_next ends past element 2^31, and the last robots'
    field-3 columns lie entirely past it.  The fleet is a 64-robot block tiled on the device; every sampled robot r must
    be robot r mod 64 of the block run alone, bit for bit.  About 27 GB of device memory."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 32 * 2 ** 30:
        pytest.skip(f"needs 32 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    npr, nb = 100, 64
    nr = (1 << 29) // npr + 1
    N, B = nr * npr, nb * npr
    assert 4 * N > 2 ** 31 and 3 * N + (nr - 1) * npr >= 2 ** 31 and nr % robots_per_cta(npr) != 0
    blk = PC.grouped_fleet(nb, npr, seed=41)
    small = check_fleet(engine, blk, npr, nth=0.75 * npr)
    assert small["res"][22].any() and not small["res"][22].all()

    def tile(a, width):   # [rows, width] block -> [rows, total] on the device, the block repeated along the columns
        a = _dev(a).reshape(-1, width)
        total = N if width == B else nr
        out = torch.empty(a.shape[0], total, dtype=a.dtype, device="cuda:0")
        full = total // width
        out[:, :full * width].view(a.shape[0], full, width).copy_(a[:, None, :].expand(-1, full, -1))
        out[:, full * width:] = a[:, :total - full * width]
        return out

    px, pw = tile(blk["px"], B), tile(blk["pw"], B).reshape(N)
    noise, uni = tile(blk["noise"], B), tile(blk["uniforms"], B).reshape(N)
    u, z_of = tile(blk["u"], nb), tile(blk["z_of"], nb).reshape(nr)
    pxn = torch.empty_like(px)
    res = torch.empty(_lib.CRB_PF_RESULT_LEN, nr, dtype=torch.float64, device="cuda:0")
    st = torch.full((nr,), -5, dtype=torch.int32, device="cuda:0")
    engine.pf_step_many(npr, px, pw, pxn, u, (_dev(blk["z"]), _dev(blk["z_off"])), z_of, noise=noise,
                        uniforms=uni, nth=0.75 * npr, result=res, status=st)
    torch.cuda.synchronize()
    first_past = (2 ** 31 - 3 * N) // npr            # the first robot whose field-3 columns reach past 2^31
    rs = sorted(set(range(0, nr, nr // 200)) | set(range(64)) | set(range(first_past - 16, nr)))
    idx = torch.tensor(rs, device="cuda:0")
    cols = (idx[:, None] * npr + torch.arange(npr, device="cuda:0")).reshape(-1)
    got = dict(px=px[:, cols].cpu().numpy(), pw=pw[cols].cpu().numpy(), pxn=pxn[:, cols].cpu().numpy(),
               res=res[:, idx].cpu().numpy(), st=st[idx].cpu().numpy())
    del px, pw, pxn, noise, uni, res
    torch.cuda.empty_cache()
    for i, r in enumerate(rs):
        c, b = slice(i * npr, (i + 1) * npr), slice((r % nb) * npr, (r % nb + 1) * npr)
        assert same(got["px"][:, c], small["px"][:, b]) and same(got["pw"][c], small["pw"][b]), r
        assert same(got["pxn"][:, c], small["pxn"][:, b]) and same(got["res"][:, i], small["res"][:, r % nb]), r
        assert got["st"][i] == small["st"][r % nb], r
