"""A particle filter per robot: crb_pf_step_many_batched runs pf_localization + resampling for n_robots independent
filters of np particles in one launch, each with its own control u and its own observation list z.

Each robot's per-particle arithmetic must be bitwise crb_pf_predict_weight_batched's on that robot's particles with its u
and list, and its tail must meet crb_pf_step's standard on that robot alone; the checker composed robot by robot
(oracle/pf_fleet.py) follows the closed loop.
CPU: argument validation without a device, synth.pf_fleet_inputs, the composed checker on a one-robot fleet, the
compiler report, the SASS pin of the single-filter kernels and the C++ fleet program (tests/cpp/pf_fleet_ref_api.cpp)
compiling.
H100 (-m gpu): per-particle bits at np 1 to CRB_PF_FLEET_MAX_NP and up to 65536 robots with 0-, 1- and 64-row lists,
Philox mode, crb_pf_step per robot, isolation of bad lists / NaN / zero weights, NULL status, n_robots = 0, graph
capture, a 50-tick closed loop against the checker and the C++ fleet program against the checker."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import pf_cases as PC
from cpprobotics_b200 import _lib, synth
from oracle import oracle as OO
from oracle import pf_fleet as PFF
from toolchain import build_ref_program, kernel_sass_hashes, ptxas_kernels

INV = -1
CAP = _lib.CRB_PF_FLEET_MAX_NP


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(bits(a[~na]), bits(b[~nb]))


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is refused with CRB_ERR_INVALID_ARG before any device work; a valid call says
    CRB_ERR_NO_DEVICE on a machine without a GPU."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d, d2 = C.c_void_p(256), C.c_void_p(512)
    prm = _lib.PfParams()
    L.crb_pf_default_params(C.byref(prm))

    def call(**over):
        a = dict(dict(ctx=ctx, nr=5, np_=100, px=d, pw=d, pxn=d2, u=d, noise=None, z=d, rows=40, off=d, ns=3, of=d,
                      prm=C.byref(prm), res=d, st=None), **over)
        return L.crb_pf_step_many_batched(a["ctx"], a["nr"], a["np_"], a["px"], a["pw"], a["pxn"], a["u"], a["noise"],
                                          1, a["z"], a["rows"], a["off"], a["ns"], a["of"], a["prm"], None, 2,
                                          C.c_float(50.0), a["res"], a["st"])

    for kw in (dict(ctx=None), dict(prm=None), dict(np_=0), dict(np_=CAP + 1), dict(np_=-3), dict(nr=-1),
               dict(ns=0), dict(ns=-1), dict(rows=-1), dict(u=None), dict(off=None), dict(of=None), dict(z=None),
               dict(px=None), dict(pw=None), dict(pxn=None), dict(res=None), dict(pxn=d),
               dict(nr=1 << 40, np_=2)):
        assert call(**kw) == INV, kw
    for kw in (dict(np_=0), dict(prm=None), dict(ns=0)):
        assert call(nr=0, **kw) == INV, kw
    if not torch.cuda.is_available():
        nd = _lib.CRB_ERR_NO_DEVICE
        assert call() == nd and call(z=None, rows=0) == nd and call(np_=CAP) == nd and call(np_=1) == nd
        assert call(nr=0, px=None, pw=None, pxn=None, u=None, z=None, off=None, of=None, res=None) == nd
        assert b"no CPU fallback" in L.crb_last_error_string()


def test_fleet_inputs_follow_the_demo():
    f = synth.pf_fleet_inputs(300, 10, seed=5)
    g = synth.pf_fleet_inputs(300, 10, seed=5)
    assert all(np.array_equal(f[k], g[k]) for k in f)
    assert f["px"].shape == (4, 3000) and f["pw"].shape == (3000,) and f["u"].shape == (2, 300)
    assert f["noise"].shape == (2, 3000) and f["uniforms"].shape == (3000,)
    assert ((f["uniforms"] >= 1) & (f["uniforms"] < 2)).all()
    assert f["z_off"].shape == (301,) and f["z_of"].dtype == np.int32 and f["z"].shape == (f["z_off"][-1], 3)
    tags = np.asarray(synth.PF_RFID, np.float32)
    counts = np.diff(f["z_off"])
    assert counts.max() <= len(tags) and len(set(counts.tolist())) > 1   # robots see different tags
    for r in (0, 17, 299):
        rows = f["z"][f["z_off"][r]:f["z_off"][r + 1]]
        d = np.hypot(f["truth"][0, r] - tags[:, 0], f["truth"][1, r] - tags[:, 1])
        seen = tags[d <= synth.PF_MAX_RANGE]
        assert np.array_equal(rows[:, 1:], seen)
        assert np.abs(rows[:, 0] - d[d <= synth.PF_MAX_RANGE]).max(initial=0) < 0.25
    # every robot's cloud sits around its own true pose
    c = f["px"][:2].reshape(2, 300, 10).mean(axis=2)
    assert np.abs(c - f["truth"][:2]).max() < 0.5


def test_composed_checker_on_one_robot_is_the_checker():
    f = synth.pf_fleet_inputs(1, 100, seed=9)
    rows = f["z"]
    c = dict(OO.pf_constants())
    c["u"] = f["u"][:, 0]
    pxp, pwr = OO.pf_predict_weight_batched(f["px"], f["pw"], f["noise"], rows, consts=c)
    pwn, xe, pe, sw = OO.pf_estimate(pxp, pwr)
    pxn, pwo, did, neff = OO.pf_resample(pxp, pwn, f["uniforms"].astype(np.float64), 50)
    px, pw, pxnext, res, st = PFF.step_many(100, f["px"], f["pw"], f["u"], f["z"], f["z_off"], f["z_of"], f["noise"],
                                            f["uniforms"])
    assert st.tolist() == [PFF.FLEET_OK]
    assert same(px, pxp) and same(pw, pwo if did else pwn) and same(pxnext, pxn if did else pxp)
    assert same(res[:4, 0].astype(np.float32), xe) and res[20, 0] == sw and res[22, 0] == float(did)
    assert same(res[4:20, 0].reshape(4, 4).T.astype(np.float32), pe)
    # a bad reference leaves the robot alone
    px2, pw2, pxn2, res2, st2 = PFF.step_many(100, f["px"], f["pw"], f["u"], f["z"], f["z_off"], np.array([3], np.int32),
                                              f["noise"], f["uniforms"])
    assert st2.tolist() == [PFF.FLEET_BAD_OBSERVATIONS] and np.isnan(res2).all()
    assert same(px2, f["px"]) and same(pw2, f["pw"]) and same(pxn2, f["px"])


# sha256 of each single-filter PF kernel's SASS (cuobjdump -sass, NVCC_FLAGS, CUDA 12.9) as they were before the fleet
# filter existed: moving their shared code into crb_pf_common.cuh must not change one instruction
SINGLE_FILTER_SASS = {
    "_Z18crb_pf_sumw_kernellPKfPd":
        "4bf1f5bf1a08cf8aa48d5d700c7a56bb6a934b871ffdc82d573cd680ae602ccd",
    "_Z19crb_pf_pivot_kernellPKfiPd":
        "0bf10c3045213e9e34f0644cd2a730533681374c966b9cd83e34b011bf9dd4b6",
    "_Z19crb_pf_scan1_kernellPKfPdS1_":
        "61a435b7b9abca8addac8470fefa5e2946afefc2cfd44e50466b1c8c193667ad",
    "_Z19crb_pf_scan2_kerneliPd":
        "2a5a8d2e241d5f2ae07053ea46c2552651ef82d580633ffb63a6340ef37409ce",
    "_Z19crb_pf_scan3_kernellPKdS0_Pf":
        "af139e1e104927e8526e0a46dedd1428efb2348469259accd5c6aff996e40e0b",
    "_Z19crb_pf_sumsq_kernellPKfPd":
        "fb88322afe7b95ccdee7daba6a670e8582cb21a5d16f9927494a317a62b7a6b0",
    "_Z20crb_pf_scan1n_kernellPfPKdPdS2_S2_":
        "f1b2d0e0445443ff82df8ea1d1c1a0c2b5206f02a4d0e48a4009129ae992060f",
    "_Z20crb_pf_scan2n_kerneliPdPKdfS_":
        "a53ceefcc3540bf7cdbdd091490471130c184192bd1e4506e0721aac0ac5a553",
    "_Z21crb_pf_combine_kernelILi10EEvPKdPd":
        "e27bbff11d13c8952e7a827844269f50ab9112a2316d6c39cd793623640de3c8",
    "_Z21crb_pf_combine_kernelILi15EEvPKdPd":
        "ccddda5b70a66b70285eadece1dd8f86a0463eb189bb911ba6adde95f910d259",
    "_Z21crb_pf_combine_kernelILi1EEvPKdPd":
        "a910987bf994a71442dada5939b1ed454f4c8f6abbaade6fc21def2a640aef4e",
    "_Z21crb_pf_combine_kernelILi5EEvPKdPd":
        "ad17a9e853ce81f3c78c0974b9baaa37d8a90f6a148fc7d124eb88d14b7d9d18",
    "_Z21crb_pf_gather2_kerneliPKfPKdS2_S2_ifS0_jjPfS3_PdS2_d":
        "2579ac9b39acb76ceffe8126d0bc8f901477b31149d92bf29c9a3eca1e5f5742",
    "_Z21crb_pf_moment1_kernellPKfS0_Pd":
        "e64e73ba36e542a573fdcc9ac521cf162112c32884df58cce09f7cb93e146f52",
    "_Z21crb_pf_moment2_kernellPKfPfPKdPd":
        "5180225f8228710b0112a83c34b8f781fefa54bbe757c08a435e1fdce9b05a2f",
    "_Z21crb_pf_moments_kernellPKfS0_PKdPd":
        "0db8eea57ab8b699274e01bf18ecf28918c85d7f972e77337dfe885e9c58065a",
    "_Z21crb_pf_scan1n3_kernellPKfPfPKdiPdS4_S4_S4_S4_i":
        "53f27a31e221745314d5c97fdacff9de32f86f4b0fa81a5361f32cd1a8bdf2e0",
    "_Z22crb_pf_finalize_kernellPKfPKdS2_Pd":
        "3b4335178e19e5a580b384c250a6cc99d82824cde7eb653001ccfed7aa3b30b0",
    "_Z29crb_pf_resample_gather_kernelILb0ELi256EEvlPKf8WcumViewIXT_EES1_jjPfS4_PKd":
        "ac634078ea45ec3ee864639bd229a692a6bc2cb40e311337887405a0e768ada5",
    "_Z29crb_pf_resample_gather_kernelILb1ELi256EEvlPKf8WcumViewIXT_EES1_jjPfS4_PKd":
        "49b6c00a36e8bf4967f12dea65f326bd5cf68f2b426db197876235bcf8ddb409",
    "_Z33crb_pf_predict_weight_lean_kernelILi128ELi12EEvjllPfS0_PKf6PfArgs":
        "64e4114e1c4721e27c269809a828b8cf577f41d70e181b5fc3d04f8749a02680",
    "_Z33crb_pf_predict_weight_sumw_kernelILi128ELi12EEvjllPfS0_PKf6PfArgsPd":
        "c850ac444d97460105384372e67517fd6b7127e50e345f5060956bf57016079a",
    "_Z34crb_pf_predict_weight_fused_kernellllPfS_PKf6PfArgs":
        "e31097ed357c6b53de4cd1b9216955c4f36d81cc72eeee7159443bc5bd50f2e7",
    "_Z35crb_pf_predict_weight_fused2_kernelILi128ELi12EEvlllPfS0_PKf6PfArgs":
        "d67d76910afaba33c608aeaf3db25e76ee88f1f22416cca9adcb5a14e3e2c36e",
}


def test_fleet_kernel_does_not_spill():
    """No spill.  The only stack frame is the 32 bytes of CUDA's sincosf large-argument reduction, reached for
    |yaw| > 1e5 on the CRB_PF_TRIG=0 path, which every single-filter predict kernel carries too."""
    kernels = ptxas_kernels("crb_pf_fleet.cu")
    assert list(kernels) == ["_Z19crb_pf_fleet_kernelPfS_S_PKfS1_S1_PKlPKiS1_PdPi11PfFleetArgs"], list(kernels)
    f = next(iter(kernels.values()))
    assert (f.spill_stores, f.spill_loads) == (0, 0) and f.stack <= 32 and f.registers <= 96, f
    lean = [f for k, f in ptxas_kernels("crb_pf.cu").items() if "lean_kernel" in k]
    assert lean and all(f.stack == 32 for f in lean), lean


def test_single_filter_kernels_keep_their_machine_code():
    assert kernel_sass_hashes("crb_pf.cu") == SINGLE_FILTER_SASS


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "pf_fleet_ref_api.cpp")


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    return t.cpu().numpy()


def run_fleet(engine, f, npr, nth=None, noise=True, uniforms=True, status=True):
    import torch
    px, pw = _dev(f["px"]), _dev(f["pw"])
    pxn = torch.full_like(px, 7.0)
    st = torch.full((f["u"].shape[1],), -5, dtype=torch.int32, device="cuda:0") if status else None
    res = engine.pf_step_many(npr, px, pw, pxn, _dev(f["u"]), (_dev(f["z"]), _dev(f["z_off"])), _dev(f["z_of"]),
                              noise=_dev(f["noise"]) if noise else None, seed=11,
                              uniforms=_dev(f["uniforms"]) if uniforms else None, resample_seed=13, nth=nth, status=st)
    torch.cuda.synchronize()
    return _host(px), _host(pw), _host(pxn), _host(res), (_host(st) if status else None)


# (np, n_robots); 1157 is the last np with 8 robots per CTA, 1158 the first with 7, 4789 the last with 2 and 4790 the
# first with 1, each with a partial last CTA where it can have one
CELLS = [(1, 65536), (2, 4096), (31, 7), (100, 65536), (100, 1), (257, 4096), (1024, 7), (1024, 4096), (1157, 13),
         (1158, 13), (4789, 5), (4790, 3), (CAP, 1), (CAP, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("npr,nr", CELLS)
def test_particles_are_the_single_filter_kernel_bitwise(engine, npr, nr):
    """With explicit noise and no resampling (nth = 0), each robot's predicted particles are bitwise
    crb_pf_predict_weight_batched's with its u and list, and its weights are those raw weights divided by the float of
    its own weight sum (result[20])."""
    import torch
    from cpprobotics_b200 import pf_default_params
    f = PC.grouped_fleet(nr, npr, seed=npr * 7 + nr)
    px, pw, pxn, res, st = run_fleet(engine, f, npr, nth=0.0)
    assert (st == _lib.CRB_PF_FLEET_OK).all()
    assert same(pxn, px) and (res[22] == 0).all()
    own = np.repeat(np.arange(nr), npr)
    key = f["z_of"][own] * 2 + f["ugroup"][own]
    for k in np.unique(key):
        cols = np.flatnonzero(key == k)
        ls, ug = divmod(int(k), 2)
        prm = pf_default_params()
        prm.u[0], prm.u[1] = float(f["us"][ug, 0]), float(f["us"][ug, 1])
        gx, gw = _dev(f["px"][:, cols]), _dev(f["pw"][cols])
        engine.pf_predict_weight(gx, gw, _dev(f["noise"][:, cols]), f["lists"][ls], params=prm)
        torch.cuda.synchronize()
        assert same(px[:, cols], _host(gx)), (ls, ug)
        sw = res[20, own[cols]].astype(np.float32)
        assert same(pw[cols], (_host(gw) / sw).astype(np.float32)), (ls, ug)


@pytest.mark.gpu
def test_philox_mode_is_the_whole_array_draws(engine):
    import torch
    from cpprobotics_b200 import pf_default_params
    nr, npr = 4096, 100
    f = synth.pf_fleet_inputs(nr, npr, seed=3)
    f["z_of"][:] = 5
    f["u"][0], f["u"][1] = 0.9, 0.05
    prm = pf_default_params()
    prm.u[0], prm.u[1] = 0.9, 0.05
    px, pw, _, res, _ = run_fleet(engine, f, npr, nth=0.0, noise=False)
    gx, gw = _dev(f["px"]), _dev(f["pw"])
    engine.pf_predict_weight(gx, gw, None, f["z"][f["z_off"][5]:f["z_off"][6]], params=prm, seed=11)
    torch.cuda.synchronize()
    assert same(px, _host(gx))
    assert same(pw, (_host(gw) / np.repeat(res[20].astype(np.float32), npr)).astype(np.float32))


def _ulp(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("npr", [100, 1024])
def test_each_robot_is_pf_step_alone(engine, npr):
    """A sample of robots against crb_pf_step run on each robot alone with the same noise and uniforms: once with
    nth = 0 (no robot resamples) and once with nth = 0.75 np (nearly every robot does)."""
    nr = 512
    f = synth.pf_fleet_inputs(nr, npr, seed=npr)
    keep = run_fleet(engine, f, npr, nth=0.0)
    for nth in (0.0, 0.75 * npr):
        check_against_pf_step(engine, f, nr, npr, nth, keep)


def resample_ids(npr, uniforms):
    """resampleid_j = j/NP + U_j/NP as the kernels form it (both quotients correctly rounded in double, j/NP narrowed to
    float first), with the running maximum over the previous particle."""
    j = np.arange(npr, dtype=np.float64)
    base = (j / npr).astype(np.float32).astype(np.float64)
    rid = (base + uniforms.astype(np.float64) / npr).astype(np.float32)
    rid[1:] = np.maximum(rid[1:], rid[:-1])
    return rid


def column_of(px, v):
    """Index of the particle (column of px [4, np]) equal to v [4]."""
    k = np.flatnonzero((px == v[:, None]).all(axis=0))
    assert len(k) >= 1
    return int(k[0])


def check_against_pf_step(engine, f, nr, npr, nth, keep):
    import torch
    from cpprobotics_b200 import pf_default_params
    px, pw, pxn, res, st = run_fleet(engine, f, npr, nth=nth)
    pw0, res0 = keep[1], keep[3]           # the normalised weights and the estimate, from the nth = 0 run
    assert (st == 0).all()
    n_bit = n_res = n_tie = 0
    for r in range(0, nr, 16):
        cols = slice(r * npr, (r + 1) * npr)
        prm = pf_default_params()
        prm.u[0], prm.u[1] = float(f["u"][0, r]), float(f["u"][1, r])
        gx, gw, gn = _dev(f["px"][:, cols]), _dev(f["pw"][cols]), torch.zeros(4, npr, device="cuda:0")
        one = engine.pf_step(gx, gw, gn, _dev(f["noise"][:, cols]), f["z"][f["z_off"][r]:f["z_off"][r + 1]],
                             params=prm, uniforms=_dev(f["uniforms"][cols]), nth=nth)
        torch.cuda.synchronize()
        one = _host(one)
        assert same(px[:, cols], _host(gx))                                     # predicted particles
        assert res[22, r] == float(np.float32(res[21, r]) < np.float32(nth))   # the decision is Neff < nth
        rest = [k for k in range(24) if k != 22]
        assert same(res[rest, r], res0[rest, r])                                # the estimate does not depend on nth
        if np.float32(res[20, r]) == np.float32(one[20]):
            n_bit += 1
            assert same(pw[cols], _host(gw)) and res[22, r] == one[22]
            # px_next: bitwise except where a resampleid sits on a cumulative weight whose float rounding the two
            # summation orders (warp scan here, block scan in crb_pf_step) put on different sides of it
            rid = resample_ids(npr, f["uniforms"][cols])
            cum = np.cumsum(pw0[cols].astype(np.float64)).astype(np.float32)
            mine, theirs, pred = pxn[:, cols], _host(gn), px[:, cols]
            for jj in np.flatnonzero((mine != theirs).any(axis=0)):
                assert res[22, r] == 1.0
                a, b = column_of(pred, mine[:, jj]), column_of(pred, theirs[:, jj])
                lo = min(a, b)
                assert abs(float(cum[lo]) - float(rid[jj])) <= 2 * _ulp(rid[jj]), (r, jj, a, b, cum[lo], rid[jj])
                assert (np.abs(cum[lo:max(a, b)].astype(np.float64) - cum[lo]) <= 2 * _ulp(rid[jj])).all()
                n_tie += 1
        n_res += int(res[22, r])
        # xEst within one ulp of the float64 mean with the robot's normalised weights; PEst to 1e-6 sqrt(P_rr P_cc)
        w = pw0[cols].astype(np.float64)
        x = px[:, cols].astype(np.float64)
        m = (x * w).sum(axis=1)
        assert (np.abs(res[:4, r] - m) <= _ulp(m)).all(), (res[:4, r], m)
        d = x - res[:4, r][:, None]
        cov = (w * d) @ d.T
        P = res[4:20, r].reshape(4, 4).T
        tol = 1e-6 * np.sqrt(np.outer(np.diag(cov), np.diag(cov))) + 1e-30
        assert (np.abs(P - cov) <= tol).all() and np.array_equal(P, P.T) and (np.diag(P) >= 0).all()
    assert n_bit >= 16 and (n_res > 0 if nth > 0 else n_res == 0)
    assert n_tie <= n_bit   # ties are rare: at most about one per robot


@pytest.mark.gpu
def test_bad_lists_nan_and_zero_weights_stay_with_their_robot(engine):
    nr, npr = 64, 100
    f = synth.pf_fleet_inputs(nr, npr, seed=21)
    base = run_fleet(engine, f, npr)
    # bad references: an index past n_sets, a negative one, a list of 65 rows, an offset past n_rows
    g = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in f.items()}
    long = np.tile(g["z"][:1], (65, 1))
    g["z"] = np.concatenate([g["z"], long])
    n0 = g["z_off"][-1]
    g["z_off"] = np.concatenate([g["z_off"], [n0 + 65, n0 + 10 ** 6]]).astype(np.int64)
    # lists nr: the 65-row list; nr + 1: rows past n_rows
    bad = {3: nr + 2, 10: -1, 20: nr, 30: nr + 1}
    for r, s in bad.items():
        g["z_of"][r] = s
    px, pw, pxn, res, st = run_fleet(engine, g, npr)
    for r in range(nr):
        cols = slice(r * npr, (r + 1) * npr)
        if r in bad:
            assert st[r] == _lib.CRB_PF_FLEET_BAD_OBSERVATIONS and np.isnan(res[:, r]).all()
            assert same(px[:, cols], f["px"][:, cols]) and same(pw[cols], f["pw"][cols]) and (pxn[:, cols] == 7).all()
        else:
            assert st[r] == 0
            assert same(px[:, cols], base[0][:, cols]) and same(pw[cols], base[1][cols])
            assert same(pxn[:, cols], base[2][:, cols]) and same(res[:, r], base[3][:, r])
    # a NaN in one list: that robot's particles are the single-filter kernel's with that list (whose clamped exponent
    # keeps the weights finite); zero weights in another robot: NaN weights and estimate, as crb_pf_step gives
    import torch
    from cpprobotics_b200 import pf_default_params
    h = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in f.items()}
    rn = int(np.flatnonzero(np.diff(h["z_off"]) > 0)[0])   # a robot that sees tags
    assert rn != 9
    h["z"][h["z_off"][rn], 0] = np.nan
    h["pw"][9 * npr:10 * npr] = 0.0
    px, pw, pxn, res, st = run_fleet(engine, h, npr)
    assert (st == 0).all()
    prm = pf_default_params()
    prm.u[0], prm.u[1] = float(h["u"][0, rn]), float(h["u"][1, rn])
    cols = slice(rn * npr, (rn + 1) * npr)
    gx, gw = _dev(h["px"][:, cols]), _dev(h["pw"][cols])
    engine.pf_predict_weight(gx, gw, _dev(h["noise"][:, cols]), h["z"][h["z_off"][rn]:h["z_off"][rn + 1]], params=prm)
    torch.cuda.synchronize()
    assert same(px[:, cols], _host(gx)) and res[20, rn] != base[3][20, rn]   # its weights changed
    cols = slice(9 * npr, 10 * npr)
    assert np.isnan(pw[cols]).all() and np.isnan(res[:20, 9]).all() and res[20, 9] == 0.0
    for r in range(nr):
        cols = slice(r * npr, (r + 1) * npr)
        if r in (rn, 9):
            continue
        else:
            assert same(px[:, cols], base[0][:, cols]) and same(pw[cols], base[1][cols])
            assert same(pxn[:, cols], base[2][:, cols]) and same(res[:, r], base[3][:, r])


@pytest.mark.gpu
def test_null_status_empty_fleet_and_graph_capture(engine):
    import torch
    nr, npr = 300, 100
    f = synth.pf_fleet_inputs(nr, npr, seed=31)
    a = run_fleet(engine, f, npr)
    b = run_fleet(engine, f, npr, status=False)
    assert all(same(x, y) for x, y in zip(a[:4], b[:4]))
    # n_robots = 0
    e = torch.zeros(0, device="cuda:0")
    res = engine.pf_step_many(npr, e.reshape(4, 0), e, e.reshape(4, 0).clone(), e.reshape(2, 0),
                              (_dev(f["z"]), _dev(f["z_off"])), torch.zeros(0, dtype=torch.int32, device="cuda:0"))
    torch.cuda.synchronize()
    assert tuple(res.shape) == (_lib.CRB_PF_RESULT_LEN, 0)

    # two eager steps (ping-pong) against a captured step replayed twice
    def bufs():
        return [_dev(f["px"]), _dev(f["pw"]), torch.zeros(4, nr * npr, device="cuda:0"),
                torch.zeros(_lib.CRB_PF_RESULT_LEN, nr, dtype=torch.float64, device="cuda:0")]
    u, zz, zo, zof = _dev(f["u"]), _dev(f["z"]), _dev(f["z_off"]), _dev(f["z_of"])
    x, w, xn, r = bufs()
    for _ in range(2):
        engine.pf_step_many(npr, x, w, xn, u, (zz, zo), zof, resample_seed=5, result=r)
        x.copy_(xn)
    torch.cuda.synchronize()
    gx, gw, gxn, gr = bufs()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        engine.bind_current_stream()
        with torch.cuda.graph(graph, stream=s):
            engine.pf_step_many(npr, gx, gw, gxn, u, (zz, zo), zof, resample_seed=5, result=gr)
            gx.copy_(gxn)
    engine.bind_current_stream()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert same(_host(gx), _host(x)) and same(_host(gw), _host(w)) and same(_host(gr), _host(r))


@pytest.mark.gpu
def test_closed_loop_against_the_checker(engine):
    """50 ticks of 1024 robots ping-ponging px / px_next; each tick the checker is fed the GPU's own state."""
    import torch
    nr, npr = 1024, 100
    f = synth.pf_fleet_inputs(nr, npr, seed=41)
    x, w, xn = _dev(f["px"]), _dev(f["pw"]), torch.zeros(4, nr * npr, device="cuda:0")
    u, zz, zo, zof = _dev(f["u"]), _dev(f["z"]), _dev(f["z_off"]), _dev(f["z_of"])
    n_res = 0
    for t in range(50):
        g = synth.pf_fleet_inputs(nr, npr, seed=1000 + t)
        x0, w0 = _host(x), _host(w)
        res = engine.pf_step_many(npr, x, w, xn, u, (zz, zo), zof, noise=_dev(g["noise"]),
                                  uniforms=_dev(g["uniforms"]))
        torch.cuda.synchronize()
        robots = range(t % 8, nr, 8)
        cpx, cpw, cpxn, cres, _ = PFF.step_many(npr, x0, w0, f["u"], f["z"], f["z_off"], f["z_of"], g["noise"],
                                                g["uniforms"], robots=robots)
        gpx, gpw, gpxn, gres = _host(x), _host(w), _host(xn), _host(res)
        for r in robots:
            cols = slice(r * npr, (r + 1) * npr)
            np.testing.assert_allclose(gpx[:, cols], cpx[:, cols], rtol=0, atol=1e-5)
            np.testing.assert_allclose(gres[:4, r], cres[:4, r], rtol=1e-4, atol=1e-5)
            if abs(cres[21, r] - npr // 2) > 1e-3 * npr:
                assert gres[22, r] == cres[22, r], (t, r)
                np.testing.assert_allclose(gpw[cols], cpw[cols], rtol=1e-4, atol=1e-12)
                moved = (np.abs(gpxn[:, cols] - cpxn[:, cols]) > 1e-5).any(axis=0).sum()
                assert moved <= 2, (t, r, moved)
            n_res += int(gres[22, r])
        x, xn = xn, x
    assert n_res > 0


@pytest.mark.gpu
def test_reference_style_program_matches_the_checker(tmp_path):
    """The C++ fleet tick (pf_localization_resampling) against the checker fed the program's inputs and the draws the
    reference's loops make with each robot's generators."""
    exe = build_ref_program(tmp_path, "pf_fleet_ref_api.cpp")
    out = subprocess.check_output([exe], text=True).strip().splitlines()
    head = out[0].split()
    nr, npr = int(head[1]), int(head[3])
    rows = {}
    for ln in out[1:-1]:
        name, *vals = ln.split()
        rows.setdefault(name, []).append(np.array([float.fromhex(v) for v in vals], np.float32))
    checksum = float(out[-1].split()[1])
    total = 0.0
    for r in range(nr):
        px = rows["px"][r].reshape(npr, 4).T.copy()          # Eigen's 4 x NP is particle-major
        noise = rows["noise"][r].reshape(2, npr)
        _, pw_c, pxn_c, res_c = PFF.step_one(px, rows["pw"][r], rows["u"][r], rows["z"][r].reshape(-1, 3), noise,
                                             rows["uniforms"][r])
        px_out = rows["px_out"][r].reshape(npr, 4).T
        moved = (np.abs(px_out - pxn_c) > 1e-5).any(axis=0).sum()
        assert moved <= 2, (r, moved)   # a resampleid on a cumulative weight can pick the neighbouring particle
        np.testing.assert_allclose(rows["pw_out"][r], pw_c, rtol=1e-4, atol=1e-12)
        np.testing.assert_allclose(rows["xEst"][r], res_c[:4], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(rows["PEst"][r], res_c[4:20], rtol=1e-3, atol=1e-7)
        total += float(np.sum(rows["xEst"][r].astype(np.float64)))
    assert checksum == pytest.approx(total, rel=1e-6, abs=1e-6)
