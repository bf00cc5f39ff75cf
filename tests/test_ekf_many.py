"""A noise model per agent: crb_ekf_step_many_batched and crb_ekf_track_step_many step agent i with
models[model_of[i]], a crb_ekf_params record (dt, Q, R) in a device table.

Each agent's x and P must be bitwise those of crb_ekf_step_batched run with its model (both run ekf_step of
crb_ekf_common.cuh); the checker composed model by model (oracle/ekf_many.py) follows with test_ekf_edges.py's rules.
CPU: argument validation without a device, the record layout, synth.ekf_fleet_inputs, the composed checker on a
one-model table, the compiler report of crb_ekf_many.cu, the SASS pin of the single-model kernels and the C++ fleet
program (tests/cpp/ekf_many_ref_api.cpp) compiling.
H100 (-m gpu): group-by-group bits at n 1 to 2^20, both launch forms, 1 and 3 steps, 1 to n models; the same batches
and the special values of test_ekf_edges.py against the checker; bad indices; NULL status; graph capture; offsets past
2^31; the resident track, pinned and pageable; the C++ program against the checker."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from cpprobotics_b200 import EKF_MODEL_DTYPE, EkfParams, _lib, ekf_models, synth
from oracle import ekf_many as EM
from oracle import oracle as O
from test_ekf_edges import NAMES, SETS, _assert_same, _params, _special_batch
from toolchain import build_ref_program, kernel_sass_hashes, ptxas_functions

INV = -1
F32 = np.float32


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


def set_table(n_models):
    """The eight parameter sets of test_ekf_edges.py as a table of n_models records, model k being set k % 8."""
    k = np.arange(n_models) % len(NAMES)
    dt = np.array([SETS[NAMES[j]][0] for j in k], np.float64)
    Q = np.stack([SETS[NAMES[j]][1] for j in k]).astype(F32)
    R = np.stack([SETS[NAMES[j]][2] for j in k]).astype(F32)
    return dt, Q, R


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_validation_needs_no_device():
    """Every bad host argument is refused with CRB_ERR_INVALID_ARG before any device work; n = 0 is a no-op; a valid
    call says CRB_ERR_NO_DEVICE on a machine without a GPU."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)

    def call(**over):
        a = dict(dict(ctx=ctx, n=5, x=d, P=d, z=d, u=d, models=d, nm=3, mof=d, ns=1, st=None), **over)
        return L.crb_ekf_step_many_batched(a["ctx"], a["n"], a["x"], a["P"], a["z"], a["u"], a["models"], a["nm"],
                                           a["mof"], a["ns"], a["st"])

    for kw in (dict(ctx=None), dict(n=-1), dict(ns=0), dict(ns=-2), dict(nm=0), dict(nm=-1), dict(x=None),
               dict(P=None), dict(z=None), dict(u=None), dict(models=None), dict(mof=None)):
        assert call(**kw) == INV, kw
    for kw in (dict(ctx=None), dict(ns=0), dict(nm=0)):
        assert call(n=0, **kw) == INV, kw
    assert call(n=0, x=None, P=None, z=None, u=None, models=None, mof=None) == _lib.CRB_OK
    if not torch.cuda.is_available():
        assert call() == _lib.CRB_ERR_NO_DEVICE and call(st=d, ns=4) == _lib.CRB_ERR_NO_DEVICE
        assert b"no CPU fallback" in L.crb_last_error_string()

    def track(**over):
        a = dict(dict(ctx=ctx, t=d, z=d, u=d, models=d, nm=3, mof=d), **over)
        return L.crb_ekf_track_step_many(a["ctx"], a["t"], a["z"], a["u"], a["models"], a["nm"], a["mof"], None,
                                         None, 0)

    for kw in (dict(ctx=None), dict(t=None), dict(z=None), dict(u=None), dict(models=None), dict(mof=None),
               dict(nm=0), dict(nm=-5)):
        assert track(**kw) == INV, kw


def test_model_record_layout():
    """ekf_models packs crb_ekf_params records: 88 bytes, dt at 0, Q at 8, R at 72, as ctypes lays the struct out."""
    assert EKF_MODEL_DTYPE.itemsize == C.sizeof(EkfParams) == 88
    assert [EKF_MODEL_DTYPE.fields[k][1] for k in ("dt", "Q", "R")] == [EkfParams.dt.offset, EkfParams.Q.offset,
                                                                         EkfParams.R.offset] == [0, 8, 72]
    dt, Q, R = set_table(8)
    t = ekf_models(dt, Q, R)
    assert t.shape == (8, 88) and t.dtype == np.uint8 and t.flags["C_CONTIGUOUS"]
    for m in range(8):
        p = EkfParams.from_buffer_copy(t[m].tobytes())
        assert p.dt == dt[m] and same(np.array(p.Q[:], F32), Q[m]) and same(np.array(p.R[:], F32), R[m])
    with pytest.raises(ValueError):
        ekf_models([], np.zeros((0, 16)), np.zeros((0, 4)))


def test_fleet_inputs_mix_the_models():
    f = synth.ekf_fleet_inputs(5000, 64, seed=5, n_steps=2)
    g = synth.ekf_fleet_inputs(5000, 64, seed=5, n_steps=2)
    assert all(np.array_equal(f[k], g[k]) for k in f)
    h = synth.ekf_fleet_inputs(5000, 64, seed=6, n_steps=2)
    assert not np.array_equal(f["dt"], h["dt"]) and not np.array_equal(f["model_of"], h["model_of"])
    x, P, z, u = synth.ekf_inputs(5000, seed=5, n_steps=2)
    assert same(f["x"], x) and same(f["P"], P) and same(f["z"], z) and same(f["u"], u)
    mof = f["model_of"]
    assert mof.dtype == np.int32 and mof.shape == (5000,) and set(mof.tolist()) == set(range(64))
    assert (np.diff(mof) != 1).mean() > 0.9                      # shuffled, not striped
    assert len(np.unique(f["dt"])) == 64 and len(np.unique(f["Q"], axis=0)) == 64 and len(np.unique(f["R"], axis=0)) == 64
    Qm = f["Q"].reshape(64, 4, 4)
    assert (Qm != Qm.transpose(0, 2, 1)).any(axis=(1, 2)).sum() >= 16    # non-symmetric Q in many models
    assert (f["R"][:, 1] != f["R"][:, 2]).sum() >= 8
    one = synth.ekf_fleet_inputs(10, 1, seed=1)
    assert (one["model_of"] == 0).all()


def test_composed_checker_on_one_model_is_the_checker():
    x, P, z, u = synth.ekf_inputs(999, seed=3, n_steps=3)
    dt, Q, R = SETS["Q_full"]
    gx, gP, st = EM.step_many(x, P, z, u, [dt], Q[None], R[None], np.zeros(999, np.int32), n_steps=3)
    xo, Po = O.ekf_step_batched(x, P, z, u, Q=Q, R=R, dt=dt, n_steps=3)
    assert (st == EM.EKF_OK).all() and same(gx, xo) and same(gP, Po)
    # two models: each group is the checker with its own constants; bad indices give NaN and BAD_MODEL
    mof = (np.arange(999) % 2).astype(np.int32)
    mof[[5, 600]] = [-1, 2]
    d2, Q2, R2 = SETS["R_asym"]
    gx, gP, st = EM.step_many(x, P, z, u, [dt, d2], np.stack([Q, Q2]), np.stack([R, R2]), mof, n_steps=3)
    assert st.tolist() == [EM.EKF_BAD_MODEL if i in (5, 600) else EM.EKF_OK for i in range(999)]
    assert np.isnan(gx[:, [5, 600]]).all() and np.isnan(gP[:, [5, 600]]).all()
    for m, (dm, Qm, Rm) in enumerate(((dt, Q, R), (d2, Q2, R2))):
        cols = np.flatnonzero(mof == m)
        xo, Po = O.ekf_step_batched(x[:, cols], P[:, cols], z[:, cols], u[:, cols], Q=Qm, R=Rm, dt=dm, n_steps=3)
        assert same(gx[:, cols], xo) and same(gP[:, cols], Po)


# sha256 of each single-model EKF kernel's SASS (cuobjdump -sass, NVCC_FLAGS, CUDA 12.9) as they were before the model
# table existed: moving their shared code into crb_ekf_common.cuh must not change one instruction
SINGLE_MODEL_SASS = {
    "_Z19crb_ekf_step_kernelILi256ELi3ELi1EEvllPfS0_PKfS2_li7EkfArgs":
        "3a3dde8cf10fc6d2579dfe944258f010246c4a8ad410289f336f07b44173d8bb",
    "_Z19crb_ekf_step_kernelILi128ELi4ELi2EEvllPfS0_PKfS2_li7EkfArgs":
        "427c56cbd749cde3b725f09a8b711cbc9340e8ee9cd7b86a56368d1eaf2f8fea",
}


def test_model_table_kernels_do_not_spill():
    """Exactly the two launch forms, with no spill and no stack frame in them or in anything they call."""
    fns = ptxas_functions("crb_ekf_many.cu")
    assert {f.name for f in fns if f.entry} == {
        "_Z19crb_ekf_many_kernelILi256ELi3ELi1EEvllPfS0_PKfS2_liPK7EkfArgsiPKiPi",
        "_Z19crb_ekf_many_kernelILi128ELi4ELi2EEvllPfS0_PKfS2_liPK7EkfArgsiPKiPi"}, fns
    assert all((f.stack, f.spill_stores, f.spill_loads) == (0, 0, 0) for f in fns), fns


def test_single_model_kernels_keep_their_machine_code():
    assert kernel_sass_hashes("crb_ekf.cu") == SINGLE_MODEL_SASS


def test_reference_style_program_compiles(tmp_path):
    build_ref_program(tmp_path, "ekf_many_ref_api.cpp")


# ---- H100 ---------------------------------------------------------------------------------------------------------------
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


def run_many(engine, x, P, z, u, table, model_of, n_steps=1, misaligned=False, status=True):
    import torch
    d = [_dev(a, misaligned) for a in (x, P, z, u)]
    st = torch.full((x.shape[1],), -7, dtype=torch.int32, device="cuda") if status else None
    engine.ekf_estimation_many(*d, _dev(ekf_models(*table)), _dev(model_of, misaligned), n_steps=n_steps, status=st)
    torch.cuda.synchronize()
    return d[0].cpu().numpy(), d[1].cpu().numpy(), (st.cpu().numpy() if status else None)


def run_single(engine, x, P, z, u, dt, Q, R, n_steps=1):
    import torch
    d = [_dev(a) for a in (x, P, z, u)]
    engine.ekf_estimation(*d, params=_params(dt, Q, R), n_steps=n_steps)
    torch.cuda.synchronize()
    return d[0].cpu().numpy(), d[1].cpu().numpy()


def assert_groups_are_single_model(engine, x, P, z, u, gx, gP, model_of, n_steps):
    """Agents of set j (models k with k % 8 == j) against ONE crb_ekf_step_batched launch of set j."""
    for j, name in enumerate(NAMES):
        cols = np.flatnonzero(model_of % len(NAMES) == j)
        if cols.size == 0:
            continue
        sx, sP = run_single(engine, *(np.ascontiguousarray(a[:, cols]) for a in (x, P, z, u)), *SETS[name], n_steps)
        assert same(gx[:, cols], sx), (name, "x")
        assert same(gP[:, cols], sP), (name, "P")


N_CASES = [1, 2, 4097, 1 << 20]
M_CASES = [1, 8, 4096, "n"]


@pytest.mark.gpu
@pytest.mark.parametrize("misaligned", [False, True], ids=["aligned", "misaligned"])
@pytest.mark.parametrize("n_steps", [1, 3])
@pytest.mark.parametrize("n_models", M_CASES)
@pytest.mark.parametrize("n", N_CASES)
def test_each_agent_is_the_single_model_step(engine, n, n_models, n_steps, misaligned):
    """Agents shuffled over a table of the eight parameter sets: every agent bitwise crb_ekf_step_batched with its
    set.  Even n with aligned arrays takes the two-agent form; odd n or arrays at a 4-byte offset the one-agent form.
    Then the same batch against the composed checker (a sample of agents when every agent has its own model)."""
    m = n if n_models == "n" else n_models
    rng = np.random.default_rng([n, m, n_steps])
    x, P, z, u = synth.ekf_inputs(n, n_steps=n_steps, seed=0x3A + n_steps)
    mof = (rng.permutation(n) % m if m >= n else rng.integers(0, m, n)).astype(np.int32)
    table = set_table(m)
    gx, gP, st = run_many(engine, x, P, z, u, table, mof, n_steps, misaligned)
    assert (st == _lib.CRB_EKF_OK).all()
    assert_groups_are_single_model(engine, x, P, z, u, gx, gP, mof, n_steps)
    agents = None if n <= 65536 else rng.choice(n, 8192, replace=False)
    cx, cP, cst = EM.step_many(x, P, z, u, *table, mof, n_steps=n_steps, agents=agents)
    sel = np.arange(n) if agents is None else np.sort(agents)
    _assert_same(gx[:, sel], cx[:, sel], "x")
    _assert_same(gP[:, sel], cP[:, sel], "P")


@pytest.mark.gpu
@pytest.mark.parametrize("n_models", [8, 4096, "n"])
@pytest.mark.parametrize("n", [4097, 65536])
def test_fleet_inputs_against_the_checker(engine, n, n_models):
    """synth.ekf_fleet_inputs (every model its own dt, Q and R) over three steps against the composed checker."""
    m = n if n_models == "n" else n_models
    f = synth.ekf_fleet_inputs(n, m, seed=0x51, n_steps=3)
    table = (f["dt"], f["Q"], f["R"])
    gx, gP, st = run_many(engine, f["x"], f["P"], f["z"], f["u"], table, f["model_of"], 3)
    cx, cP, cst = EM.step_many(f["x"], f["P"], f["z"], f["u"], *table, f["model_of"], n_steps=3)
    assert (st == cst).all()
    _assert_same(gx, cx, "x")
    _assert_same(gP, cP, "P")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 65])
def test_special_values_are_the_single_model_step(engine, n):
    """test_ekf_edges.py's poisoned agents (NaN, inf, signed zeros, subnormals, overflow) over a shuffled table of the
    eight sets: bitwise crb_ekf_step_batched group by group, which carries every documented deviation of the dense
    evaluation along unchanged."""
    x, P, z, u, _ = _special_batch(n)
    mof = np.random.default_rng(n).integers(0, 8, n).astype(np.int32)
    gx, gP, st = run_many(engine, x, P, z, u, set_table(8), mof)
    assert (st == 0).all()
    assert np.isnan(gx).any()
    assert_groups_are_single_model(engine, x, P, z, u, gx, gP, mof, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4096, 4097])
def test_bad_indices_stay_with_their_agent(engine, n):
    """model_of -1, n_models and INT32_MAX: those agents NaN with BAD_MODEL, every other agent bitwise the run without
    them; the same without status."""
    x, P, z, u = synth.ekf_inputs(n, seed=0x77, n_steps=3)
    mof = np.random.default_rng(n).integers(0, 8, n).astype(np.int32)
    table = set_table(8)
    base = run_many(engine, x, P, z, u, table, mof, 3)
    bad = {3: -1, 10: 8, 11: 2 ** 31 - 1, n - 1: -(2 ** 31), n // 2: 9}
    mb = mof.copy()
    for i, v in bad.items():
        mb[i] = v
    gx, gP, st = run_many(engine, x, P, z, u, table, mb, 3)
    idx = np.array(sorted(bad))
    keep = np.setdiff1d(np.arange(n), idx)
    assert (st[idx] == _lib.CRB_EKF_BAD_MODEL).all() and (st[keep] == _lib.CRB_EKF_OK).all()
    assert np.isnan(gx[:, idx]).all() and np.isnan(gP[:, idx]).all()
    assert same(gx[:, keep], base[0][:, keep]) and same(gP[:, keep], base[1][:, keep])
    nx, nP, _ = run_many(engine, x, P, z, u, table, mb, 3, status=False)
    assert same(nx, gx) and same(nP, gP)
    cx, cP, cst = EM.step_many(x, P, z, u, *table, mb, n_steps=3)
    assert (cst == st).all()
    _assert_same(gx, cx, "x")
    _assert_same(gP, cP, "P")


@pytest.mark.gpu
def test_empty_batch_and_graph_capture(engine):
    import torch
    e = torch.zeros(0, device="cuda")
    tab = _dev(ekf_models(*set_table(8)))
    engine.ekf_estimation_many(e.reshape(4, 0), e.reshape(16, 0), e.reshape(2, 0), e.reshape(2, 0), tab,
                               torch.zeros(0, dtype=torch.int32, device="cuda"))
    n = 65536
    f = synth.ekf_fleet_inputs(n, 4096, seed=0x61, n_steps=2)
    tab = _dev(ekf_models(f["dt"], f["Q"], f["R"]))
    mof = _dev(f["model_of"])

    def bufs():
        return [_dev(f[k]) for k in ("x", "P", "z", "u")] + [torch.zeros(n, dtype=torch.int32, device="cuda")]
    x, P, z, u, st = bufs()
    for _ in range(2):
        engine.ekf_estimation_many(x, P, z, u, tab, mof, n_steps=2, status=st)
    torch.cuda.synchronize()
    gx, gP, gz, gu, gst = bufs()
    gst.fill_(-1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        engine.bind_current_stream()
        with torch.cuda.graph(graph, stream=s):
            engine.ekf_estimation_many(gx, gP, gz, gu, tab, mof, n_steps=2, status=gst)
    engine.bind_current_stream()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert same(gx.cpu().numpy(), x.cpu().numpy()) and same(gP.cpu().numpy(), P.cpu().numpy())
    assert (gst.cpu().numpy() == 0).all()


BLOCK = 65_521   # prime: an offset wrapped by a multiple of 2^31 lands on an agent of another residue


@pytest.mark.gpu
def test_offsets_past_2_31(engine):
    """n = 2^27 + 2 agents (the two-agent form): 19 * n + i passes 2^31.  Agent i gets the inputs and the model index
    of agent i mod L of one block of L = 65521 agents over 8 models, so it must reproduce the checker's result for
    that agent; a 32-bit offset would bring another agent's numbers."""
    import torch
    n = (1 << 27) + 2
    need = 4 * n * 25 + (3 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    f = synth.ekf_fleet_inputs(BLOCK, 8, seed=0xF9)
    table = (f["dt"], f["Q"], f["R"])
    cx, cP, _ = EM.step_many(f["x"], f["P"], f["z"], f["u"], *table, f["model_of"])
    reps = -(-n // BLOCK)

    def tile(a):
        src = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        if src.dim() == 1:
            return src.repeat(reps)[:n].contiguous()
        out = torch.empty((a.shape[0], n), dtype=src.dtype, device="cuda")
        for k in range(a.shape[0]):
            out[k].copy_(src[k].repeat(reps)[:n])
        return out
    d = [tile(f[k]) for k in ("x", "P", "z", "u", "model_of")]
    try:
        engine.ekf_estimation_many(*d[:4], _dev(ekf_models(*table)), d[4])
        torch.cuda.synchronize()
        want = [torch.from_numpy(a).cuda() for a in (cx, cP)]
        rng = np.random.default_rng(31)
        for a0 in [0, n - (1 << 20)] + sorted(rng.integers(0, n - (1 << 20), 6).tolist()):
            a1 = a0 + (1 << 20)
            idx = torch.arange(a0, a1, device="cuda") % BLOCK
            for got, w, what in ((d[0], want[0], "x"), (d[1], want[1], "P")):
                assert torch.equal(got[:, a0:a1], w[:, idx]), f"{what}: agents [{a0}, {a1}) differ"
    finally:
        del d
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_track_is_the_many_launch(engine, pinned):
    """50 ticks of crb_ekf_track_step_many (x_out every tick, alternating async and synchronous ticks) against 50
    crb_ekf_step_many_batched launches; then a one-model table over the same ticks against crb_ekf_track_step."""
    import torch
    n, K = 4098, 50
    f = synth.ekf_fleet_inputs(n, 8, seed=0x71, n_steps=K)
    tab = _dev(ekf_models(f["dt"], f["Q"], f["R"]))
    mof = _dev(f["model_of"])

    def host(a):
        t = torch.from_numpy(np.ascontiguousarray(a))
        return t.pin_memory() if pinned else t
    zs = [host(f["z"][2 * k:2 * k + 2]) for k in range(K)]
    us = [host(f["u"][2 * k:2 * k + 2]) for k in range(K)]
    outs = [host(np.zeros((4, n), F32)) for _ in range(2)]
    dx, dP = _dev(f["x"]), _dev(f["P"])
    st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    one = _dev(ekf_models(*set_table(1)))
    zero = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for table, ids, single in ((tab, mof, False), (one, zero, True)):
        trk = engine.ekf_track_open(f["x"], f["P"])
        ref = engine.ekf_track_open(f["x"], f["P"]) if single else None
        dx.copy_(_dev(f["x"]))
        dP.copy_(_dev(f["P"]))
        try:
            for k in range(K):
                async_ = k % 2 == 0
                engine.ekf_track_step_many(trk, zs[k], us[k], table, ids, status=st, x_out=outs[k % 2],
                                           async_=async_)
                if async_:
                    engine.ekf_track_sync(trk)
                if single:
                    want = host(np.zeros((4, n), F32))
                    engine.ekf_track_step(ref, zs[k], us[k], params=_params(*SETS[NAMES[0]]), x_out=want)
                    assert same(outs[k % 2].numpy(), want.numpy()), k
                else:
                    engine.ekf_estimation_many(dx, dP, _dev(f["z"][2 * k:2 * k + 2]), _dev(f["u"][2 * k:2 * k + 2]),
                                               tab, mof)
                    torch.cuda.synchronize()
                    assert same(outs[k % 2].numpy(), dx.cpu().numpy()), k
            gx, gP = np.empty_like(f["x"]), np.empty_like(f["P"])
            engine.ekf_track_read(trk, gx, gP)
            if single:
                rx, rP = np.empty_like(f["x"]), np.empty_like(f["P"])
                engine.ekf_track_read(ref, rx, rP)
                assert same(gx, rx) and same(gP, rP)
            else:
                assert same(gx, dx.cpu().numpy()) and same(gP, dP.cpu().numpy())
            assert (st.cpu().numpy() == 0).all()
        finally:
            engine.ekf_track_close(trk)
            if ref is not None:
                engine.ekf_track_close(ref)


@pytest.mark.gpu
def test_reference_style_program_matches_the_checker(tmp_path):
    """The C++ fleet (ekf_estimation over vectors of robots, 50 ticks) against the checker fed the program's inputs."""
    exe = build_ref_program(tmp_path, "ekf_many_ref_api.cpp")
    out = subprocess.check_output([exe], text=True).strip().splitlines()
    head = out[0].split()
    nr, steps = int(head[1]), int(head[3])
    rows = {}
    for ln in out[1:-1]:
        name, *vals = ln.split()
        rows.setdefault(name, []).append(np.array([float.fromhex(v) for v in vals], F32))
    Q, R = np.stack(rows["Q"]), np.stack(rows["R"])
    x, P = np.stack(rows["x0"], axis=1), np.stack(rows["P0"], axis=1)
    dt = np.full(nr, O.ekf_constants()[0])
    mof = np.arange(nr, dtype=np.int32)
    for t in range(steps):
        z = np.stack(rows["z"][t * nr:(t + 1) * nr], axis=1)
        u = np.stack(rows["ud"][t * nr:(t + 1) * nr], axis=1)
        x, P, st = EM.step_many(x, P, z, u, dt, Q, R, mof)
    _assert_same(np.stack(rows["xEst"], axis=1), x, "xEst")
    _assert_same(np.stack(rows["PEst"], axis=1), P, "PEst")
    assert np.isfinite(x).all() and float(out[-1].split()[1]) == pytest.approx(float(x.astype(np.float64).sum()),
                                                                               rel=1e-6)
