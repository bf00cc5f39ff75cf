"""Model-predictive trajectory generation (include/trajectory_optimizer.h, include/motion_model.h).
CPU: the restated tanf is bitwise the host tanf on every float with |x| < 120; the checker is bitwise the reference's
own text (seeded problems and corner cases) and the golden fixture; statuses, parameters, layouts and argument
validation.  H100: crb_mptg_optimize_batched and crb_mptg_generate_trajectory_batched are bitwise the checker (batch
sizes, corner cases, shard invariance), the golden fixture, the reference-style C++ program, and a device census of
crb_tanf_libm against the checker's restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mptg_cases as MC
from cpprobotics_b200 import _lib, synth
from oracle import mptg as OM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libref_mptg.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "mptg_golden.npz")
CPP = os.path.join(ROOT, "tests", "cpp", "mptg_ref_api.cpp")
MAX_PTS = 128  # the golden fixture's


def same(a, b):
    """Bitwise equal, except that any NaN equals any NaN (NaN payloads are not specified by either side)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def lib_params(p):
    q = _lib.MptgParams()
    q.base_l, q.ds, q.max_iter, q.cost_th = p.base_l, p.ds, p.max_iter, p.cost_th
    for k in range(3):
        q.h_step[k] = p.h_step[k]
    return q


def prm_of(v):
    return OM.mptg_params(base_l=v[0], ds=v[1], max_iter=int(v[2]), cost_th=v[3], h_step=tuple(v[4:7]))


# ---- CPU ------------------------------------------------------------------------------------------------------
def test_tanf_restatement_is_the_host_tanf_on_every_float_below_120():
    assert OM.libm_tanf_census(0, 0x42F00000) == 0     # |x| < 120, both signs, every bit pattern
    libm = C.CDLL("libm.so.6")
    libm.tanf.restype, libm.tanf.argtypes = C.c_float, [C.c_float]
    for v in np.array([0.0, -0.0, 0.78539816, 0.7853982, 1.5707964, -1.5707964, 3.1415927, 119.99999, np.inf,
                       -np.inf, np.nan], np.float32):
        a, b = np.float32(libm.tanf(float(v))), np.float32(OM.libm_tanf(float(v)))
        assert same(a, b), (v, a, b)


def _ref_lib():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref not built (needs the reference tree: make -C oracle -f mptg.mk)")
    import golden.make_mptg_golden as G
    return C.CDLL(REF), G


def _compare_with_reference(L, G, st, tg, pa, prm, max_pts=MAX_PTS):
    o = OM.optimize(st, tg, pa, prm, max_pts=max_pts)
    sel = np.flatnonzero(o["status"] <= OM.MAX_ITER_REACHED)   # the reference's UB / endless loops are not fed to it
    sub = [np.ascontiguousarray(a[:, sel]) for a in (st, tg, pa)]
    q, traj, tl, cost = G.reference(L, *sub, prm, max_pts)
    assert same(o["param"][:, sel], q) and same(o["traj"][:, sel], traj)
    assert np.array_equal(o["traj_len"][sel], tl) and same(o["cost"][sel], cost)
    conv = o["status"][sel] == OM.CONVERGED
    assert np.array_equal(conv, np.nan_to_num(cost, nan=np.inf) < np.float32(prm.cost_th))
    return o, sel


def test_oracle_is_bitwise_the_reference_text_on_synth_problems():
    L, G = _ref_lib()
    st, tg, pa = synth.mptg_inputs(2400, seed=11)
    o, sel = _compare_with_reference(L, G, st, tg, pa, OM.mptg_params())
    assert len(sel) >= 2000
    counts = np.bincount(o["status"], minlength=5)
    assert counts[OM.CONVERGED] > 1800 and counts[OM.MAX_ITER_REACHED] > 0
    assert all(counts[s] > 0 for s in (OM.EMPTY_TRAJ, OM.STEP_CAP, OM.OUT_OF_RANGE))
    assert ((o["quirks"][sel] & OM.Q_STEER_BEYOND_PIO4) != 0).sum() > 100   # glibc's tanf range reduction
    # generate_trajectory / generate_last_state of the returned parameters
    g = OM.generate(st[:, sel], o["param"][:, sel], max_pts=MAX_PTS)
    ok = np.flatnonzero(g["status"] == 0)
    for i in ok[:300]:
        s, q = (np.ascontiguousarray(a[:, sel[i]], np.float32) for a in (st, o["param"]))
        tr, last, k = np.full(3 * MAX_PTS, np.nan, np.float32), np.zeros(3, np.float32), C.c_int(0)
        L.ref_mptg_generate(s.ctypes.data, q.ctypes.data, C.c_float(1.0), C.c_float(0.1),
                            tr.ctypes.data, MAX_PTS, C.byref(k), last.ctypes.data)
        assert k.value == g["traj_len"][i] and same(tr, g["traj"][:, i]) and same(last, g["last"][:, i])


@pytest.mark.parametrize("case", [c[0] for c in MC.quirk_sets()])
def test_oracle_is_bitwise_the_reference_text_on_corner_cases(case):
    L, G = _ref_lib()
    name, st, tg, pa, prm = next(c for c in MC.quirk_sets() if c[0] == case)
    o, sel = _compare_with_reference(L, G, st, tg, pa, prm, max_pts=8192)
    q = np.bitwise_or.reduce(o["quirks"])
    if case == "converged_at_0":
        assert o["status"][0] == OM.CONVERGED and o["iters"][0] == 0 and q & OM.Q_CONVERGED_AT_0
    elif case == "ls_tie":
        assert q & OM.Q_LS_TIE and o["status"][0] == OM.MAX_ITER_REACHED
    elif case == "max_iter_2":   # the trajectory is the roll-out of the parameter before the last update
        assert o["status"][0] == OM.MAX_ITER_REACHED and o["iters"][0] == 2
        g = OM.generate(st, o["param"], max_pts=8192)
        assert g["traj_len"][0] != o["traj_len"][0] or not same(g["traj"], o["traj"])
    elif case == "max_iter_0":
        assert o["status"][0] == OM.MAX_ITER_REACHED and o["traj_len"][0] == 0 and np.isnan(o["cost"][0])
        assert same(o["param"], pa)
    elif case == "singular_j":
        assert q & OM.Q_SINGULAR_J and np.isnan(o["param"][[0, 2, 3], 0]).all() and o["param"][1, 0] == 0.0
    elif case == "nan_costs":
        assert q & OM.Q_LS_NAN
    elif case == "steer_beyond_pio4":
        assert q & OM.Q_STEER_BEYOND_PIO4 and len(sel) == 1
    elif case == "distance_sweep":
        assert q & OM.Q_STEPS_OFF_CEIL and len(sel) > 100


def test_statuses_of_the_cases_the_reference_does_not_define():
    (name, st, tg, pa, prm), want = MC.stopping_sets()
    o = OM.optimize(st, tg, pa, prm, max_pts=16)
    assert o["status"].tolist() == want
    assert (o["traj_len"] == 0).all() and np.isnan(o["cost"]).all() and (o["iters"] == 0).all()
    assert np.isnan(o["traj"]).all()   # nothing written
    g = OM.generate(st, pa, max_pts=16)
    assert g["status"].tolist() == [0, OM.STEP_CAP, OM.OUT_OF_RANGE, OM.OUT_OF_RANGE, 0]
    assert g["traj_len"].tolist() == [0, 0, 0, 0, 0] and same(g["last"][:, 0], st[:3, 0])


def test_oracle_reproduces_the_golden_fixture():
    d = np.load(GOLDEN)
    for name in d["names"]:
        prm = prm_of(d[f"{name}_prm"])
        o = OM.optimize(d[f"{name}_state"], d[f"{name}_target"], d[f"{name}_param_in"], prm, max_pts=MAX_PTS)
        sel = o["status"] <= OM.MAX_ITER_REACHED
        assert same(o["param"][:, sel], d[f"{name}_param"][:, sel]), name
        assert same(o["traj"][:, sel], d[f"{name}_traj"][:, sel]), name
        assert np.array_equal(o["traj_len"][sel], d[f"{name}_traj_len"][sel]), name
        assert same(o["cost"][sel], d[f"{name}_cost"][sel]), name
        assert sel.sum() >= (d[f"{name}_cost"].size - 8), name


def test_defaults_and_layout(tmp_path):
    from cpprobotics_b200 import mptg_default_params
    lp, op = mptg_default_params(), OM.mptg_params()
    assert (lp.base_l, lp.ds, lp.max_iter, lp.cost_th, list(lp.h_step)) == \
        (op.base_l, op.ds, op.max_iter, op.cost_th, list(op.h_step))
    assert np.float32(lp.cost_th) == np.float32(0.1) and np.float32(lp.h_step[1]) == np.float32(0.005)
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(void){printf("%zu %zu %zu %zu '
                   '%d %d %d %d %d %d %d\\n",sizeof(crb_mptg_params),offsetof(crb_mptg_params,max_iter),'
                   'offsetof(crb_mptg_params,cost_th),offsetof(crb_mptg_params,h_step),CRB_MPTG_MAX_ITER,'
                   'CRB_MPTG_MAX_STEPS,CRB_MPTG_CONVERGED,CRB_MPTG_MAX_ITER_REACHED,CRB_MPTG_EMPTY_TRAJ,'
                   'CRB_MPTG_STEP_CAP,CRB_MPTG_OUT_OF_RANGE);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    M = _lib.MptgParams
    assert got == [C.sizeof(M), M.max_iter.offset, M.cost_th.offset, M.h_step.offset, _lib.CRB_MPTG_MAX_ITER,
                   _lib.CRB_MPTG_MAX_STEPS, _lib.CRB_MPTG_CONVERGED, _lib.CRB_MPTG_MAX_ITER_REACHED,
                   _lib.CRB_MPTG_EMPTY_TRAJ, _lib.CRB_MPTG_STEP_CAP, _lib.CRB_MPTG_OUT_OF_RANGE]
    assert got[4:] == [OM.MAX_ITER, OM.MAX_STEPS, OM.CONVERGED, OM.MAX_ITER_REACHED, OM.EMPTY_TRAJ, OM.STEP_CAP,
                       OM.OUT_OF_RANGE]


def _invalid_params():
    cases = []
    for field, value in [("ds", 0.0), ("ds", -0.1), ("ds", np.nan), ("ds", np.inf), ("base_l", 0.0),
                         ("base_l", np.nan), ("base_l", -np.inf), ("cost_th", np.nan), ("cost_th", np.inf),
                         ("max_iter", -1), ("max_iter", _lib.CRB_MPTG_MAX_ITER + 1)]:
        p = OM.mptg_params()
        setattr(p, field, value)
        cases.append(lib_params(p))
    for k in range(3):
        for value in (0.0, -0.005, np.nan, np.inf):
            p = OM.mptg_params()
            p.h_step[k] = float(value)
            cases.append(lib_params(p))
    return cases


def test_validation_needs_no_device():
    """Bad arguments are refused before any device work; valid ones fail with CRB_ERR_NO_DEVICE on a machine without
    a GPU.  The context handle is an opaque non-NULL buffer that these paths never dereference."""
    import torch
    L = _lib.load_library()
    ctx = C.create_string_buffer(64)
    d = C.c_void_p(256)
    good = lib_params(OM.mptg_params())
    inv = -1

    def opt(**over):
        a = dict(dict(ctx=ctx, n=1, state=d, target=d, param=d, prm=C.byref(good), max_pts=4), **over)
        return L.crb_mptg_optimize_batched(a["ctx"], a["n"], a["state"], a["target"], a["param"], a["prm"],
                                           a["max_pts"], d, d, d, d, d)

    def gen(**over):
        a = dict(dict(ctx=ctx, n=1, state=d, param=d, prm=C.byref(good), max_pts=4), **over)
        return L.crb_mptg_generate_trajectory_batched(a["ctx"], a["n"], a["state"], a["param"], a["prm"],
                                                      a["max_pts"], d, d, d, d)
    for k in ("ctx", "state", "target", "param", "prm"):
        assert opt(**{k: None}) == inv, k
    for k in ("ctx", "state", "param", "prm"):
        assert gen(**{k: None}) == inv, k
    for f in (opt, gen):
        assert f(n=-1) == inv and f(max_pts=-1) == inv
        for p in _invalid_params():
            assert f(prm=C.byref(p)) == inv
    if not torch.cuda.is_available():
        for f in (opt, gen):
            assert f() == _lib.CRB_ERR_NO_DEVICE
            assert f(n=0, state=None, param=None, **({"target": None} if f is opt else {})) == _lib.CRB_ERR_NO_DEVICE
            assert f(max_pts=0) == _lib.CRB_ERR_NO_DEVICE
        assert b"no CPU fallback" in L.crb_last_error_string()
        p = OM.mptg_params(max_iter=0)
        assert opt(prm=C.byref(lib_params(p))) == _lib.CRB_ERR_NO_DEVICE


def _build_cpp(tmp_path):
    exe = str(tmp_path / "mptg_ref_api")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), CPP,
                           "-L", libdir, "-lcrb", f"-Wl,-rpath,{libdir}", "-o", exe])
    return exe


def test_reference_style_program_compiles(tmp_path):
    _build_cpp(tmp_path)


# ---- H100 -----------------------------------------------------------------------------------------------------
FILL = -7.25   # sentinel: points beyond what is written must keep it


def _gpu_optimize(engine, st, tg, pa, prm, max_pts, outputs=True):
    import torch
    dev = torch.device("cuda:0")
    n = st.shape[1]
    sd, td, qd = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev) for a in (st, tg, pa))
    traj = torch.full((3 * max_pts, n), FILL, dtype=torch.float32, device=dev) if outputs else None
    i32 = [torch.empty(n, dtype=torch.int32, device=dev) if outputs else None for _ in range(3)]
    cost = torch.empty(n, dtype=torch.float32, device=dev) if outputs else None
    engine.mptg_optimize(sd, td, qd, lib_params(prm), traj=traj, traj_len=i32[0], cost=cost, status=i32[1],
                         iters=i32[2])
    torch.cuda.synchronize()
    r = dict(param=qd.cpu().numpy())
    if outputs:
        r.update(traj=traj.cpu().numpy(), traj_len=i32[0].cpu().numpy(), cost=cost.cpu().numpy(),
                 status=i32[1].cpu().numpy(), iters=i32[2].cpu().numpy())
    return r


def _same_all(r, o):
    return all(same(r[k], o[k]) for k in ("param", "traj", "traj_len", "cost", "status", "iters"))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097, 65536])
def test_gpu_is_bitwise_the_oracle(engine, n):
    st, tg, pa = synth.mptg_inputs(n, seed=0x900 + n)
    if n == 1:
        st, tg, pa = MC.demo()
    max_pts = 48 if n == 4097 else 96   # shorter than many trajectories (up to ~100 points here)
    o = OM.optimize(st, tg, pa, OM.mptg_params(), max_pts=max_pts, traj_fill=FILL)
    r = _gpu_optimize(engine, st, tg, pa, OM.mptg_params(), max_pts)
    assert _same_all(r, o)
    if n >= 4097:
        assert (o["traj_len"] > max_pts).any() and len(np.unique(o["status"])) == 5
        assert same(_gpu_optimize(engine, st, tg, pa, OM.mptg_params(), 0, outputs=False)["param"], o["param"])


@pytest.mark.gpu
def test_gpu_corner_cases_are_bitwise_the_oracle(engine):
    sets = MC.quirk_sets() + [MC.stopping_sets()[0]]
    for name, st, tg, pa, prm in sets:
        o = OM.optimize(st, tg, pa, prm, max_pts=64, traj_fill=FILL)
        r = _gpu_optimize(engine, st, tg, pa, prm, 64)
        assert _same_all(r, o), name


@pytest.mark.gpu
def test_gpu_n_zero_is_a_no_op(engine):
    import torch
    e = torch.empty((4, 0), dtype=torch.float32, device="cuda:0")
    engine.mptg_optimize(e, e[:3], e)
    engine.mptg_generate_trajectory(e, e)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_reproduces_the_golden_fixture(engine):
    d = np.load(GOLDEN)
    for name in d["names"]:
        prm = prm_of(d[f"{name}_prm"])
        r = _gpu_optimize(engine, d[f"{name}_state"], d[f"{name}_target"], d[f"{name}_param_in"], prm, MAX_PTS)
        sel = r["status"] <= OM.MAX_ITER_REACHED
        assert sel.sum() >= d[f"{name}_cost"].size - 8, name
        traj = np.where(r["traj"] == np.float32(FILL), np.float32(np.nan), r["traj"])
        for k, v in (("param", r["param"]), ("traj", traj)):
            assert same(v[:, sel], d[f"{name}_{k}"][:, sel]), (name, k)
        assert np.array_equal(r["traj_len"][sel], d[f"{name}_traj_len"][sel]), name
        assert same(r["cost"][sel], d[f"{name}_cost"][sel]), name


@pytest.mark.gpu
def test_gpu_shard_invariance(engine):
    st, tg, pa = synth.mptg_inputs(10000, seed=77)
    full = _gpu_optimize(engine, st, tg, pa, OM.mptg_params(), 32)
    i0, i1 = 3001, 7203
    part = _gpu_optimize(engine, *(np.ascontiguousarray(a[:, i0:i1]) for a in (st, tg, pa)), OM.mptg_params(), 32)
    for k in ("param", "traj"):
        assert same(part[k], np.ascontiguousarray(full[k][:, i0:i1])), k
    for k in ("traj_len", "cost", "status", "iters"):
        assert same(part[k], full[k][i0:i1]), k
    shard = synth.mptg_inputs(i1 - i0, seed=77, i0=i0)
    for a, b in zip(shard, (st, tg, pa)):
        assert same(a, np.ascontiguousarray(b[:, i0:i1]))


@pytest.mark.gpu
def test_gpu_generate_trajectory_alone(engine):
    import torch
    dev = torch.device("cuda:0")
    st, tg, pa = synth.mptg_inputs(4097, seed=5)
    pa = OM.optimize(st, tg, pa)["param"]   # converged parameters, plus every corner of mptg_inputs
    (_, s2, _, p2, _), _ = MC.stopping_sets()
    st, pa = np.concatenate([st, s2], axis=1), np.concatenate([pa, p2], axis=1)
    n, max_pts = st.shape[1], 64
    o = OM.generate(st, pa, max_pts=max_pts, traj_fill=FILL)
    sd, qd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (st, pa))
    traj = torch.full((3 * max_pts, n), FILL, dtype=torch.float32, device=dev)
    tl, status = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
    last = torch.empty((3, n), dtype=torch.float32, device=dev)
    engine.mptg_generate_trajectory(sd, qd, traj=traj, traj_len=tl, last=last, status=status)
    torch.cuda.synchronize()
    for k, v in (("traj", traj), ("traj_len", tl), ("last", last), ("status", status)):
        assert same(v.cpu().numpy(), o[k]), k
    assert (o["traj_len"] > max_pts).any() and (o["status"] != 0).any()


@pytest.mark.gpu
def test_gpu_reference_style_program_matches_oracle(tmp_path):
    exe = _build_cpp(tmp_path)
    st, tg, pa = synth.mptg_inputs(300, seed=21)
    keep = np.flatnonzero(OM.optimize(st, tg, pa)["status"] <= OM.MAX_ITER_REACHED)[:40]
    d0 = MC.demo()
    st, tg, pa = (np.ascontiguousarray(np.concatenate([a[:, keep], b], axis=1)) for a, b in zip((st, tg, pa), d0))
    m = st.shape[1]
    blob = np.concatenate([np.float32([m]), np.concatenate([st, tg, pa], axis=0).T.reshape(-1)]).astype(np.float32)
    blob.tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    o = OM.optimize(st, tg, pa, max_pts=4096)
    g = OM.generate(st, o["param"])
    p = 0
    for i in range(m):
        assert same(out[p:p + 4], o["param"][:, i]); p += 4
        k = int(out[p]); p += 1
        assert k == o["traj_len"][i]
        assert same(out[p:p + 3 * k], o["traj"][:3 * k, i]); p += 3 * k
        assert same(out[p:p + 3], g["last"][:, i]); p += 3
    assert p == out.size


TANF_CENSUS_CU = r"""
// crb_tanf_libm on the device for every float of [lo, hi) (both signs, in chunks), checked on the host by the
// checker's crb_oracle_libm_tanf_check (argv[3] = liboracle_mptg.so).  Prints the number of mismatches.
#include <dlfcn.h>

#include "crb_common.cuh"
__global__ void census(unsigned lo, unsigned long long count, float* out) {
  for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned b = (lo + (unsigned)(k >> 1)) | ((k & 1) ? 0x80000000u : 0u);
    out[k] = crb_tanf_libm(__uint_as_float(b));
  }
}
int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const unsigned lo = (unsigned)strtoul(argv[1], 0, 0), hi = (unsigned)strtoul(argv[2], 0, 0);
  void* so = dlopen(argv[3], RTLD_NOW);
  if (!so) return 2;
  typedef long long (*check_fn)(unsigned, unsigned, const float*);
  check_fn check = (check_fn)dlsym(so, "crb_oracle_libm_tanf_check");
  if (!check) return 2;
  const unsigned chunk = 1u << 26;
  float *d, *h;
  if (cudaMalloc(&d, 2ull * chunk * 4) != cudaSuccess || cudaMallocHost(&h, 2ull * chunk * 4) != cudaSuccess) return 3;
  long long bad = 0;
  for (unsigned a = lo; a < hi; a = (hi - a > chunk) ? a + chunk : hi) {
    const unsigned b = (hi - a > chunk) ? a + chunk : hi;
    census<<<2048, 256>>>(a, 2ull * (b - a), d);
    if (cudaMemcpy(h, d, 2ull * (b - a) * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 4;
    bad += check(a, b, h);
  }
  printf("%lld\n", bad);
  cudaFreeHost(h);
  cudaFree(d);
  return 0;
}
"""


@pytest.mark.gpu
def test_gpu_tanf_census_against_the_checker(tmp_path):
    """crb_tanf_libm on the device against the checker's C restatement (itself pinned to glibc 2.39 by the CPU
    census), not the libm of the machine the test runs on: every float with |x| < 120."""
    src = tmp_path / "census.cu"
    src.write_text(TANF_CENSUS_CU)
    exe = tmp_path / "census"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                           "-I", os.path.join(ROOT, "cpprobotics_b200", "csrc"), str(src), "-o", str(exe), "-ldl"])
    out = subprocess.check_output([str(exe), "0x0", "0x42F00000", OM.LIB_PATH], text=True)
    assert int(out.strip()) == 0
