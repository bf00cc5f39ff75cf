"""The C++ host layer with the reference's own signatures (include/crb/reference_api.hpp).
CPU: it compiles as C++11 against the C ABI, links libcrb.so, and fails loudly without a GPU.
GPU: a reference-style main() (tests/cpp/ref_api_demo.cpp) reproduces the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

from cpprobotics_b200 import synth
from oracle import oracle as O
from toolchain import build_ref_program

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, T, NP = 40, 6, 100


def build(tmp_path):
    return build_ref_program(tmp_path, "ref_api_demo.cpp", werror=False)


def make_inputs():
    x, P, z, u = synth.ekf_inputs(1, seed=77, n_steps=K)
    zu = np.stack([z[0::2, 0], z[1::2, 0], u[0::2, 0], u[1::2, 0]], axis=1).astype(np.float32)  # per step
    course = synth.mpc_course(length=120.0)
    st = np.array([10.2, 20 * np.sin(10.2 / 20) + 0.4, 0.6, 2.5], np.float32)
    px, pw, _ = synth.pf_inputs(NP, seed=77)
    lm = synth.pf_landmarks(4, seed=77)
    buf = [np.float32([K]), zu.reshape(-1), np.float32([len(course[0])]), *course, st, np.float32([5]),
           px.T.reshape(-1), pw, np.float32([len(lm)]), lm.reshape(-1), np.float32([1234])]
    return np.concatenate([np.asarray(b, np.float32).reshape(-1) for b in buf]), zu, course, st, px, pw, lm


def test_every_reference_signature_compiles_and_links(tmp_path):
    """ekf_estimation, pf_localization, resampling, mpc_solve, update, calc_ref_trajectory, solve_DARE and dlqr
    (both LQR demos) with the argument types a CppRobotics main() passes: -std=c++11 -Wall -Werror."""
    build_ref_program(tmp_path, "ref_api_all_signatures.cpp")


def test_compiles_links_and_fails_loudly_without_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: the failure path is covered on the CPU box")
    blob = make_inputs()[0]
    blob.tofile(tmp_path / "in.bin")
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 3 and "no CPU fallback" in r.stderr
    assert not os.path.exists(tmp_path / "out.bin")


@pytest.mark.gpu
def test_reference_style_main_matches_oracle(tmp_path):
    exe = build(tmp_path)
    blob, zu, course, st, px, pw, lm = make_inputs()
    blob.tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    out = np.fromfile(tmp_path / "out.bin", np.float32)
    p = 0

    def take(n):
        nonlocal p
        v = out[p:p + n]; p += n
        return v
    # EKF: config 1 plumbing (one agent, K steps through ekf_estimation)
    xg, Pg = take(4), take(16)
    xo, Po = np.zeros(4, np.float32), np.eye(4, dtype=np.float32).reshape(-1)
    for k in range(K):
        xo, Po = O.ekf_estimation(xo, Po, zu[k, :2], zu[k, 2:])
    assert np.abs(xg - xo).max() <= 1e-5 * np.abs(xo).max() and np.abs(Pg - Po).max() <= 1e-5 * np.abs(Po).max()
    # calc_ref_trajectory: integer index work bit-exact
    xr, ti = take(4 * T), int(take(1)[0])
    xro, tio = O.calc_ref_trajectory(st, *course, 1.0, T, 5)
    assert ti == tio and np.array_equal(xr, xro.reshape(-1))       # col-major 4xT == [T][4]
    # mpc_solve: bit-exact vs the oracle (reference return layout), status word
    sol, status = take(4 * T + 2 * (T - 1)), int(take(1)[0])
    ro = O.mpc_solve_batched(st.reshape(4, 1), xro.reshape(-1, 1), T)
    assert np.array_equal(sol, ro["sol"][:, 0]) and status == ro["status"][0]
    # update(): plant step on the first control
    sg = take(4)
    so = O.plant_update(st, ro["u0"][0, 0], ro["u0"][1, 0])
    assert np.abs(sg - so).max() <= 1e-5 * np.abs(so).max()
    # pf_localization with the reference's by-value generator
    pxg, pwg, xeg, Peg, noise = take(4 * NP).reshape(NP, 4).T, take(NP), take(4), take(16), take(2 * NP)
    nz = np.stack([noise[0::2], noise[1::2]])
    pxo, pwo = O.pf_predict_weight_batched(px, pw, nz, lm)
    assert np.abs(pxg - pxo).max() <= 1e-5 * max(1.0, np.abs(pxo).max())
    pwn, xeo, Peo, _ = O.pf_estimate(pxo, pwo)
    assert np.abs(pwg - pwn).max() <= 2e-3 * np.abs(pwn).max()       # weight conditioning, see DESIGN.md 3.1
    assert np.abs(xeg - xeo).max() <= 1e-3 and np.abs(Peg - Peo.T.reshape(-1)).max() <= 1e-3
    assert p == out.size


# ---- resampling / solve_DARE / dlqr shims: marshalling checked on the CPU through a mock of the C ABI ------------
def _shim_inputs():
    px, pw, noise = synth.pf_inputs(NP, seed=21)
    lm = synth.pf_landmarks(4, seed=21)
    px, pw = O.pf_predict_weight_batched(px, pw, noise, lm)          # peaked weights -> Neff < NP/2 -> resample
    pw = (pw / np.float32(pw.sum())).astype(np.float32)
    A4, B4, Q4, R4 = synth.lqr_inputs(1, 4, seed=5)
    A5, B5, Q5, R5 = synth.lqr_inputs(1, 5, seed=5)
    blob = np.concatenate([np.float32([4321]), px.T.reshape(-1), pw, A4[:, 0], B4[:, 0], Q4.reshape(-1),
                           np.float32([R4.reshape(-1)[0]]), A5[:, 0], B5[:, 0], Q5.reshape(-1),
                           R5.reshape(-1)]).astype(np.float32)
    return blob, px, pw, (A4, B4, Q4, R4), (A5, B5, Q5, R5)


def _check_shim_outputs(out, px, pw, l4, l5):
    gpx, gpw, draws = out[:400].reshape(NP, 4).T, out[400:500], out[500:600]
    assert (draws >= 1.0).all() and (draws <= 2.0).all()
    pxo, pwo, did, _ = O.pf_resample(px, pw, draws.astype(np.float64))
    assert did and np.array_equal(gpx, pxo) and np.array_equal(gpw, pwo)
    p = 600
    for (A, B, Q, R), nx, nu in ((l4, 4, 1), (l5, 5, 2)):
        r = O.dlqr_batched(A, B, Q, R, nx, nu)
        X, K = out[p:p + nx * nx], out[p + nx * nx:p + nx * nx + nu * nx]
        p += nx * nx + nu * nx
        assert np.array_equal(X, r["X"][:, 0]) and np.array_equal(K, r["K"][:, 0])
    assert p == out.size


def test_resampling_and_dlqr_shims_marshal_correctly_through_a_cpu_mock(tmp_path):
    """tests/cpp/mock_crb.c implements the few C-ABI calls these shims make with the oracle, so their AoS<->SoA
    and column-major marshalling and the by-value RNG semantics are executed and checked without a GPU."""
    odir = os.path.join(ROOT, "oracle", "lib")
    obj, exe = str(tmp_path / "mock_crb.o"), str(tmp_path / "shim_check")
    subprocess.check_call(["gcc", "-O1", "-Wall", "-c", os.path.join(ROOT, "tests", "cpp", "mock_crb.c"), "-o", obj])
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "ref_api_shim_check.cpp"), obj, "-L", odir, "-loracle",
                           f"-Wl,-rpath,{odir}", "-o", exe])
    blob, px, pw, l4, l5 = _shim_inputs()
    blob.tofile(tmp_path / "in.bin")
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    _check_shim_outputs(np.fromfile(tmp_path / "out.bin", np.float32), px, pw, l4, l5)
