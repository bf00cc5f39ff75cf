"""CPU: the task state machine of the resident-slot MPC kernel (cpprobotics_b200/csrc/crb_mpc_tasks.cu).

tests/cpp/mpc_tasks_sim.cpp compiles the kernel's own arithmetic header (crb_mpc_core.cuh: the per-sweep task
functions the CUDA kernel inlines) with g++ and emulates one CTA: S problem slots, a problem counter, sweeps
handed out in a pseudo-random order.  The outputs must equal oracle/crb_oracle_mpc.c BIT FOR BIT for every
schedule and every slot count: a problem's arithmetic may not depend on which warp ran which of its sweeps.
(The lock / ballot scheduling code itself only exists on the GPU and is covered by the -m gpu parity tests.)
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mpc_cases as MC
from cpprobotics_b200 import synth
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "mpc_tasks_sim.cpp")
HDR = os.path.join(ROOT, "cpprobotics_b200", "csrc", "crb_mpc_core.cuh")


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mpcsim") / "libmpc_tasks_sim.so")
    fma = ["-mfma"] if " fma " in open("/proc/cpuinfo").read() else []
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fno-strict-aliasing", "-Wall",
                           "-DCRB_HOST_SIM", "-shared", "-fPIC", SRC, "-o", so] + fma)
    L = C.CDLL(so)
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    L.mpc_tasks_sim_solve.argtypes = [C.c_int64, C.c_int, f32p, f32p, C.c_void_p, C.POINTER(O.MpcParams),
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_uint64, C.c_void_p, C.c_void_p]
    return L


def run_sim(L, st, xref, T, prm, S, seed, u_init=None, hint=None):
    st = np.ascontiguousarray(st, np.float32)
    xref = np.ascontiguousarray(xref, np.float32)
    n = st.shape[1]
    out = dict(sol=np.full((4 * T + 2 * (T - 1), n), np.nan, np.float32), u0=np.full((2, n), np.nan, np.float32),
               cost=np.full(n, np.nan, np.float32), status=np.full(n, -1, np.int32), iters=np.full(n, -1, np.int32))
    ui = None
    if u_init is not None:
        u_init = np.ascontiguousarray(u_init, np.float32)
        ui = u_init.ctypes.data
    counts = np.zeros(3, np.int64)
    hp = None
    if hint is not None:
        hint = np.ascontiguousarray(hint, np.int32)
        assert hint.shape == (n,)
        hp = hint.ctypes.data
    rc = L.mpc_tasks_sim_solve(n, T, st, xref, ui, C.byref(prm), out["sol"].ctypes.data, out["u0"].ctypes.data,
                               out["cost"].ctypes.data, out["status"].ctypes.data, out["iters"].ctypes.data, S, seed,
                               counts.ctypes.data, hp)
    assert rc == 0
    out["tasks"] = counts
    return out


def case(n, T, seed=0xC0FFEE, dt=0.2):
    course = synth.mpc_course()
    st, pind = synth.mpc_states(n, seed=seed, course=course)
    xref, _ = synth.mpc_xref_numpy(st, pind, T, course=course, dt=dt)
    return st, xref


def same(got, want):
    for k in ("status", "iters", "u0", "cost", "sol"):
        assert np.array_equal(got[k], want[k]), k


@pytest.mark.parametrize("n,T,S,seed", [(1, 20, 224, 1), (700, 20, 224, 2), (700, 20, 33, 3), (257, 6, 64, 4),
                                         (300, 32, 140, 5), (97, 2, 8, 6), (500, 20, 1, 7)])
def test_task_machine_is_bit_exact_for_any_schedule(sim, n, T, S, seed):
    st, xref = case(n, T)
    prm = O.mpc_params()
    want = O.mpc_solve_batched(st, xref, T, prm)
    got = run_sim(sim, st, xref, T, prm, S, seed)
    same(got, want)
    # every problem was refilled once; sweeps were really regrouped (more than one task of each kind)
    assert got["tasks"].min() >= 1


@pytest.mark.parametrize("S", [64, 17])
@pytest.mark.parametrize("T", [7, 20])
@pytest.mark.parametrize("name", ["W", "B", "S"])
def test_task_machine_is_bit_exact_at_non_default_constants(sim, name, T, S):
    """The parameter sets of tests/mpc_cases.py: every weight distinct (W), other model and bounds with the speed
    bound active (B), a slow vehicle (S).  (The simulator fills the kernel's parameter block itself; the GPU tests
    in test_mpc_constants.py check libcrb's own fill.)"""
    over = MC.SETS[name]
    st, xref = case(300, T, seed=T + S, dt=O.plant_constant(O.mpc_params(**over), "dt"))
    prm = O.mpc_params(**over)
    want = O.mpc_solve_batched(st, xref, T, prm)
    got = run_sim(sim, st, xref, T, prm, S, seed=T * S)
    same(got, want)
    assert (want["status"] == 0).all() and got["tasks"].min() >= 1


@pytest.mark.parametrize("kind", ["iters", "random", "constant", "negative_and_huge", "one_long"])
def test_hinted_order_solves_every_problem_once_with_the_same_bits(sim, kind):
    """crb_mpc_solve_batched_hinted starts the ~15 % of the problems with the largest hints first (sorted by decreasing
    hint), then the others.  Whatever the hints are, every problem is solved exactly once (outputs pre-filled with NaN / -1 would
    show a skipped one) and its bits do not depend on the order."""
    n, T = 900, 20
    st, xref = case(n, T)
    prm = O.mpc_params()
    want = O.mpc_solve_batched(st, xref, T, prm)
    rng = np.random.default_rng(11)
    hint = {"iters": want["iters"], "random": rng.integers(0, 40, n), "constant": np.full(n, 7),
            "negative_and_huge": rng.integers(-5, 10_000, n),
            "one_long": np.where(np.arange(n) == 123, 50, 3)}[kind].astype(np.int32)
    for S, seed in ((224, 1), (33, 2)):
        got = run_sim(sim, st, xref, T, prm, S, seed, hint=hint)
        same(got, want)


def test_two_schedules_agree_and_line_search_limits(sim):
    st, xref = case(400, 20, seed=99)
    for over in (dict(max_ls=8), dict(max_ls=0), dict(max_iter=3), dict(max_iter=0), dict(du_th=1e-2, j_tol=0.0)):
        prm = O.mpc_params(**over)
        want = O.mpc_solve_batched(st, xref, 20, prm)
        a = run_sim(sim, st, xref, 20, prm, 200, 11)
        b = run_sim(sim, st, xref, 20, prm, 48, 12)
        same(a, want)
        same(b, want)


def test_warm_start_speed_limits_and_nonfinite_inputs(sim):
    n, T = 300, 20
    st, xref = case(n, T, seed=7)
    xref = xref.copy()
    xref[3::4] = 20.0                       # ask for 20 m/s > 55/3.6: the speed bound (:298-301) is active
    st = st.copy(); st[3] = 14.9 + 0.3 * (np.arange(n) % 3)
    rng = np.random.default_rng(0)
    u_init = rng.uniform(-1.2, 1.2, size=(2 * (T - 1), n)).astype(np.float32)  # partly infeasible
    st[2, 5] = np.nan
    xref[8, 9] = np.inf
    prm = O.mpc_params(max_iter=30, max_ls=8)
    want = O.mpc_solve_batched(st, xref, T, prm, u_init=u_init)
    got = run_sim(sim, st, xref, T, prm, 100, 5, u_init=u_init)
    assert got["status"][5] == 3 and got["status"][9] == 3
    assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["iters"], want["iters"])
    ok = got["status"] != 3
    for k in ("u0", "cost", "sol"):
        assert np.array_equal(got[k][..., ok], want[k][..., ok]), k
