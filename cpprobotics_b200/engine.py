"""Host-side mirror of the reference's hot functions, batched, on top of the C ABI (libcrb.so).

Method names follow the reference functions they replace:

  Engine.ekf_estimation      <- ekf_estimation()       src/extended_kalman_filter.cpp:64-78
  Engine.pf_predict_weight   <- pf_localization() loop  src/particle_filter.cpp:81-102
  Engine.pf_estimate         <- pf_localization() tail  src/particle_filter.cpp:104-107
  Engine.mpc_solve           <- mpc_solve()             src/model_predictive_control.cpp:255-346
  Engine.mpc_plant_update    <- update()                src/model_predictive_control.cpp:69-81
  Engine.calc_ref_trajectory <- calc_ref_trajectory()   src/model_predictive_control.cpp:130-170
  Engine.dwa_control         <- dwa_control()           src/dynamic_window_approach.cpp:148-155
  Engine.dwa_motion          <- motion()                src/dynamic_window_approach.cpp:43-50
  Engine.mptg_optimize       <- TrajectoryOptimizer::optimizer_traj()  include/trajectory_optimizer.h:53-128
  Engine.mptg_generate_trajectory <- MotionModel::generate_trajectory() include/motion_model.h:110-131

All arrays are SoA field-major float32 (`[fields, n]`, C-contiguous); see include/crb.h.  Methods
without a suffix take CUDA tensors (torch is only the device allocator / stream owner); `*_host`
methods take host arrays (numpy or CPU torch tensors, ideally pinned) and run the chunked
copy/compute pipeline inside libcrb.  Nothing here computes: every call goes through the C ABI, and
raises when libcrb.so or an H100 is missing.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from ._lib import DwaParams, EkfParams, MpcParams, MptgParams, PfParams, check, load_library

try:  # torch is the device-memory / stream / distributed plumbing, never the compute path
    import torch
except Exception:  # pragma: no cover
    torch = None


def ekf_default_params() -> EkfParams:
    p = EkfParams()
    load_library().crb_ekf_default_params(C.byref(p))
    return p


def pf_default_params() -> PfParams:
    p = PfParams()
    load_library().crb_pf_default_params(C.byref(p))
    return p


def mpc_default_params() -> MpcParams:
    p = MpcParams()
    load_library().crb_mpc_default_params(C.byref(p))
    return p


def dwa_default_params() -> DwaParams:
    p = DwaParams()
    load_library().crb_dwa_default_params(C.byref(p))
    return p


def mptg_default_params() -> MptgParams:
    p = MptgParams()
    load_library().crb_mptg_default_params(C.byref(p))
    return p


def _ptr(a, dtype, *, device: Optional[bool], name: str) -> int:
    """Raw pointer of a contiguous array after checking dtype and placement."""
    if a is None:
        return None
    if torch is not None and isinstance(a, torch.Tensor):
        want = {np.float32: torch.float32, np.int32: torch.int32, np.float64: torch.float64}[dtype]
        if a.dtype != want:
            raise TypeError(f"{name}: expected {want}, got {a.dtype}")
        if not a.is_contiguous():
            raise ValueError(f"{name}: tensor must be contiguous")
        if device is True and not a.is_cuda:
            raise ValueError(f"{name}: expected a CUDA tensor")
        if device is False and a.is_cuda:
            raise ValueError(f"{name}: expected a host tensor")
        return a.data_ptr()
    if isinstance(a, np.ndarray):
        if device is True:
            raise ValueError(f"{name}: expected a CUDA tensor, got numpy")
        if a.dtype != dtype:
            raise TypeError(f"{name}: expected {dtype}, got {a.dtype}")
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError(f"{name}: array must be C-contiguous")
        return a.ctypes.data
    raise TypeError(f"{name}: unsupported array type {type(a)}")


def _shape(a, fields: int, n: int, name: str) -> None:
    shp = tuple(a.shape)
    if shp != (fields, n) and not (fields == 1 and shp == (n,)):
        raise ValueError(f"{name}: expected shape ({fields}, {n}), got {shp}")


class Engine:
    """One context = one GPU = one stream.  One process per GPU creates one Engine."""

    def __init__(self, device: Optional[int] = None, use_torch_stream: bool = True):
        self.lib = load_library()
        h = C.c_void_p()
        check(self.lib.crb_init(C.byref(h), -1 if device is None else int(device)), "crb_init")
        self.ctx = h
        self.device = device
        self._torch_stream = use_torch_stream and torch is not None
        if self._torch_stream:
            self.bind_current_stream()

    def bind_current_stream(self) -> None:
        """Enqueue on torch's current stream so torch events / collectives order with our kernels."""
        st = torch.cuda.current_stream(self.device).cuda_stream
        check(self.lib.crb_set_stream(self.ctx, C.c_void_p(st)), "crb_set_stream")

    def close(self) -> None:
        if getattr(self, "ctx", None):
            self.lib.crb_destroy(self.ctx)
            self.ctx = None

    def __del__(self):  # best effort
        try:
            self.close()
        except Exception:
            pass

    def sync(self) -> None:
        check(self.lib.crb_sync(self.ctx), "crb_sync")

    @property
    def launches(self) -> int:
        return int(self.lib.crb_launch_count(self.ctx))

    # ---- EKF --------------------------------------------------------------------------------------
    def _ekf(self, fn, dev, x, P, z, u, params, n_steps):
        n = int(x.shape[-1])
        _shape(x, 4, n, "x"); _shape(P, 16, n, "P")
        _shape(z, 2 * n_steps, n, "z"); _shape(u, 2 * n_steps, n, "u")
        prm = params if params is not None else ekf_default_params()
        check(fn(self.ctx, n, _ptr(x, np.float32, device=dev, name="x"),
                 _ptr(P, np.float32, device=dev, name="P"), _ptr(z, np.float32, device=dev, name="z"),
                 _ptr(u, np.float32, device=dev, name="u"), C.byref(prm), int(n_steps)),
              "crb_ekf_step_batched")

    def ekf_estimation(self, x, P, z, u, params: Optional[EkfParams] = None, n_steps: int = 1):
        """In place on x [4,n], P [16,n] (column-major 4x4); z, u [2*n_steps, n].  CUDA tensors."""
        self._ekf(self.lib.crb_ekf_step_batched, True, x, P, z, u, params, n_steps)

    def ekf_estimation_host(self, x, P, z, u, params: Optional[EkfParams] = None, n_steps: int = 1):
        self._ekf(self.lib.crb_ekf_step_batched_host, False, x, P, z, u, params, n_steps)

    # ---- PF ---------------------------------------------------------------------------------------
    # resident-state tracking: the reference's time loop (:171-183), 16 B in / 16 B out per update
    def ekf_track_open(self, x0, P0):
        n = int(x0.shape[-1])
        _shape(x0, 4, n, "x0"); _shape(P0, 16, n, "P0")
        h = C.c_void_p()
        check(self.lib.crb_ekf_track_open(self.ctx, n, _ptr(x0, np.float32, device=False, name="x0"),
                                          _ptr(P0, np.float32, device=False, name="P0"), C.byref(h)),
              "crb_ekf_track_open")
        return h

    def ekf_track_step(self, trk, z, u, params: Optional[EkfParams] = None, x_out=None, async_: bool = False):
        prm = params if params is not None else ekf_default_params()
        check(self.lib.crb_ekf_track_step(self.ctx, trk, _ptr(z, np.float32, device=False, name="z"),
                                          _ptr(u, np.float32, device=False, name="u"), C.byref(prm),
                                          _ptr(x_out, np.float32, device=False, name="x_out"), int(bool(async_))),
              "crb_ekf_track_step")

    def ekf_track_sync(self, trk):
        check(self.lib.crb_ekf_track_sync(self.ctx, trk), "crb_ekf_track_sync")

    def ekf_track_read(self, trk, x=None, P=None):
        check(self.lib.crb_ekf_track_read(self.ctx, trk, _ptr(x, np.float32, device=False, name="x"),
                                          _ptr(P, np.float32, device=False, name="P")), "crb_ekf_track_read")

    def ekf_track_close(self, trk):
        check(self.lib.crb_ekf_track_close(self.ctx, trk), "crb_ekf_track_close")

    def _pf(self, fn, dev, px, pw, noise, landmarks, params, seed):
        n = int(px.shape[-1])
        _shape(px, 4, n, "px"); _shape(pw, 1, n, "pw")
        if noise is not None:
            _shape(noise, 2, n, "noise")
        lm = np.ascontiguousarray(np.asarray(landmarks, dtype=np.float32).reshape(-1, 3))
        prm = params if params is not None else pf_default_params()
        check(fn(self.ctx, n, _ptr(px, np.float32, device=dev, name="px"),
                 _ptr(pw, np.float32, device=dev, name="pw"),
                 _ptr(noise, np.float32, device=dev, name="noise"), C.c_uint64(int(seed)),
                 lm.ctypes.data, int(lm.shape[0]), C.byref(prm)), "crb_pf_predict_weight_batched")

    def pf_predict_weight(self, px, pw, noise, landmarks, params: Optional[PfParams] = None,
                          seed: int = 0):
        """In place on px [4,n], pw [n].  noise [2,n] or None (in-kernel Philox).  landmarks: host
        array of rows (range, lx, ly)."""
        self._pf(self.lib.crb_pf_predict_weight_batched, True, px, pw, noise, landmarks, params, seed)

    def pf_predict_weight_host(self, px, pw, noise, landmarks, params: Optional[PfParams] = None,
                               seed: int = 0):
        self._pf(self.lib.crb_pf_predict_weight_batched_host, False, px, pw, noise, landmarks,
                 params, seed)

    def pf_estimate(self, px, pw):
        """Normalises pw in place; returns (xEst[4], PEst[4,4], sum_w)."""
        n = int(px.shape[-1])
        xe = np.zeros(4, np.float32)
        pe = np.zeros(16, np.float32)
        sw = C.c_double(0.0)
        check(self.lib.crb_pf_estimate(self.ctx, n, _ptr(px, np.float32, device=True, name="px"),
                                       _ptr(pw, np.float32, device=True, name="pw"),
                                       xe.ctypes.data, pe.ctypes.data, C.addressof(sw)),
              "crb_pf_estimate")
        return xe, pe.reshape(4, 4).T.copy(), sw.value

    def pf_resample(self, px, pw, uniforms=None, seed: int = 0, nth: Optional[float] = None, px_tmp=None):
        """resampling() :120-148.  In place on px [4,n], pw [n]; returns (did_resample, Neff)."""
        n = int(px.shape[-1])
        _shape(px, 4, n, "px"); _shape(pw, 1, n, "pw")
        if px_tmp is None:
            px_tmp = torch.empty_like(px)
        did = C.c_int(0)
        neff = C.c_double(0.0)
        check(self.lib.crb_pf_resample(
            self.ctx, n, _ptr(px, np.float32, device=True, name="px"), _ptr(pw, np.float32, device=True, name="pw"),
            _ptr(px_tmp, np.float32, device=True, name="px_tmp"),
            _ptr(uniforms, np.float32, device=True, name="uniforms"), C.c_uint64(int(seed)),
            C.c_float(n // 2 if nth is None else nth), C.addressof(did), C.addressof(neff)), "crb_pf_resample")
        return bool(did.value), neff.value

    def pf_step(self, px, pw, px_next, noise, landmarks, params: Optional[PfParams] = None, seed: int = 0,
                uniforms=None, resample_seed: int = 0, nth: Optional[float] = None, result=None):
        """One complete filter iteration on the device (crb_pf_step): predict + weight on px / pw, estimate,
        resampling decided on the device, next particle set in px_next.  Returns the float64 CUDA result tensor
        [xEst(4) | PEst(16, column-major) | sum_w | Neff | resampled | sum wn^2]; nothing is synchronised."""
        n = int(px.shape[-1])
        _shape(px, 4, n, "px"); _shape(px_next, 4, n, "px_next")
        lm = np.ascontiguousarray(landmarks, np.float32).reshape(-1, 3)
        prm = params if params is not None else pf_default_params()
        if result is None:
            result = torch.zeros(_lib.CRB_PF_RESULT_LEN, dtype=torch.float64, device=px.device)
        check(self.lib.crb_pf_step(
            self.ctx, n, _ptr(px, np.float32, device=True, name="px"), _ptr(pw, np.float32, device=True, name="pw"),
            _ptr(px_next, np.float32, device=True, name="px_next"),
            _ptr(noise, np.float32, device=True, name="noise"), C.c_uint64(int(seed)),
            lm.ctypes.data if lm.size else None, int(lm.shape[0]), C.byref(prm),
            _ptr(uniforms, np.float32, device=True, name="uniforms"), C.c_uint64(int(resample_seed)),
            C.c_float(n // 2 if nth is None else nth), _ptr(result, np.float64, device=True, name="result")),
            "crb_pf_step")
        return result

    # ---- MPC --------------------------------------------------------------------------------------
    def _mpc(self, fn, dev, x0, xref, T, params, u_init, sol, u0, cost, status, iters, hint=None):
        n = int(x0.shape[-1])
        _shape(x0, 4, n, "x0"); _shape(xref, 4 * T, n, "xref")
        nu = 2 * (T - 1)
        if u_init is not None:
            _shape(u_init, nu, n, "u_init")
        if sol is not None:
            _shape(sol, 4 * T + nu, n, "sol")
        if u0 is not None:
            _shape(u0, 2, n, "u0")
        prm = params if params is not None else mpc_default_params()
        check(fn(self.ctx, n, int(T), _ptr(x0, np.float32, device=dev, name="x0"),
                 _ptr(xref, np.float32, device=dev, name="xref"),
                 _ptr(u_init, np.float32, device=dev, name="u_init"), C.byref(prm),
                 _ptr(sol, np.float32, device=dev, name="sol"),
                 _ptr(u0, np.float32, device=dev, name="u0"),
                 _ptr(cost, np.float32, device=dev, name="cost"),
                 _ptr(status, np.int32, device=dev, name="status"),
                 _ptr(iters, np.int32, device=dev, name="iters"),
                 *(() if hint is None else (_ptr(hint, np.int32, device=dev, name="hint"),))),
              "crb_mpc_solve_batched")

    def mpc_solve(self, x0, xref, T: int, params: Optional[MpcParams] = None, u_init=None, sol=None,
                  u0=None, cost=None, status=None, iters=None):
        """x0 [4,n], xref [4T,n] (field 4t+k) -> any of sol [4T+2(T-1),n], u0 [2,n]=(a0,delta0),
        cost [n], status [n] int32, iters [n] int32 (pre-allocated CUDA tensors or None)."""
        self._mpc(self.lib.crb_mpc_solve_batched, True, x0, xref, T, params, u_init, sol, u0, cost,
                  status, iters)

    def mpc_solve_hinted(self, x0, xref, T: int, hint, params: Optional[MpcParams] = None, u_init=None,
                         sol=None, u0=None, cost=None, status=None, iters=None):
        """mpc_solve with a scheduling hint per problem (int32 [n] CUDA tensor, e.g. the previous solve's `iters`):
        problems with the largest hints start first; the results are bit-identical to mpc_solve."""
        if int(hint.shape[-1]) != int(x0.shape[-1]):
            raise ValueError("hint must have one entry per problem")
        self._mpc(self.lib.crb_mpc_solve_batched_hinted, True, x0, xref, T, params, u_init, sol, u0, cost,
                  status, iters, hint=hint)

    def mpc_solve_host(self, x0, xref, T: int, params: Optional[MpcParams] = None, u_init=None,
                       sol=None, u0=None, cost=None, status=None, iters=None):
        self._mpc(self.lib.crb_mpc_solve_batched_host, False, x0, xref, T, params, u_init, sol, u0,
                  cost, status, iters)

    def mpc_plant_update(self, state, u0, params: Optional[MpcParams] = None):
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(u0, 2, n, "u0")
        prm = params if params is not None else mpc_default_params()
        check(self.lib.crb_mpc_plant_update_batched(
            self.ctx, n, _ptr(state, np.float32, device=True, name="state"),
            _ptr(u0, np.float32, device=True, name="u0"), C.byref(prm)),
            "crb_mpc_plant_update_batched")

    def calc_ref_trajectory(self, state, cx, cy, cyaw, sp, dl: float, target_ind, xref, T: int,
                            params: Optional[MpcParams] = None):
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(xref, 4 * T, n, "xref")
        nc = int(cx.shape[0])
        prm = params if params is not None else mpc_default_params()
        check(self.lib.crb_mpc_calc_ref_trajectory_batched(
            self.ctx, n, int(T), _ptr(state, np.float32, device=True, name="state"),
            _ptr(cx, np.float32, device=True, name="cx"), _ptr(cy, np.float32, device=True, name="cy"),
            _ptr(cyaw, np.float32, device=True, name="cyaw"),
            _ptr(sp, np.float32, device=True, name="sp"), nc, C.c_float(dl),
            _ptr(target_ind, np.int32, device=True, name="target_ind"),
            _ptr(xref, np.float32, device=True, name="xref"), C.byref(prm)),
            "crb_mpc_calc_ref_trajectory_batched")

    # ---- LQR --------------------------------------------------------------------------------------
    def dlqr(self, A, B, Q, R, nx: int, nu: int, maxiter: int = 150, eps: float = 0.01, K=None, X=None,
             iters=None):
        """solve_DARE + dlqr (lqr_steer_control.cpp:75-96 / lqr_speed_steer_control.cpp:85-106).
        A [nx*nx,n], B [nx*nu,n] per agent, Q [nx*nx], R [nu*nu] shared: CUDA tensors.  Returns K [nu*nx,n]."""
        n = int(A.shape[-1])
        _shape(A, nx * nx, n, "A"); _shape(B, nx * nu, n, "B")
        if K is None:
            K = torch.empty((nu * nx, n), dtype=torch.float32, device=A.device)
        check(self.lib.crb_lqr_dlqr_batched(
            self.ctx, n, int(nx), int(nu), _ptr(A, np.float32, device=True, name="A"),
            _ptr(B, np.float32, device=True, name="B"), _ptr(Q, np.float32, device=True, name="Q"),
            _ptr(R, np.float32, device=True, name="R"), int(maxiter), C.c_float(eps),
            _ptr(K, np.float32, device=True, name="K"), _ptr(X, np.float32, device=True, name="X"),
            _ptr(iters, np.int32, device=True, name="iters")), "crb_lqr_dlqr_batched")
        return K

    # ---- DWA ----------------------------------------------------------------------------------------
    def dwa_control(self, x, u, goal, obstacles, params: Optional[DwaParams] = None, cost=None, best=None,
                    traj=None):
        """dwa_control() for n robots: x [5,n] (x, y, yaw, v, yawrate), u [2,n] in/out (only u[1] is read),
        goal [2,n], obstacles [n_ob,2] shared by all robots; optional outputs cost [n] f32, best [n] int32 (flat
        v-major sample index or -1), traj [5*n_pts,n] (n_pts from dwa_rollout_points).  CUDA tensors; only
        enqueues."""
        n = int(x.shape[-1])
        _shape(x, 5, n, "x"); _shape(u, 2, n, "u"); _shape(goal, 2, n, "goal")
        if obstacles.dim() != 2 or int(obstacles.shape[1]) != 2:
            raise ValueError(f"obstacles: expected shape (n_ob, 2), got {tuple(obstacles.shape)}")
        prm = params if params is not None else dwa_default_params()
        if cost is not None:
            _shape(cost, 1, n, "cost")
        if best is not None:
            _shape(best, 1, n, "best")
        if traj is not None:
            _shape(traj, 5 * self.dwa_rollout_points(prm), n, "traj")
        check(self.lib.crb_dwa_control_batched(
            self.ctx, n, _ptr(x, np.float32, device=True, name="x"), _ptr(u, np.float32, device=True, name="u"),
            _ptr(goal, np.float32, device=True, name="goal"),
            _ptr(obstacles, np.float32, device=True, name="obstacles"), int(obstacles.shape[0]), C.byref(prm),
            _ptr(cost, np.float32, device=True, name="cost"), _ptr(best, np.int32, device=True, name="best"),
            _ptr(traj, np.float32, device=True, name="traj")), "crb_dwa_control_batched")

    def dwa_rollout_points(self, params: Optional[DwaParams] = None) -> int:
        """Points per rollout (steps + 1): 32 for the reference's Config."""
        k = C.c_int(0)
        prm = params if params is not None else dwa_default_params()
        check(self.lib.crb_dwa_rollout_points(C.byref(prm), C.byref(k)), "crb_dwa_rollout_points")
        return int(k.value)

    def dwa_motion(self, x, u, dt: Optional[float] = None):
        """motion() in place on x [5,n] with u [2,n]; dt defaults to the reference's Config.dt."""
        n = int(x.shape[-1])
        _shape(x, 5, n, "x"); _shape(u, 2, n, "u")
        d = dwa_default_params().dt if dt is None else dt
        check(self.lib.crb_dwa_motion_batched(self.ctx, n, _ptr(x, np.float32, device=True, name="x"),
                                              _ptr(u, np.float32, device=True, name="u"), C.c_float(d)),
              "crb_dwa_motion_batched")

    # ---- model-predictive trajectory generation ---------------------------------------------------------
    @staticmethod
    def mptg_default_params() -> MptgParams:
        """The demo's base_l, ds, max_iter, cost_th and h_step (src/model_predictive_trajectory_generator.cpp)."""
        return mptg_default_params()

    def mptg_optimize(self, state, target, param, params: Optional[MptgParams] = None, traj=None, traj_len=None,
                      cost=None, status=None, iters=None):
        """optimizer_traj() for n problems: state [4,n] (x, y, yaw, v), target [3,n] (x, y, yaw), param [4,n] in/out
        (distance, steering_sequence[0..2]).  Optional outputs: traj [3*max_pts,n] (max_pts = traj.shape[0] // 3; the
        first min(traj_len, max_pts) points are written), traj_len [n] int32, cost [n] f32, status [n] int32
        (CRB_MPTG_*), iters [n] int32.  CUDA tensors; only enqueues."""
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(target, 3, n, "target"); _shape(param, 4, n, "param")
        prm = params if params is not None else mptg_default_params()
        max_pts = self._mptg_max_pts(traj, n)
        for a, name in ((traj_len, "traj_len"), (cost, "cost"), (status, "status"), (iters, "iters")):
            if a is not None:
                _shape(a, 1, n, name)
        check(self.lib.crb_mptg_optimize_batched(
            self.ctx, n, _ptr(state, np.float32, device=True, name="state"),
            _ptr(target, np.float32, device=True, name="target"), _ptr(param, np.float32, device=True, name="param"),
            C.byref(prm), max_pts, _ptr(traj, np.float32, device=True, name="traj"),
            _ptr(traj_len, np.int32, device=True, name="traj_len"), _ptr(cost, np.float32, device=True, name="cost"),
            _ptr(status, np.int32, device=True, name="status"), _ptr(iters, np.int32, device=True, name="iters")),
            "crb_mptg_optimize_batched")

    def mptg_generate_trajectory(self, state, param, params: Optional[MptgParams] = None, traj=None, traj_len=None,
                                 last=None, status=None):
        """MotionModel::generate_trajectory() for n parameters: state [4,n], param [4,n]; optional outputs traj
        [3*max_pts,n], traj_len [n] int32, last [3,n] (generate_last_state), status [n] int32.  CUDA tensors."""
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(param, 4, n, "param")
        prm = params if params is not None else mptg_default_params()
        max_pts = self._mptg_max_pts(traj, n)
        if last is not None:
            _shape(last, 3, n, "last")
        for a, name in ((traj_len, "traj_len"), (status, "status")):
            if a is not None:
                _shape(a, 1, n, name)
        check(self.lib.crb_mptg_generate_trajectory_batched(
            self.ctx, n, _ptr(state, np.float32, device=True, name="state"),
            _ptr(param, np.float32, device=True, name="param"), C.byref(prm), max_pts,
            _ptr(traj, np.float32, device=True, name="traj"), _ptr(traj_len, np.int32, device=True, name="traj_len"),
            _ptr(last, np.float32, device=True, name="last"), _ptr(status, np.int32, device=True, name="status")),
            "crb_mptg_generate_trajectory_batched")

    @staticmethod
    def _mptg_max_pts(traj, n: int) -> int:
        if traj is None:
            return 0
        if traj.dim() != 2 or int(traj.shape[0]) % 3 or int(traj.shape[1]) != n:
            raise ValueError(f"traj: expected shape (3*max_pts, {n}), got {tuple(traj.shape)}")
        return int(traj.shape[0]) // 3

    # ---- multi-GPU: the communicator lives in libcrb (crb_comm.cu), not in torch --------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        """Rank 0 calls this and hands the bytes to every rank (any channel: a store, MPI, a socket)."""
        buf = C.create_string_buffer(_lib.CRB_COMM_ID_BYTES)
        check(load_library().crb_comm_get_unique_id(buf), "crb_comm_get_unique_id")
        return buf.raw

    def comm_init(self, world: int, rank: int, unique_id: bytes) -> None:
        """Collective: every rank of the job calls it with the same unique_id."""
        if len(unique_id) != _lib.CRB_COMM_ID_BYTES:
            raise ValueError("unique_id must be CRB_COMM_ID_BYTES long")
        buf = C.create_string_buffer(unique_id, _lib.CRB_COMM_ID_BYTES)
        check(self.lib.crb_comm_init_rank(self.ctx, int(world), int(rank), buf), "crb_comm_init_rank")

    @property
    def world(self) -> int:
        return int(self.lib.crb_comm_world(self.ctx))

    @property
    def rank(self) -> int:
        return int(self.lib.crb_comm_rank(self.ctx))

    def gather_stats(self, stats, out=None):
        """All-gather of CRB_STATS_LEN doubles per rank on the engine's stream -> [world, CRB_STATS_LEN]."""
        w = self.world
        if out is None:
            out = torch.empty((w, _lib.CRB_STATS_LEN), dtype=torch.float64, device=stats.device)
        check(self.lib.crb_gather_stats(self.ctx, _ptr(stats, np.float64, device=True, name="stats"),
                                        _ptr(out, np.float64, device=True, name="out")), "crb_gather_stats")
        return out

    def allreduce_sum(self, buf):
        """In-place sum over ranks of a float64 CUDA tensor (no-op without a communicator)."""
        check(self.lib.crb_comm_allreduce_sum_f64(self.ctx, _ptr(buf, np.float64, device=True, name="buf"),
                                                  int(buf.numel())), "crb_comm_allreduce_sum_f64")
        return buf

    def probe_fp32_peak(self) -> float:
        """Measured non-tensor fp32 FMA rate of this GPU, TFLOP/s (crb_probe.cu)."""
        v = C.c_double()
        check(self.lib.crb_probe_fp32_peak(self.ctx, C.byref(v)), "crb_probe_fp32_peak")
        return float(v.value)

    # ---- stats ------------------------------------------------------------------------------------
    def stats_reduce(self, values, status=None, iters=None, i0: int = 0, out=None):
        """Per-GPU summary of a per-agent f32 array -> float64 CUDA tensor of CRB_STATS_LEN."""
        n = int(values.shape[-1])
        if out is None:
            out = torch.empty(_lib.CRB_STATS_LEN, dtype=torch.float64, device=values.device)
        check(self.lib.crb_stats_reduce(
            self.ctx, n, int(i0), _ptr(values, np.float32, device=True, name="values"),
            _ptr(status, np.int32, device=True, name="status"),
            _ptr(iters, np.int32, device=True, name="iters"),
            _ptr(out, np.float64, device=True, name="out")), "crb_stats_reduce")
        return out
