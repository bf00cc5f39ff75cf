"""Host-side mirror of the reference's hot functions, batched, on top of the C ABI (libcrb.so).

Method names follow the reference functions they replace:

  Engine.ekf_estimation      <- ekf_estimation()       src/extended_kalman_filter.cpp:64-78
  Engine.ekf_estimation_many <- the same, each agent with its own Q, R and DT (ekf_models)
  Engine.pf_predict_weight   <- pf_localization() loop  src/particle_filter.cpp:81-102
  Engine.pf_estimate         <- pf_localization() tail  src/particle_filter.cpp:104-107
  Engine.mpc_solve           <- mpc_solve()             src/model_predictive_control.cpp:255-346
  Engine.mpc_plant_update    <- update()                src/model_predictive_control.cpp:69-81
  Engine.calc_ref_trajectory <- calc_ref_trajectory()   src/model_predictive_control.cpp:130-170
  Engine.calc_ref_trajectory_many <- the same, each agent on its own course (synth.pack_courses)
  Engine.dwa_control         <- dwa_control()           src/dynamic_window_approach.cpp:148-155
  Engine.dwa_control_many    <- the same, each robot among its own obstacles (synth.pack_obstacles)
  Engine.dwa_motion          <- motion()                src/dynamic_window_approach.cpp:43-50
  Engine.dwa_control_fleet, Engine.dwa_motion_fleet <- the same two, each robot with its own Config (dwa_config_table)
  Engine.mptg_optimize       <- TrajectoryOptimizer::optimizer_traj()  include/trajectory_optimizer.h:53-128
  Engine.mptg_generate_trajectory <- MotionModel::generate_trajectory() include/motion_model.h:110-131
  Engine.slp_sample_states   <- calc_{uniform_polar,biased_polar,lane}_states()  src/state_lattice_planner.cpp:29-113
  Engine.slp_search_nearest  <- search_nearest_one_from_lookuptable()            src/state_lattice_planner.cpp:115-135
  Engine.slp_generate_path   <- generate_path()                                  src/state_lattice_planner.cpp:137-155
  slp_load_table             <- main()'s CSVIterator + std::stod reading         src/state_lattice_planner.cpp:214-226
  grid_box_of_obstacles      <- a_star_planning() / dijkstra_star_planning() :115-140 (obstacle cells, the box)
  Engine.grid_obstacle_map   <- calc_obstacle_map()                              src/a_star.cpp:48-78
  Engine.grid_plan           <- a_star_planning() / dijkstra_star_planning()     src/a_star.cpp:110-244, src/dijkstra.cpp
  Engine.grid_obstacle_map_many, Engine.grid_plan_many <- the same, each query on its own map (grid_map_table)
  Engine.rrt_plan            <- RRT::planning()                                  include/rrt.h:75-159
  Engine.rrt_plan_many       <- the same, each query among its own obstacles (synth.pack_obstacles)
  Engine.lqr_steering_control <- lqr_steering_control() (+ calc_nearest_index)   src/lqr_steer_control.cpp:98-133,
                                                                                 src/lqr_speed_steer_control.cpp:108-151
  Engine.lqr_steering_control_many <- the same, each vehicle on its own course (synth.pack_courses)
  Engine.lqr_update          <- update()                 src/lqr_steer_control.cpp:136-146 (same text in both programs)

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
from ._lib import (DwaParams, EkfParams, GridBox, LqrTrackParams, MpcParams, MptgParams, PfParams, RrtParams, check,
                   load_library)

try:  # torch is the device-memory / stream / distributed plumbing, never the compute path
    import torch
except Exception:  # pragma: no cover
    torch = None


def ekf_default_params() -> EkfParams:
    p = EkfParams()
    load_library().crb_ekf_default_params(C.byref(p))
    return p


# one crb_ekf_params record (include/crb.h): a model table is a device array of these
EKF_MODEL_DTYPE = np.dtype({"names": ["dt", "Q", "R"], "formats": [np.float64, (np.float32, 16), (np.float32, 4)],
                            "offsets": [EkfParams.dt.offset, EkfParams.Q.offset, EkfParams.R.offset],
                            "itemsize": C.sizeof(EkfParams)})
assert EKF_MODEL_DTYPE.itemsize == 88 and [EKF_MODEL_DTYPE.fields[k][1] for k in ("dt", "Q", "R")] == [0, 8, 72]


def ekf_models(dt, Q, R) -> np.ndarray:
    """A model table for ekf_estimation_many / ekf_track_step_many: dt [m], Q [m, 16] and R [m, 4] (column-major, as
    crb_ekf_params) packed into m 88-byte records.  Returns a host uint8 array [m, 88]; torch.from_numpy(...).cuda()
    uploads it as it is."""
    d = np.asarray(dt, np.float64).reshape(-1)
    q = np.asarray(Q, np.float32).reshape(d.size, 16)
    r = np.asarray(R, np.float32).reshape(d.size, 4)
    if d.size < 1:
        raise ValueError("a model table needs at least one model")
    t = np.zeros(d.size, EKF_MODEL_DTYPE)
    t["dt"], t["Q"], t["R"] = d, q, r
    return t.view(np.uint8).reshape(d.size, EKF_MODEL_DTYPE.itemsize)


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


DWA_CONFIG_FIELDS = tuple(name for name, _ in DwaParams._fields_)   # one crb_dwa_params record: 12 float32


def dwa_config_table(params) -> np.ndarray:
    """A config table for dwa_control_fleet: a sequence of DwaParams packed into float32 [m, 12], one 48-byte
    crb_dwa_params record per row in the struct's order.  Returns a host array; torch.from_numpy(...).cuda() uploads it
    as it is.  Records are not checked here: the kernel gives a robot on a refused record CRB_DWA_BAD_CONFIG."""
    rows = [[getattr(p, k) for k in DWA_CONFIG_FIELDS] for p in params]
    if not rows:
        raise ValueError("a config table needs at least one record")
    return np.ascontiguousarray(np.asarray(rows, np.float32).reshape(len(rows), len(DWA_CONFIG_FIELDS)))


def mptg_default_params() -> MptgParams:
    p = MptgParams()
    load_library().crb_mptg_default_params(C.byref(p))
    return p


def slp_default_params():
    """The state lattice planner's optimizer settings and start speed (src/state_lattice_planner.cpp:22-24,
    :146-148): (MptgParams, CONST_V)."""
    p, v = MptgParams(), C.c_float(0.0)
    load_library().crb_slp_default_params(C.byref(p), C.byref(v))
    return p, float(v.value)


def rrt_default_params() -> RrtParams:
    """RRT's constructor defaults (expand_dis 1.0, goal_sample_rate 5, max_iter 500) and the demo's rand_area {-2, 15}."""
    p = RrtParams()
    load_library().crb_rrt_default_params(C.byref(p))
    return p


def lqr_track_default_params(nx: int) -> LqrTrackParams:
    """The LQR programs' constants for nx = 4 (lqr_steer_control) or 5 (lqr_speed_steer_control): dt 0.1, wheelbase
    0.5, max_steer 45/180*pi (doubles), Q = I, R = I or 1, maxiter 150, eps 0.01f."""
    p = LqrTrackParams()
    load_library().crb_lqr_track_default_params(C.byref(p), int(nx))
    return p


def grid_box_of_obstacles(ox, oy, reso: float) -> GridBox:
    """The box of cells [min, max) of an obstacle list, as the planners compute it (src/a_star.cpp:115-140): every
    obstacle rounded as (int)round(o * 1.0 / reso) in double.  ox, oy host arrays (float32); no device needed."""
    x = np.ascontiguousarray(ox, np.float32)
    y = np.ascontiguousarray(oy, np.float32)
    if x.shape != y.shape or x.ndim != 1:
        raise ValueError(f"ox, oy: expected two 1-D arrays of one length, got {x.shape} and {y.shape}")
    b = GridBox()
    check(load_library().crb_grid_box_of_obstacles(x.size, x.ctypes.data, y.ctypes.data, float(reso), C.byref(b)),
          "crb_grid_box_of_obstacles")
    return b


def grid_map_table(boxes, reso):
    """The map table of grid_obstacle_map_many / grid_plan_many for boxes int [n_maps, 4] (min_x, min_y, max_x, max_y)
    and reso [n_maps]: (boxes int32 [n_maps, 4], reso float32 [n_maps], map_off int64 [n_maps + 1], max_cells), map m
    being bytes [map_off[m], map_off[m + 1]) of the store and max_cells the largest W * H.  Host arrays (numpy); a box
    outside the limits of include/crb.h raises ValueError.  A box per obstacle list comes from grid_box_of_obstacles."""
    b = np.ascontiguousarray(np.asarray(boxes, np.int64).reshape(-1, 4))
    r = np.ascontiguousarray(np.asarray(reso, np.float32).reshape(-1))
    if b.shape[0] < 1 or r.shape != (b.shape[0],):
        raise ValueError(f"boxes, reso: expected [n_maps, 4] and [n_maps] with n_maps >= 1, got {b.shape}, {r.shape}")
    W, H = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
    bad = (W < 1) | (H < 1) | (W > _lib.CRB_GRID_MAX_SIDE) | (H > _lib.CRB_GRID_MAX_SIDE) | (
        W * H > _lib.CRB_GRID_MAX_CELLS)
    if bad.any():
        raise ValueError(f"box {int(np.flatnonzero(bad)[0])} is empty or exceeds CRB_GRID_MAX_SIDE / MAX_CELLS")
    off = np.zeros(b.shape[0] + 1, np.int64)
    off[1:] = np.cumsum(W * H)
    return np.ascontiguousarray(b.astype(np.int32)), r, off, int((W * H).max())


_libc = None


def _strtod(s: str) -> float:
    """std::stod: C's strtod on the field (leading blanks skipped, the longest valid prefix parsed); ValueError where
    stod throws (nothing parsed, or ERANGE)."""
    global _libc
    if _libc is None:
        _libc = C.CDLL(None, use_errno=True)
        _libc.strtod.restype = C.c_double
        _libc.strtod.argtypes = [C.c_char_p, C.POINTER(C.c_char_p)]
    b = s.encode()
    buf = C.create_string_buffer(b)
    end = C.c_char_p()
    C.set_errno(0)
    v = _libc.strtod(buf, C.byref(end))
    if C.cast(end, C.c_void_p).value == C.addressof(buf):
        raise ValueError(f"stod: no conversion of {s!r}")
    if C.get_errno() == 34:  # ERANGE
        raise ValueError(f"stod: {s!r} is out of range")
    return v


def slp_load_table(path) -> np.ndarray:
    """Reads a lookup table the way the reference's main() does (src/state_lattice_planner.cpp:214-226): CSV rows
    split at ',', the first row (the header) skipped, the first 6 fields of each row parsed with std::stod and
    narrowed to float.  Returns float32 [rows, 6] (x, y, yaw, s, km, kf).  A row with fewer than 6 fields, or a field
    stod refuses, raises ValueError."""
    rows = []
    with open(path, "rb") as fh:
        lines = fh.read().decode().split("\n")
    if lines and lines[-1] == "":
        lines.pop()   # the newline that ends the last row starts no row
    for k, line in enumerate(lines[1:], start=2):
        cells = line.split(",")
        if len(cells) < 6:
            raise ValueError(f"{path}:{k}: {len(cells)} fields, 6 needed")
        rows.append([_strtod(c) for c in cells[:6]])
    return np.asarray(rows, np.float64).reshape(-1, 6).astype(np.float32)


def _ptr(a, dtype, *, device: Optional[bool], name: str) -> int:
    """Raw pointer of a contiguous array after checking dtype and placement."""
    if a is None:
        return None
    if torch is not None and isinstance(a, torch.Tensor):
        want = {np.float32: torch.float32, np.int32: torch.int32, np.float64: torch.float64,
                np.uint8: torch.uint8, np.int64: torch.int64}[dtype]
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

    def _ekf_table(self, models, model_of, n, status, dev):
        if tuple(models.shape[1:]) != (EKF_MODEL_DTYPE.itemsize,) or models.shape[0] < 1:
            raise ValueError(f"models: expected [n_models >= 1, {EKF_MODEL_DTYPE.itemsize}] bytes (ekf_models), "
                             f"got {tuple(models.shape)}")
        _shape(model_of, 1, n, "model_of")
        if status is not None:
            _shape(status, 1, n, "status")
        return (_ptr(models, np.uint8, device=dev, name="models"), int(models.shape[0]),
                _ptr(model_of, np.int32, device=dev, name="model_of"),
                _ptr(status, np.int32, device=dev, name="status"))

    def ekf_estimation_many(self, x, P, z, u, models, model_of, n_steps: int = 1, status=None):
        """ekf_estimation with a noise model per agent: agent i steps with models[model_of[i]].  In place on x [4,n],
        P [16,n]; z, u [2*n_steps, n]; models uint8 [n_models, 88] (ekf_models); model_of int32 [n]; status int32 [n]
        or None (CRB_EKF_OK / CRB_EKF_BAD_MODEL).  CUDA tensors."""
        n = int(x.shape[-1])
        _shape(x, 4, n, "x"); _shape(P, 16, n, "P")
        _shape(z, 2 * n_steps, n, "z"); _shape(u, 2 * n_steps, n, "u")
        tab, nm, mof, st = self._ekf_table(models, model_of, n, status, True)
        check(self.lib.crb_ekf_step_many_batched(
            self.ctx, n, _ptr(x, np.float32, device=True, name="x"), _ptr(P, np.float32, device=True, name="P"),
            _ptr(z, np.float32, device=True, name="z"), _ptr(u, np.float32, device=True, name="u"), tab, nm, mof,
            int(n_steps), st), "crb_ekf_step_many_batched")

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

    def ekf_track_step_many(self, trk, z, u, models, model_of, status=None, x_out=None, async_: bool = False):
        """ekf_track_step with a noise model per agent.  z, u, x_out host arrays as in ekf_track_step; models,
        model_of and status CUDA tensors as in ekf_estimation_many, complete on the device before the call (the track
        runs on the context's pipeline streams)."""
        n = int(model_of.shape[-1])
        tab, nm, mof, st = self._ekf_table(models, model_of, n, status, True)
        check(self.lib.crb_ekf_track_step_many(self.ctx, trk, _ptr(z, np.float32, device=False, name="z"),
                                               _ptr(u, np.float32, device=False, name="u"), tab, nm, mof, st,
                                               _ptr(x_out, np.float32, device=False, name="x_out"),
                                               int(bool(async_))),
              "crb_ekf_track_step_many")

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

    def pf_step_many(self, np_per_robot: int, px, pw, px_next, u, observations, z_of, noise=None,
                     params: Optional[PfParams] = None, seed: int = 0, uniforms=None, resample_seed: int = 0,
                     nth: Optional[float] = None, result=None, status=None):
        """pf_step for a fleet (crb_pf_step_many_batched): n_robots independent filters of np_per_robot particles,
        robot r in columns [r*np, (r+1)*np) of px [4, n] / pw [n] / px_next [4, n], n = n_robots * np.  u [2, n_robots]
        holds each robot's control; observations (z, z_off) are the lists' rows z [n_rows, 3] (range, lx, ly) back to
        back and z_off [n_sets + 1] int64 (synth.pack_obstacles); z_of [n_robots] int32, the list of each robot.
        nth defaults to np // 2.  Returns the float64 CUDA result tensor [CRB_PF_RESULT_LEN, n_robots]; status
        [n_robots] int32 (CRB_PF_FLEET_*) is written when given.  Only enqueues."""
        npr = int(np_per_robot)
        nr = int(u.shape[-1])
        n = nr * npr
        _shape(px, 4, n, "px"); _shape(px_next, 4, n, "px_next"); _shape(pw, 1, n, "pw")
        _shape(u, 2, nr, "u"); _shape(z_of, 1, nr, "z_of")
        if noise is not None:
            _shape(noise, 2, n, "noise")
        if uniforms is not None:
            _shape(uniforms, 1, n, "uniforms")
        z, off = observations
        if z.dim() != 2 or int(z.shape[1]) != 3:
            raise ValueError(f"z: expected shape (n_rows, 3), got {tuple(z.shape)}")
        if off.dim() != 1:
            raise ValueError(f"z_off: expected shape (n_sets + 1,), got {tuple(off.shape)}")
        prm = params if params is not None else pf_default_params()
        if result is None:
            result = torch.empty((_lib.CRB_PF_RESULT_LEN, nr), dtype=torch.float64, device=px.device)
        _shape(result, _lib.CRB_PF_RESULT_LEN, nr, "result")
        if status is not None:
            _shape(status, 1, nr, "status")
        check(self.lib.crb_pf_step_many_batched(
            self.ctx, nr, npr, _ptr(px, np.float32, device=True, name="px"),
            _ptr(pw, np.float32, device=True, name="pw"), _ptr(px_next, np.float32, device=True, name="px_next"),
            _ptr(u, np.float32, device=True, name="u"), _ptr(noise, np.float32, device=True, name="noise"),
            C.c_uint64(int(seed)), _ptr(z, np.float32, device=True, name="z"), int(z.shape[0]),
            _ptr(off, np.int64, device=True, name="z_off"), int(off.shape[0]) - 1,
            _ptr(z_of, np.int32, device=True, name="z_of"), C.byref(prm),
            _ptr(uniforms, np.float32, device=True, name="uniforms"), C.c_uint64(int(resample_seed)),
            C.c_float(npr // 2 if nth is None else nth), _ptr(result, np.float64, device=True, name="result"),
            _ptr(status, np.int32, device=True, name="status")),
            "crb_pf_step_many_batched")
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

    def calc_ref_trajectory_many(self, state, courses, course_of, dl: float, target_ind, xref, T: int,
                                 params: Optional[MpcParams] = None, status=None):
        """calc_ref_trajectory with a course per agent.  courses (cx, cy, cyaw, sp, course_off): the concatenated
        courses [npts] float32 and course_off [n_courses + 1] int64 (synth.pack_courses); course_of [n] int32, the
        course of each agent; target_ind [n] in/out, course-local; xref [4*T, n] out; status [n] int32
        (CRB_MPC_REF_*) is allocated when not given.  Returns status.  CUDA tensors; only enqueues."""
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(xref, 4 * T, n, "xref")
        cx, cy, cyaw, sp, off = courses
        npts = int(cx.shape[0])
        for a, name in ((cx, "cx"), (cy, "cy"), (cyaw, "cyaw"), (sp, "sp")):
            _shape(a, 1, npts, name)
        _shape(course_of, 1, n, "course_of"); _shape(target_ind, 1, n, "target_ind")
        status = status if status is not None else torch.empty(n, dtype=torch.int32, device=state.device)
        _shape(status, 1, n, "status")
        prm = params if params is not None else mpc_default_params()
        f = lambda a, name: _ptr(a, np.float32, device=True, name=name)  # noqa: E731
        check(self.lib.crb_mpc_calc_ref_trajectory_many_batched(
            self.ctx, n, int(T), f(state, "state"), f(cx, "cx"), f(cy, "cy"), f(cyaw, "cyaw"), f(sp, "sp"),
            _ptr(off, np.int64, device=True, name="course_off"), int(off.shape[0]) - 1, npts,
            _ptr(course_of, np.int32, device=True, name="course_of"), C.c_float(dl),
            _ptr(target_ind, np.int32, device=True, name="target_ind"), f(xref, "xref"),
            _ptr(status, np.int32, device=True, name="status"), C.byref(prm)),
            "crb_mpc_calc_ref_trajectory_many_batched")
        return status

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

    def dwa_control_many(self, x, u, goal, obstacles, ob_of, params: Optional[DwaParams] = None, cost=None, best=None,
                         traj=None, status=None):
        """dwa_control() for n robots, each among its own obstacles.  obstacles (ob, ob_off): the lists' rows ob
        [n_rows, 2] float32 back to back and ob_off [n_sets + 1] int64 (synth.pack_obstacles); ob_of [n] int32, the list
        of each robot.  Everything else as dwa_control; status [n] int32 (CRB_DWA_*) is allocated when not given.
        Returns status.  CUDA tensors; only enqueues."""
        n = int(x.shape[-1])
        _shape(x, 5, n, "x"); _shape(u, 2, n, "u"); _shape(goal, 2, n, "goal"); _shape(ob_of, 1, n, "ob_of")
        ob, off = obstacles
        if ob.dim() != 2 or int(ob.shape[1]) != 2:
            raise ValueError(f"ob: expected shape (n_rows, 2), got {tuple(ob.shape)}")
        if off.dim() != 1:
            raise ValueError(f"ob_off: expected shape (n_sets + 1,), got {tuple(off.shape)}")
        prm = params if params is not None else dwa_default_params()
        if cost is not None:
            _shape(cost, 1, n, "cost")
        if best is not None:
            _shape(best, 1, n, "best")
        if traj is not None:
            _shape(traj, 5 * self.dwa_rollout_points(prm), n, "traj")
        status = status if status is not None else torch.empty(n, dtype=torch.int32, device=x.device)
        _shape(status, 1, n, "status")
        check(self.lib.crb_dwa_control_many_batched(
            self.ctx, n, _ptr(x, np.float32, device=True, name="x"), _ptr(u, np.float32, device=True, name="u"),
            _ptr(goal, np.float32, device=True, name="goal"), _ptr(ob, np.float32, device=True, name="ob"),
            int(ob.shape[0]), _ptr(off, np.int64, device=True, name="ob_off"), int(off.shape[0]) - 1,
            _ptr(ob_of, np.int32, device=True, name="ob_of"), C.byref(prm),
            _ptr(cost, np.float32, device=True, name="cost"), _ptr(best, np.int32, device=True, name="best"),
            _ptr(traj, np.float32, device=True, name="traj"), _ptr(status, np.int32, device=True, name="status")),
            "crb_dwa_control_many_batched")
        return status

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

    def dwa_max_rollout_points(self, configs) -> int:
        """The largest dwa_rollout_points over the records of a config table (float32 [m, 12]; copied to the host when
        on the device), refused records left out; 0 when every record is refused."""
        rows = configs.cpu().numpy() if torch is not None and isinstance(configs, torch.Tensor) else configs
        best = 0
        for row in np.asarray(rows, np.float32).reshape(-1, len(DWA_CONFIG_FIELDS)):
            k = C.c_int(0)
            if self.lib.crb_dwa_rollout_points(C.byref(DwaParams(*(float(v) for v in row))), C.byref(k)) == 0:
                best = max(best, int(k.value))
        return best

    def dwa_control_fleet(self, x, u, goal, obstacles, ob_of, configs, config_of, max_pts: Optional[int] = None,
                          cost=None, best=None, traj=None, traj_len=None, status=None):
        """dwa_control() for a fleet whose robots each have their own Config and obstacle list: robot i plans with
        configs[config_of[i]] among its list ob_of[i].  configs float32 [n_configs, 12] (dwa_config_table), config_of
        int32 [n]; x, u, goal, obstacles and ob_of as dwa_control_many.  Optional outputs cost [n], best [n] int32,
        traj [5*max_pts, n] (the first min(traj_len[i], max_pts) points of robot i's rollout are written), traj_len
        [n] int32 (each robot's point count); status [n] int32 (CRB_DWA_*) is allocated when not given.  max_pts
        defaults to the largest point count in the table (read from it on the host).  Returns status.  CUDA tensors;
        only enqueues when max_pts is given or traj is None."""
        n = int(x.shape[-1])
        _shape(x, 5, n, "x"); _shape(u, 2, n, "u"); _shape(goal, 2, n, "goal"); _shape(ob_of, 1, n, "ob_of")
        _shape(config_of, 1, n, "config_of")
        ob, off = obstacles
        if ob.dim() != 2 or int(ob.shape[1]) != 2:
            raise ValueError(f"ob: expected shape (n_rows, 2), got {tuple(ob.shape)}")
        if off.dim() != 1:
            raise ValueError(f"ob_off: expected shape (n_sets + 1,), got {tuple(off.shape)}")
        if configs.dim() != 2 or int(configs.shape[1]) != len(DWA_CONFIG_FIELDS):
            raise ValueError(f"configs: expected shape (n_configs, 12) (dwa_config_table), got {tuple(configs.shape)}")
        if max_pts is None:
            max_pts = self.dwa_max_rollout_points(configs) if traj is not None else 0
        if traj is not None:
            _shape(traj, 5 * int(max_pts), n, "traj")
        for a, name in ((cost, "cost"), (best, "best"), (traj_len, "traj_len")):
            if a is not None:
                _shape(a, 1, n, name)
        status = status if status is not None else torch.empty(n, dtype=torch.int32, device=x.device)
        _shape(status, 1, n, "status")
        check(self.lib.crb_dwa_control_fleet_batched(
            self.ctx, n, _ptr(x, np.float32, device=True, name="x"), _ptr(u, np.float32, device=True, name="u"),
            _ptr(goal, np.float32, device=True, name="goal"), _ptr(ob, np.float32, device=True, name="ob"),
            int(ob.shape[0]), _ptr(off, np.int64, device=True, name="ob_off"), int(off.shape[0]) - 1,
            _ptr(ob_of, np.int32, device=True, name="ob_of"), _ptr(configs, np.float32, device=True, name="configs"),
            int(configs.shape[0]), _ptr(config_of, np.int32, device=True, name="config_of"), int(max_pts),
            _ptr(cost, np.float32, device=True, name="cost"), _ptr(best, np.int32, device=True, name="best"),
            _ptr(traj, np.float32, device=True, name="traj"), _ptr(traj_len, np.int32, device=True, name="traj_len"),
            _ptr(status, np.int32, device=True, name="status")), "crb_dwa_control_fleet_batched")
        return status

    def dwa_motion_fleet(self, x, u, dt):
        """motion() in place on x [5,n] with u [2,n] and each robot's own dt [n] float32 (for example
        configs[:, DWA_CONFIG_FIELDS.index("dt")][config_of]), applied as given.  CUDA tensors; only enqueues."""
        n = int(x.shape[-1])
        _shape(x, 5, n, "x"); _shape(u, 2, n, "u"); _shape(dt, 1, n, "dt")
        check(self.lib.crb_dwa_motion_fleet_batched(self.ctx, n, _ptr(x, np.float32, device=True, name="x"),
                                                    _ptr(u, np.float32, device=True, name="u"),
                                                    _ptr(dt, np.float32, device=True, name="dt")),
              "crb_dwa_motion_fleet_batched")

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

    # ---- state lattice planner ----------------------------------------------------------------------------
    @staticmethod
    def slp_default_params():
        """(MptgParams, CONST_V): the optimizer settings and start speed generate_path uses."""
        return slp_default_params()

    @staticmethod
    def slp_load_table(path) -> np.ndarray:
        """lookuptable.csv read the reference's way: float32 [rows, 6] on the host (see slp_load_table)."""
        return slp_load_table(path)

    def slp_states_per_query(self, sampler) -> int:
        """S, the output slots per query of a crb_slp_sampler (SlpSampler)."""
        s = self.lib.crb_slp_states_per_query(C.byref(sampler))
        if s < 0:
            check(s, "crb_slp_states_per_query")
        return int(s)

    def slp_sample_states(self, sampler, qp, target=None, n_states=None, status=None):
        """The terminal-state samplers for n_q queries: sampler a SlpSampler (kind, nxy, nh, ns, d shared by the batch),
        qp [F,n_q] per-query floats (UNIFORM F = 4: a_min, a_max, p_min, p_max; BIASED F = 5: goal_angle and the same
        four; LANE F = 5: l_center, l_heading, l_width, v_width, d).  Returns (target [3, n_q*S], state j of query q in
        column q*S + j, NaN past n_states[q]; n_states [n_q] int32; status [n_q] int32, CRB_SLP_*), allocating what is
        not given.  CUDA tensors; only enqueues."""
        n = int(qp.shape[-1])
        S = self.slp_states_per_query(sampler)
        _shape(qp, 4 if sampler.kind == _lib.CRB_SLP_UNIFORM else 5, n, "qp")
        if target is None:
            target = torch.empty((3, n * S), dtype=torch.float32, device=qp.device)
        if n_states is None:
            n_states = torch.empty(n, dtype=torch.int32, device=qp.device)
        if status is None:
            status = torch.empty(n, dtype=torch.int32, device=qp.device)
        _shape(target, 3, n * S, "target"); _shape(n_states, 1, n, "n_states"); _shape(status, 1, n, "status")
        check(self.lib.crb_slp_sample_states_batched(
            self.ctx, n, C.byref(sampler), _ptr(qp, np.float32, device=True, name="qp"),
            _ptr(target, np.float32, device=True, name="target"),
            _ptr(n_states, np.int32, device=True, name="n_states"), _ptr(status, np.int32, device=True, name="status")),
            "crb_slp_sample_states_batched")
        return target, n_states, status

    def slp_search_nearest(self, target, table, k0=None, param=None, row=None):
        """search_nearest_one_from_lookuptable() for n targets: target [3,n], table [rows,6] (lookuptable.csv's
        columns), k0 [n] or None (0).  Returns (param [4,n] = (|xy|, k0, km, kf) of the nearest row, NaN when none is
        nearer than FLT_MAX; row [n] int32, -1 then), allocating what is not given.  CUDA tensors; only enqueues."""
        n = int(target.shape[-1])
        _shape(target, 3, n, "target")
        if table.dim() != 2 or int(table.shape[1]) != 6:
            raise ValueError(f"table: expected shape (rows, 6), got {tuple(table.shape)}")
        if k0 is not None:
            _shape(k0, 1, n, "k0")
        if param is None:
            param = torch.empty((4, n), dtype=torch.float32, device=target.device)
        if row is None:
            row = torch.empty(n, dtype=torch.int32, device=target.device)
        _shape(param, 4, n, "param"); _shape(row, 1, n, "row")
        check(self.lib.crb_slp_search_nearest_batched(
            self.ctx, n, _ptr(target, np.float32, device=True, name="target"),
            _ptr(table, np.float32, device=True, name="table"), int(table.shape[0]),
            _ptr(k0, np.float32, device=True, name="k0"), _ptr(param, np.float32, device=True, name="param"),
            _ptr(row, np.int32, device=True, name="row")), "crb_slp_search_nearest_batched")
        return param, row

    def slp_generate_path(self, target, table, k0=None, params: Optional[MptgParams] = None, v: Optional[float] = None,
                          max_pts: int = 0):
        """generate_path() :137-155 for n terminal states: the lookup-table search, start states (0, 0, 0, v) and
        optimizer_traj, one launch each.  target [3,n], table [rows,6], k0 [n] or None; params and v default to
        slp_default_params().  Returns dict(param [4,n] as optimised, traj [3*max_pts,n] (NaN past traj_len, None when
        max_pts = 0), traj_len, cost, status (CRB_MPTG_*), iters, row).  CUDA tensors; only enqueues."""
        p0, v0 = slp_default_params()
        n = int(target.shape[-1])
        dev = target.device
        param, row = self.slp_search_nearest(target, table, k0)
        state = torch.zeros((4, n), dtype=torch.float32, device=dev)
        state[3] = v0 if v is None else v
        traj = torch.full((3 * max_pts, n), float("nan"), dtype=torch.float32, device=dev) if max_pts > 0 else None
        traj_len, status, iters = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(3))
        cost = torch.empty(n, dtype=torch.float32, device=dev)
        self.mptg_optimize(state, target, param, params if params is not None else p0, traj=traj, traj_len=traj_len,
                           cost=cost, status=status, iters=iters)
        return dict(param=param, traj=traj, traj_len=traj_len, cost=cost, status=status, iters=iters, row=row)

    # ---- grid A* / Dijkstra ------------------------------------------------------------------------------------
    @staticmethod
    def grid_box_of_obstacles(ox, oy, reso: float) -> GridBox:
        """The planners' box of cells from host obstacle arrays (see grid_box_of_obstacles)."""
        return grid_box_of_obstacles(ox, oy, reso)

    @staticmethod
    def _grid_dims(box: GridBox):
        return int(box.max_x) - int(box.min_x), int(box.max_y) - int(box.min_y)

    def grid_obstacle_map(self, ox, oy, reso: float, rr: float, box: GridBox, map=None):
        """calc_obstacle_map() :48-78 for the box: ox, oy [n_obs] CUDA float32.  Returns map [W, H] uint8 (1 =
        blocked; cell (x, y) at [x - min_x, y - min_y]), allocated when not given.  Only enqueues."""
        n = int(ox.shape[-1])
        _shape(ox, 1, n, "ox"); _shape(oy, 1, n, "oy")
        W, H = self._grid_dims(box)
        if map is None:
            map = torch.empty((max(W, 0), max(H, 0)), dtype=torch.uint8, device=ox.device)
        elif tuple(map.shape) != (W, H):
            raise ValueError(f"map: expected shape ({W}, {H}), got {tuple(map.shape)}")
        check(self.lib.crb_grid_obstacle_map(
            self.ctx, n, _ptr(ox, np.float32, device=True, name="ox"), _ptr(oy, np.float32, device=True, name="oy"),
            float(reso), float(rr), C.byref(box), _ptr(map, np.uint8, device=True, name="map")),
            "crb_grid_obstacle_map")
        return map

    def grid_plan_slots(self, algo: int, box: GridBox, n: int) -> int:
        """The number of searches grid_plan runs at once for n queries on this box."""
        s = C.c_int64(0)
        check(self.lib.crb_grid_plan_slots(self.ctx, int(algo), C.byref(box), int(n), C.byref(s)),
              "crb_grid_plan_slots")
        return int(s.value)

    def grid_plan(self, algo: int, box: GridBox, map, reso: float, sg, max_pts: int = 0, path=None, path_len=None,
                  cost=None, n_visited=None, status=None):
        """a_star_planning() (algo CRB_GRID_ASTAR) or dijkstra_star_planning() (CRB_GRID_DIJKSTRA) for n queries on
        one map: map [W, H] uint8 (grid_obstacle_map's), sg [4, n] float32 (sx, sy, gx, gy).  Returns dict(path
        [2*max_pts, n] (point k's x, y in rows 2k, 2k+1, the goal first; NaN past path_len; None when max_pts = 0),
        path_len, cost, n_visited, status (CRB_GRID_*)), allocating what is not given.  CUDA tensors; only enqueues
        (the first call at a larger workspace allocates it)."""
        n = int(sg.shape[-1])
        _shape(sg, 4, n, "sg")
        W, H = self._grid_dims(box)
        if tuple(map.shape) not in ((W, H), (W * H,)):
            raise ValueError(f"map: expected shape ({W}, {H}), got {tuple(map.shape)}")
        dev = sg.device
        if path is None and max_pts > 0:
            path = torch.full((2 * max_pts, n), float("nan"), dtype=torch.float32, device=dev)
        if path is not None:
            _shape(path, 2 * max_pts, n, "path")
        i32 = lambda a: a if a is not None else torch.empty(n, dtype=torch.int32, device=dev)  # noqa: E731
        path_len, n_visited, status = i32(path_len), i32(n_visited), i32(status)
        if cost is None:
            cost = torch.empty(n, dtype=torch.float32, device=dev)
        for a, name in ((path_len, "path_len"), (cost, "cost"), (n_visited, "n_visited"), (status, "status")):
            _shape(a, 1, n, name)
        check(self.lib.crb_grid_plan_batched(
            self.ctx, int(algo), C.byref(box), _ptr(map, np.uint8, device=True, name="map"), float(reso), n,
            _ptr(sg, np.float32, device=True, name="sg"), int(max_pts),
            _ptr(path, np.float32, device=True, name="path"), _ptr(path_len, np.int32, device=True, name="path_len"),
            _ptr(cost, np.float32, device=True, name="cost"), _ptr(n_visited, np.int32, device=True, name="n_visited"),
            _ptr(status, np.int32, device=True, name="status")), "crb_grid_plan_batched")
        return dict(path=path, path_len=path_len, cost=cost, n_visited=n_visited, status=status)

    def grid_obstacle_map_many(self, obstacles, ob_of, rr, table, maps=None, map_status=None):
        """calc_obstacle_map() for every map of a table in one launch.  obstacles (ob, ob_off): obstacle lists ob
        [n_rows, 2] float32 rows (ox, oy) back to back and ob_off [n_sets + 1] int64 (synth.pack_obstacles); ob_of
        [n_maps] int32, the list of each map; rr [n_maps] float32, each map's robot radius; table (boxes int32
        [n_maps, 4], reso float32 [n_maps], map_off int64 [n_maps + 1], max_cells) from grid_map_table, its arrays on
        the device.  Returns (maps [n_cells] uint8, map_status [n_maps] int32 CRB_GRID_MAP_*), allocating what is not
        given (maps zeroed, after one read of map_off[-1]).  CUDA tensors; only enqueues."""
        boxes, reso, off, max_cells = table
        n_maps = int(reso.shape[0])
        ob, ob_off = obstacles
        if ob.dim() != 2 or int(ob.shape[1]) != 2:
            raise ValueError(f"ob: expected shape (n_rows, 2), got {tuple(ob.shape)}")
        if ob_off.dim() != 1:
            raise ValueError(f"ob_off: expected shape (n_sets + 1,), got {tuple(ob_off.shape)}")
        self._grid_table_shapes(boxes, reso, off)
        _shape(ob_of, 1, n_maps, "ob_of"); _shape(rr, 1, n_maps, "rr")
        if maps is None:
            maps = torch.zeros(int(off[-1].item()), dtype=torch.uint8, device=reso.device)
        if map_status is None:
            map_status = torch.empty(n_maps, dtype=torch.int32, device=reso.device)
        _shape(map_status, 1, n_maps, "map_status")
        check(self.lib.crb_grid_obstacle_map_many(
            self.ctx, _ptr(ob, np.float32, device=True, name="ob"), int(ob.shape[0]),
            _ptr(ob_off, np.int64, device=True, name="ob_off"), int(ob_off.shape[0]) - 1,
            _ptr(ob_of, np.int32, device=True, name="ob_of"), _ptr(rr, np.float32, device=True, name="rr"),
            _ptr(boxes, np.int32, device=True, name="boxes"), _ptr(reso, np.float32, device=True, name="reso"),
            _ptr(off, np.int64, device=True, name="map_off"), n_maps, int(maps.numel()), int(max_cells),
            _ptr(maps, np.uint8, device=True, name="maps"), _ptr(map_status, np.int32, device=True, name="map_status")),
            "crb_grid_obstacle_map_many")
        return maps, map_status

    @staticmethod
    def _grid_table_shapes(boxes, reso, off):
        n_maps = int(reso.shape[0])
        if tuple(boxes.shape) != (n_maps, 4) or tuple(reso.shape) != (n_maps,) or tuple(off.shape) != (n_maps + 1,):
            raise ValueError(f"table: expected boxes [n_maps, 4], reso [n_maps], map_off [n_maps + 1], got "
                             f"{tuple(boxes.shape)}, {tuple(reso.shape)}, {tuple(off.shape)}")

    def grid_plan_many_slots(self, algo: int, max_cells: int, n: int) -> int:
        """The number of searches grid_plan_many runs at once for n queries on a table with this max_cells."""
        s = C.c_int64(0)
        check(self.lib.crb_grid_plan_many_slots(self.ctx, int(algo), int(max_cells), int(n), C.byref(s)),
              "crb_grid_plan_many_slots")
        return int(s.value)

    def grid_plan_many(self, algo: int, table, maps, map_of, sg, max_pts: int = 0, path=None, path_len=None,
                       cost=None, n_visited=None, status=None):
        """grid_plan with a map per query: query q plans on map map_of[q] (int32 [n]) of the table (grid_map_table's
        tuple, arrays on the device) and its byte store maps [n_cells] uint8 (grid_obstacle_map_many's).  sg [4, n]
        float32 in each query's own map's metres.  Returns grid_plan's dict; status may be CRB_GRID_BAD_MAP.  CUDA
        tensors; only enqueues (the first call at a larger workspace allocates it)."""
        boxes, reso, off, max_cells = table
        self._grid_table_shapes(boxes, reso, off)
        n = int(sg.shape[-1])
        _shape(sg, 4, n, "sg"); _shape(map_of, 1, n, "map_of")
        dev = sg.device
        if path is None and max_pts > 0:
            path = torch.full((2 * max_pts, n), float("nan"), dtype=torch.float32, device=dev)
        if path is not None:
            _shape(path, 2 * max_pts, n, "path")
        i32 = lambda a: a if a is not None else torch.empty(n, dtype=torch.int32, device=dev)  # noqa: E731
        path_len, n_visited, status = i32(path_len), i32(n_visited), i32(status)
        if cost is None:
            cost = torch.empty(n, dtype=torch.float32, device=dev)
        for a, name in ((path_len, "path_len"), (cost, "cost"), (n_visited, "n_visited"), (status, "status")):
            _shape(a, 1, n, name)
        check(self.lib.crb_grid_plan_many_batched(
            self.ctx, int(algo), _ptr(boxes, np.int32, device=True, name="boxes"),
            _ptr(reso, np.float32, device=True, name="reso"), _ptr(off, np.int64, device=True, name="map_off"),
            int(reso.shape[0]), _ptr(maps, np.uint8, device=True, name="maps"), int(maps.numel()), int(max_cells), n,
            _ptr(map_of, np.int32, device=True, name="map_of"), _ptr(sg, np.float32, device=True, name="sg"),
            int(max_pts), _ptr(path, np.float32, device=True, name="path"),
            _ptr(path_len, np.int32, device=True, name="path_len"), _ptr(cost, np.float32, device=True, name="cost"),
            _ptr(n_visited, np.int32, device=True, name="n_visited"), _ptr(status, np.int32, device=True, name="status")),
            "crb_grid_plan_many_batched")
        return dict(path=path, path_len=path_len, cost=cost, n_visited=n_visited, status=status)

    # ---- RRT ----------------------------------------------------------------------------------------------------
    @staticmethod
    def rrt_default_params() -> RrtParams:
        return rrt_default_params()

    def rrt_plan(self, ob, se, seed, params: Optional[RrtParams] = None, max_pts: int = 0, max_nodes: int = 0,
                 path=None, path_len=None, tree=None, parent=None, n_nodes=None, n_iter=None, status=None):
        """RRT::planning() for n seeded queries on one obstacle list: ob [n_ob, 3] float32 rows (x, y, r), se [4, n]
        float32 (sx, sy, gx, gy), seed [n] int32 or uint32 bits (goal_gen.seed(seed[i])).  Returns dict(path [2*max_pts,
        n] (point k's x, y in rows 2k, 2k+1, the goal first, the start last; NaN past path_len), path_len, tree
        [2*max_nodes, n] (node k's x, y in rows 2k, 2k+1; NaN past n_nodes), parent [max_nodes, n] (-1 for the start
        and past n_nodes), n_nodes, n_iter, status (CRB_RRT_*)), allocating what is not given (path / tree / parent
        None when their capacity is 0).  CUDA tensors; only enqueues (the first call on an Engine allocates the query
        counter)."""
        n = int(se.shape[-1])
        _shape(se, 4, n, "se")
        _shape(seed, 1, n, "seed")
        if ob.dim() != 2 or int(ob.shape[1]) != 3:
            raise ValueError(f"ob: expected shape (n_ob, 3), got {tuple(ob.shape)}")
        if seed.dtype not in (torch.int32, torch.uint32):
            raise TypeError(f"seed: expected int32 or uint32, got {seed.dtype}")
        if not seed.is_cuda or not seed.is_contiguous():
            raise ValueError("seed: expected a contiguous CUDA tensor")
        prm = params if params is not None else rrt_default_params()
        dev = se.device
        full = lambda rows, v, dt: torch.full((rows, n), v, dtype=dt, device=dev)  # noqa: E731
        if path is None and max_pts > 0:
            path = full(2 * max_pts, float("nan"), torch.float32)
        if tree is None and max_nodes > 0:
            tree = full(2 * max_nodes, float("nan"), torch.float32)
        if parent is None and max_nodes > 0:
            parent = full(max_nodes, -1, torch.int32)
        for a, rows, name in ((path, 2 * max_pts, "path"), (tree, 2 * max_nodes, "tree"), (parent, max_nodes, "parent")):
            if a is not None:
                _shape(a, rows, n, name)
        i32 = lambda a: a if a is not None else torch.empty(n, dtype=torch.int32, device=dev)  # noqa: E731
        path_len, n_nodes, n_iter, status = i32(path_len), i32(n_nodes), i32(n_iter), i32(status)
        for a, name in ((path_len, "path_len"), (n_nodes, "n_nodes"), (n_iter, "n_iter"), (status, "status")):
            _shape(a, 1, n, name)
        check(self.lib.crb_rrt_plan_batched(
            self.ctx, C.byref(prm), _ptr(ob, np.float32, device=True, name="ob"), int(ob.shape[0]), n,
            _ptr(se, np.float32, device=True, name="se"), seed.data_ptr(), int(max_pts),
            _ptr(path, np.float32, device=True, name="path"), _ptr(path_len, np.int32, device=True, name="path_len"),
            int(max_nodes), _ptr(tree, np.float32, device=True, name="tree"),
            _ptr(parent, np.int32, device=True, name="parent"), _ptr(n_nodes, np.int32, device=True, name="n_nodes"),
            _ptr(n_iter, np.int32, device=True, name="n_iter"), _ptr(status, np.int32, device=True, name="status")),
            "crb_rrt_plan_batched")
        return dict(path=path, path_len=path_len, tree=tree, parent=parent, n_nodes=n_nodes, n_iter=n_iter,
                    status=status)

    def rrt_plan_many(self, obstacles, ob_of, se, seed, params: Optional[RrtParams] = None, max_pts: int = 0,
                      max_nodes: int = 0, path=None, path_len=None, tree=None, parent=None, n_nodes=None, n_iter=None,
                      status=None):
        """RRT::planning() for n seeded queries, each among its own obstacles.  obstacles (ob, ob_off): the lists' rows
        ob [n_rows, 3] float32 (x, y, r) back to back and ob_off [n_sets + 1] int64 (synth.pack_obstacles); ob_of [n]
        int32, the list of each query.  Everything else, and the returned dict, as rrt_plan; status may be
        CRB_RRT_BAD_OBSTACLES."""
        n = int(se.shape[-1])
        _shape(se, 4, n, "se")
        _shape(seed, 1, n, "seed")
        _shape(ob_of, 1, n, "ob_of")
        ob, off = obstacles
        if ob.dim() != 2 or int(ob.shape[1]) != 3:
            raise ValueError(f"ob: expected shape (n_rows, 3), got {tuple(ob.shape)}")
        if off.dim() != 1:
            raise ValueError(f"ob_off: expected shape (n_sets + 1,), got {tuple(off.shape)}")
        if seed.dtype not in (torch.int32, torch.uint32):
            raise TypeError(f"seed: expected int32 or uint32, got {seed.dtype}")
        if not seed.is_cuda or not seed.is_contiguous():
            raise ValueError("seed: expected a contiguous CUDA tensor")
        prm = params if params is not None else rrt_default_params()
        dev = se.device
        full = lambda rows, v, dt: torch.full((rows, n), v, dtype=dt, device=dev)  # noqa: E731
        if path is None and max_pts > 0:
            path = full(2 * max_pts, float("nan"), torch.float32)
        if tree is None and max_nodes > 0:
            tree = full(2 * max_nodes, float("nan"), torch.float32)
        if parent is None and max_nodes > 0:
            parent = full(max_nodes, -1, torch.int32)
        for a, rows, name in ((path, 2 * max_pts, "path"), (tree, 2 * max_nodes, "tree"), (parent, max_nodes, "parent")):
            if a is not None:
                _shape(a, rows, n, name)
        i32 = lambda a: a if a is not None else torch.empty(n, dtype=torch.int32, device=dev)  # noqa: E731
        path_len, n_nodes, n_iter, status = i32(path_len), i32(n_nodes), i32(n_iter), i32(status)
        for a, name in ((path_len, "path_len"), (n_nodes, "n_nodes"), (n_iter, "n_iter"), (status, "status")):
            _shape(a, 1, n, name)
        check(self.lib.crb_rrt_plan_many_batched(
            self.ctx, C.byref(prm), _ptr(ob, np.float32, device=True, name="ob"), int(ob.shape[0]),
            _ptr(off, np.int64, device=True, name="ob_off"), int(off.shape[0]) - 1,
            _ptr(ob_of, np.int32, device=True, name="ob_of"), n, _ptr(se, np.float32, device=True, name="se"),
            seed.data_ptr(), int(max_pts), _ptr(path, np.float32, device=True, name="path"),
            _ptr(path_len, np.int32, device=True, name="path_len"), int(max_nodes),
            _ptr(tree, np.float32, device=True, name="tree"), _ptr(parent, np.int32, device=True, name="parent"),
            _ptr(n_nodes, np.int32, device=True, name="n_nodes"), _ptr(n_iter, np.int32, device=True, name="n_iter"),
            _ptr(status, np.int32, device=True, name="status")),
            "crb_rrt_plan_many_batched")
        return dict(path=path, path_len=path_len, tree=tree, parent=parent, n_nodes=n_nodes, n_iter=n_iter,
                    status=status)

    # ---- LQR path tracking ------------------------------------------------------------------------------------------
    def lqr_steering_control(self, nx: int, state, course, ind, pe, pth_e, params: Optional[LqrTrackParams] = None,
                             u=None, K=None, iters=None, status=None):
        """lqr_steering_control() for n vehicles on one course.  nx 4 (lqr_steer_control) or 5
        (lqr_speed_steer_control); state [4, n] (x, y, yaw, v); course (cx, cy, cyaw, ck) for nx 4 or (cx, cy, cyaw,
        ck, sp) for nx 5, 1-D float32 each; ind [n] int32 (in/out for nx 4, out for nx 5), pe, pth_e [n] in/out.
        Returns dict(u [nu, n] (delta | ai, delta), K [nu*nx, n] or None, iters, status (CRB_LQR_TRACK_*)); u, iters
        and status are allocated when not given, K only when passed.  CUDA tensors; only enqueues."""
        n = int(state.shape[-1])
        nu = 1 if nx == 4 else 2
        _shape(state, 4, n, "state")
        if len(course) != (4 if nx == 4 else 5):
            raise ValueError(f"course: expected {4 if nx == 4 else 5} arrays for nx = {nx}, got {len(course)}")
        nc = int(course[0].shape[0])
        for a, name in zip(course, ("cx", "cy", "cyaw", "ck", "sp")):
            _shape(a, 1, nc, name)
        for a, name in ((ind, "ind"), (pe, "pe"), (pth_e, "pth_e")):
            _shape(a, 1, n, name)
        dev = state.device
        if u is None:
            u = torch.empty((nu, n), dtype=torch.float32, device=dev)
        iters = iters if iters is not None else torch.empty(n, dtype=torch.int32, device=dev)
        status = status if status is not None else torch.empty(n, dtype=torch.int32, device=dev)
        _shape(u, nu, n, "u")
        if K is not None:
            _shape(K, nu * nx, n, "K")
        prm = params if params is not None else lqr_track_default_params(nx)
        f = lambda a, name: _ptr(a, np.float32, device=True, name=name)  # noqa: E731
        check(self.lib.crb_lqr_steering_control_batched(
            self.ctx, n, int(nx), f(state, "state"), f(course[0], "cx"), f(course[1], "cy"), f(course[2], "cyaw"),
            f(course[3], "ck"), f(course[4], "sp") if nx == 5 else None, nc, C.byref(prm),
            _ptr(ind, np.int32, device=True, name="ind"), f(pe, "pe"), f(pth_e, "pth_e"), f(u, "u"), f(K, "K"),
            _ptr(iters, np.int32, device=True, name="iters"), _ptr(status, np.int32, device=True, name="status")),
            "crb_lqr_steering_control_batched")
        return dict(u=u, K=K, iters=iters, status=status)

    def lqr_steering_control_many(self, nx: int, state, courses, course_of, ind, pe, pth_e,
                                  params: Optional[LqrTrackParams] = None, u=None, K=None, iters=None, status=None):
        """lqr_steering_control() for n vehicles, each on its own course.  courses (cx, cy, cyaw, ck, course_off) for
        nx 4 or (cx, cy, cyaw, ck, sp, course_off) for nx 5: the concatenated courses [npts] float32 and course_off
        [n_courses + 1] int64 (synth.pack_courses); course_of [n] int32, the course of each vehicle.  ind is
        course-local.  Everything else as lqr_steering_control; status may be CRB_LQR_TRACK_BAD_COURSE."""
        n = int(state.shape[-1])
        nu = 1 if nx == 4 else 2
        _shape(state, 4, n, "state")
        if len(courses) != (5 if nx == 4 else 6):
            raise ValueError(f"courses: expected {5 if nx == 4 else 6} arrays for nx = {nx}, got {len(courses)}")
        pts, off = courses[:-1], courses[-1]
        npts = int(pts[0].shape[0])
        for a, name in zip(pts, ("cx", "cy", "cyaw", "ck", "sp")):
            _shape(a, 1, npts, name)
        for a, name in ((course_of, "course_of"), (ind, "ind"), (pe, "pe"), (pth_e, "pth_e")):
            _shape(a, 1, n, name)
        dev = state.device
        if u is None:
            u = torch.empty((nu, n), dtype=torch.float32, device=dev)
        iters = iters if iters is not None else torch.empty(n, dtype=torch.int32, device=dev)
        status = status if status is not None else torch.empty(n, dtype=torch.int32, device=dev)
        _shape(u, nu, n, "u")
        if K is not None:
            _shape(K, nu * nx, n, "K")
        prm = params if params is not None else lqr_track_default_params(nx)
        f = lambda a, name: _ptr(a, np.float32, device=True, name=name)  # noqa: E731
        check(self.lib.crb_lqr_steering_control_many_batched(
            self.ctx, n, int(nx), f(state, "state"), f(pts[0], "cx"), f(pts[1], "cy"), f(pts[2], "cyaw"),
            f(pts[3], "ck"), f(pts[4], "sp") if nx == 5 else None, _ptr(off, np.int64, device=True, name="course_off"),
            int(off.shape[0]) - 1, npts, _ptr(course_of, np.int32, device=True, name="course_of"), C.byref(prm),
            _ptr(ind, np.int32, device=True, name="ind"), f(pe, "pe"), f(pth_e, "pth_e"), f(u, "u"), f(K, "K"),
            _ptr(iters, np.int32, device=True, name="iters"), _ptr(status, np.int32, device=True, name="status")),
            "crb_lqr_steering_control_many_batched")
        return dict(u=u, K=K, iters=iters, status=status)

    def lqr_update(self, state, a, delta, params: Optional[LqrTrackParams] = None):
        """update() of the LQR programs for n vehicles, in place: state [4, n], a [n], delta [n].  CUDA tensors."""
        n = int(state.shape[-1])
        _shape(state, 4, n, "state"); _shape(a, 1, n, "a"); _shape(delta, 1, n, "delta")
        prm = params if params is not None else lqr_track_default_params(4)
        check(self.lib.crb_lqr_update_batched(
            self.ctx, n, _ptr(state, np.float32, device=True, name="state"), _ptr(a, np.float32, device=True, name="a"),
            _ptr(delta, np.float32, device=True, name="delta"), C.byref(prm)), "crb_lqr_update_batched")
        return state

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

    def probe_ekf_pattern(self, x, P, z, u) -> None:
        """One launch of the EKF step's access pattern with trivial arithmetic (crb_probe.cu), in place on
        x [4,n] and P [16,n]; z, u [2,n].  CUDA tensors."""
        n = int(x.shape[-1])
        _shape(x, 4, n, "x"); _shape(P, 16, n, "P"); _shape(z, 2, n, "z"); _shape(u, 2, n, "u")
        check(self.lib.crb_probe_ekf_pattern(
            self.ctx, n, _ptr(x, np.float32, device=True, name="x"), _ptr(P, np.float32, device=True, name="P"),
            _ptr(z, np.float32, device=True, name="z"), _ptr(u, np.float32, device=True, name="u")),
            "crb_probe_ekf_pattern")

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
