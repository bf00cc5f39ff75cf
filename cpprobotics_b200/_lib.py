"""ctypes binding of libcrb.so (the C ABI declared in include/crb.h).

This is the binding a maintainer of the reference would add on their side (see INTEGRATION.md for
the C++ one); Python is only used here because the tests / bench harness are Python.  There is NO
fallback: if the shared library is missing or a CUDA device is not usable, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcrb.so")

CRB_OK = 0
CRB_ERR_NO_DEVICE = -2
CRB_STATS_LEN = 8
CRB_COMM_ID_BYTES = 128
CRB_PF_RESULT_LEN = 24
CRB_PF_MAX_LANDMARKS = 64
CRB_MPC_MAX_T = 32
CRB_DWA_MAX_OBSTACLES = 256
CRB_DWA_MAX_SPEED_SAMPLES = 64
CRB_DWA_MAX_YAWRATE_SAMPLES = 512
CRB_DWA_MAX_STEPS = 1000
CRB_MPTG_MAX_ITER = 1000
CRB_MPTG_MAX_STEPS = 16384
CRB_MPTG_CONVERGED = 0
CRB_MPTG_MAX_ITER_REACHED = 1
CRB_MPTG_EMPTY_TRAJ = 2
CRB_MPTG_STEP_CAP = 3
CRB_MPTG_OUT_OF_RANGE = 4

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)
c_f64p = C.POINTER(C.c_double)


class EkfParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("Q", C.c_float * 16), ("R", C.c_float * 4)]


class PfParams(C.Structure):
    _fields_ = [("dt", C.c_double), ("pi", C.c_double), ("Q", C.c_float),
                ("rsim_diag", C.c_float * 2), ("u", C.c_float * 2)]


class MpcParams(C.Structure):
    _fields_ = [("dt", C.c_float), ("wb", C.c_float), ("max_steer", C.c_float),
                ("max_accel", C.c_float), ("max_speed", C.c_float), ("min_speed", C.c_float),
                ("w_a", C.c_float), ("w_delta", C.c_float), ("w_da", C.c_float),
                ("w_ddelta", C.c_float), ("w_x", C.c_float), ("w_y", C.c_float),
                ("w_yaw", C.c_float), ("w_v", C.c_float), ("max_iter", C.c_int),
                ("du_th", C.c_float), ("max_ls", C.c_int), ("j_tol", C.c_float)]


class DwaParams(C.Structure):
    _fields_ = [(name, C.c_float) for name in (
        "max_speed", "min_speed", "max_yawrate", "max_accel", "robot_radius", "max_dyawrate",
        "v_reso", "yawrate_reso", "dt", "predict_time", "to_goal_cost_gain", "speed_cost_gain")]


class MptgParams(C.Structure):
    _fields_ = [("base_l", C.c_float), ("ds", C.c_float), ("max_iter", C.c_int32), ("cost_th", C.c_float),
                ("h_step", C.c_float * 3)]


# name -> (restype, argtypes); every symbol include/crb.h declares
PROTOTYPES = {
    "crb_abi_version": (C.c_int, []),
    "crb_last_error_string": (C.c_char_p, []),
    "crb_init": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "crb_destroy": (C.c_int, [C.c_void_p]),
    "crb_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "crb_use_own_stream": (C.c_int, [C.c_void_p]),
    "crb_get_stream": (C.c_void_p, [C.c_void_p]),
    "crb_sync": (C.c_int, [C.c_void_p]),
    "crb_launch_count": (C.c_int64, [C.c_void_p]),
    "crb_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "crb_host_free": (C.c_int, [C.c_void_p]),
    "crb_device_alloc": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_size_t]),
    "crb_device_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "crb_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "crb_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "crb_timer_start": (C.c_int, [C.c_void_p]),
    "crb_timer_stop_ms": (C.c_int, [C.c_void_p, c_f32p]),
    "crb_ekf_default_params": (None, [C.POINTER(EkfParams)]),
    "crb_ekf_step_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(EkfParams), C.c_int]),
    "crb_ekf_step_batched_host": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.POINTER(EkfParams), C.c_int]),
    "crb_ekf_track_open": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "crb_ekf_track_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(EkfParams),
                                     C.c_void_p, C.c_int]),
    "crb_ekf_track_sync": (C.c_int, [C.c_void_p, C.c_void_p]),
    "crb_ekf_track_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_ekf_track_close": (C.c_int, [C.c_void_p, C.c_void_p]),
    "crb_pf_default_params": (None, [C.POINTER(PfParams)]),
    "crb_pf_predict_weight_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_uint64, C.c_void_p, C.c_int,
                                                C.POINTER(PfParams)]),
    "crb_pf_predict_weight_batched_host": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                     C.c_void_p, C.c_uint64, C.c_void_p, C.c_int,
                                                     C.POINTER(PfParams)]),
    "crb_pf_estimate": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "crb_pf_resample": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_uint64, C.c_float, C.c_void_p, C.c_void_p]),
    "crb_pf_step": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                              C.c_void_p, C.c_int, C.POINTER(PfParams), C.c_void_p, C.c_uint64, C.c_float,
                              C.c_void_p]),
    "crb_mpc_default_params": (None, [C.POINTER(MpcParams)]),
    "crb_mpc_solve_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.POINTER(MpcParams), C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_mpc_solve_batched_hinted": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.POINTER(MpcParams), C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_mpc_solve_batched_host": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.POINTER(MpcParams), C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_mpc_plant_update_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                               C.POINTER(MpcParams)]),
    "crb_mpc_calc_ref_trajectory_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_void_p, C.c_int32, C.c_float, C.c_void_p,
                                                      C.c_void_p, C.POINTER(MpcParams)]),
    "crb_lqr_dlqr_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "crb_dwa_default_params": (None, [C.POINTER(DwaParams)]),
    "crb_dwa_rollout_points": (C.c_int, [C.POINTER(DwaParams), C.POINTER(C.c_int)]),
    "crb_dwa_control_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int, C.POINTER(DwaParams), C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_dwa_motion_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float]),
    "crb_mptg_default_params": (None, [C.POINTER(MptgParams)]),
    "crb_mptg_optimize_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.POINTER(MptgParams), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "crb_mptg_generate_trajectory_batched": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                       C.POINTER(MptgParams), C.c_int, C.c_void_p, C.c_void_p,
                                                       C.c_void_p, C.c_void_p]),
    "crb_stats_reduce": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]),
    "crb_probe_fp32_peak": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "crb_comm_nccl_version": (C.c_int, []),
    "crb_comm_get_unique_id": (C.c_int, [C.c_void_p]),
    "crb_comm_init_rank": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "crb_comm_destroy": (C.c_int, [C.c_void_p]),
    "crb_comm_world": (C.c_int, [C.c_void_p]),
    "crb_comm_rank": (C.c_int, [C.c_void_p]),
    "crb_gather_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "crb_comm_allreduce_sum_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
}

_lib = None


class CrbError(RuntimeError):
    pass


def load_library() -> C.CDLL:
    """Load libcrb.so and attach prototypes.  Raises if the library is missing (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CrbError(
            f"{LIB_PATH} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "cpprobotics_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the ABI lost a symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != CRB_OK:
        msg = load_library().crb_last_error_string()
        raise CrbError(f"{what} failed with status {rc}: {msg.decode() if msg else ''}")
