"""cpprobotics_b200 — H100-native batched small-matrix engine for the CppRobotics hot paths.

The product is libcrb.so (hand-written sm_90a CUDA behind the C ABI of include/crb.h); this package
is the thin Python host layer the tests and the bench use to reach it.  There is no CPU path here:
importing works anywhere (so the build can be checked without a GPU), computing needs an H100.
"""
from ._lib import (CrbError, DwaParams, EkfParams, GridBox, LqrTrackParams, MpcParams, MptgParams,  # noqa: F401
                   PfParams, RrtParams, SlpSampler, load_library)
from .engine import (DWA_CONFIG_FIELDS, EKF_MODEL_DTYPE, Engine, dwa_config_table,  # noqa: F401
                     dwa_default_params, ekf_default_params, ekf_models,
                     grid_box_of_obstacles, grid_map_table, lqr_track_default_params, mpc_default_params,
                     mptg_default_params, pf_default_params, rrt_default_params, slp_default_params, slp_load_table)

__all__ = ["Engine", "CrbError", "EkfParams", "PfParams", "MpcParams", "DwaParams", "MptgParams", "SlpSampler",
           "GridBox", "RrtParams", "LqrTrackParams", "load_library", "grid_box_of_obstacles", "grid_map_table",
           "ekf_default_params", "ekf_models", "EKF_MODEL_DTYPE", "pf_default_params", "mpc_default_params",
           "dwa_default_params", "dwa_config_table", "DWA_CONFIG_FIELDS", "mptg_default_params", "slp_default_params",
           "slp_load_table", "rrt_default_params", "lqr_track_default_params"]
