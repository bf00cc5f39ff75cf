"""cpprobotics_b200 — H100-native batched small-matrix engine for the CppRobotics hot paths.

The product is libcrb.so (hand-written sm_90a CUDA behind the C ABI of include/crb.h); this package
is the thin Python host layer the tests and the bench use to reach it.  There is no CPU path here:
importing works anywhere (so the build can be checked without a GPU), computing needs an H100.
"""
from ._lib import CrbError, DwaParams, EkfParams, MpcParams, MptgParams, PfParams, load_library  # noqa: F401
from .engine import (Engine, dwa_default_params, ekf_default_params,  # noqa: F401
                     mpc_default_params, mptg_default_params, pf_default_params)

__all__ = ["Engine", "CrbError", "EkfParams", "PfParams", "MpcParams", "DwaParams", "MptgParams", "load_library",
           "ekf_default_params", "pf_default_params", "mpc_default_params", "dwa_default_params",
           "mptg_default_params"]
