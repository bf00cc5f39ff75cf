"""Where oracle/Makefile puts the checkers and the reference libraries, and how the oracle modules load them.

TEST INFRASTRUCTURE ONLY, like oracle.py: the product package (cpprobotics_b200/) never imports it.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(_HERE, "lib")    # lib/liboracle*.so, the checkers
REF_DIR = os.path.join(_HERE, "_ref")   # _ref/libref_*.so, built only where the reference tree is present

_loaded: dict[str, C.CDLL] = {}


def checker(path: str, prototypes: dict) -> C.CDLL:
    """The checker at path, loaded once, with prototypes {symbol: (restype, argtypes)} applied when it is."""
    L = _loaded.get(path)
    if L is None:
        if not os.path.exists(path):
            raise RuntimeError(f"{path} missing: run `make -C oracle` (or python __graft_entry__.py)")
        L = C.CDLL(path)
        for name, (res, args) in prototypes.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _loaded[path] = L
    return L


def reference(name: str) -> C.CDLL | None:
    """_ref/libref_<name>.so, or None when it was not built."""
    path = os.path.join(REF_DIR, f"libref_{name}.so")
    return C.CDLL(path) if os.path.exists(path) else None
