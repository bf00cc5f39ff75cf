"""CPU: the C-ABI shared library loads, exports every symbol include/crb.h declares, its structs have
the layout the bindings assume, and every compute entry point fails LOUDLY without a GPU."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from cpprobotics_b200 import _lib
from toolchain import run_layout_probe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "crb.h")


def declared_symbols():
    src = open(HDR).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(crb_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_what_the_binding_binds():
    assert set(declared_symbols()) == set(_lib.PROTOTYPES)


def test_library_exports_every_declared_symbol():
    lib = _lib.load_library()
    for name in declared_symbols():
        assert hasattr(lib, name), name
    assert lib.crb_abi_version() == 2


def test_struct_layouts_match_the_header(tmp_path):
    got = run_layout_probe(
        tmp_path, '#include <stdio.h>\n#include <stddef.h>\n#include "crb.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n",'
        "sizeof(crb_ekf_params),sizeof(crb_pf_params),sizeof(crb_mpc_params),"
        "offsetof(crb_ekf_params,R),offsetof(crb_pf_params,u),offsetof(crb_mpc_params,j_tol));return 0;}\n")
    want = [C.sizeof(_lib.EkfParams), C.sizeof(_lib.PfParams), C.sizeof(_lib.MpcParams),
            _lib.EkfParams.R.offset, _lib.PfParams.u.offset, _lib.MpcParams.j_tol.offset]
    assert got == want


def test_default_params_are_the_reference_constants():
    from cpprobotics_b200 import ekf_default_params, mpc_default_params, pf_default_params
    from oracle import oracle as O
    e = ekf_default_params()
    dt, Q, R = O.ekf_constants()
    assert e.dt == dt and np.array_equal(np.array(e.Q[:], np.float32), Q) and np.array_equal(np.array(e.R[:], np.float32), R)
    p = pf_default_params()
    c = O.pf_constants()
    assert p.dt == c["dt"] and p.pi == c["pi"] and np.float32(p.Q) == c["Q"]
    assert np.array_equal(np.array(p.rsim_diag[:], np.float32), c["rsim_diag"])
    m, mo = mpc_default_params(), O.mpc_params()
    for name, _ in _lib.MpcParams._fields_:
        assert getattr(m, name) == getattr(mo, name), name


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "c.c"
    src.write_text('#include "crb.h"\nint main(void){crb_ekf_params p; void (*f)(crb_ekf_params*) = crb_ekf_default_params; (void)p; (void)f; return 0;}\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-c", "-I",
                           os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "c.o")])


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


@pytest.mark.skipif(not _no_gpu(), reason="checks the failure path of a box without a GPU")
def test_no_gpu_means_loud_failure_not_fallback():
    lib = _lib.load_library()
    h = C.c_void_p()
    rc = lib.crb_init(C.byref(h), -1)
    assert rc == _lib.CRB_ERR_NO_DEVICE and not h.value
    assert b"no CPU fallback" in lib.crb_last_error_string()
    from cpprobotics_b200 import CrbError, Engine
    with pytest.raises(CrbError):
        Engine(0)


def test_argument_validation_needs_no_device():
    lib = _lib.load_library()
    assert lib.crb_init(None, 0) == -1                       # CRB_ERR_INVALID_ARG
    assert lib.crb_ekf_step_batched(None, 1, None, None, None, None, None, 1) == -1
    assert lib.crb_mpc_solve_batched(None, 1, 20, None, None, None, None, None, None, None, None, None) == -1
    assert lib.crb_sync(None) == -1 and lib.crb_launch_count(None) == -1


def test_product_never_imports_the_oracle():
    """Only tests/, __graft_entry__.smoke() (cpprobotics_b200/smoke.py) and bench.py may touch oracle/."""
    pkg = os.path.join(ROOT, "cpprobotics_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith(".py") and f != "smoke.py":
                txt = open(path).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "liboracle" not in txt, f
            if f.endswith((".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = re.sub(r"//[^\n]*|/\*.*?\*/", "", open(path).read(), flags=re.S)   # code, not comments
                assert "crb_oracle_" not in txt and not re.search(r'#include\s*[<"].*oracle', txt), f
    for hdr in os.listdir(os.path.join(ROOT, "include")):
        if hdr.endswith((".h", ".hpp")):
            assert "crb_oracle_" not in open(os.path.join(ROOT, "include", hdr)).read()
    out = subprocess.check_output(["nm", "-D", _lib.LIB_PATH], text=True)
    assert "crb_oracle" not in out
