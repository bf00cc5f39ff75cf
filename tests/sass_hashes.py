"""sha256 of each kernel's SASS in one libcrb source, the machine-code pins' common method.

The source is compiled with NVCC_FLAGS and disassembled with cuobjdump -sass; a kernel's hash covers its instructions
and the device functions it calls, without the fatbin and section header lines.  The pinned values are CUDA 12.9's, so
a test skips with any other nvcc."""
import hashlib
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false", "-Xptxas", "-v"]


def compile_source(tmp_path, src):
    """(object path, ptxas report) of cpprobotics_b200/csrc/<src>; skips without nvcc."""
    if not os.path.exists(NVCC):
        pytest.skip("no nvcc")
    obj = str(tmp_path / (src + ".o"))
    log = subprocess.run([NVCC] + NVCC_FLAGS + ["-c", os.path.join(ROOT, "cpprobotics_b200", "csrc", src), "-o", obj],
                         capture_output=True, text=True, check=True).stderr
    return obj, log


def kernel_sass_hashes(tmp_path, src):
    """{mangled kernel name: sha256 of its SASS} for every kernel of <src>; skips unless nvcc is CUDA 12.9's."""
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout if os.path.exists(NVCC) else ""
    if "release 12.9" not in ver:
        pytest.skip("the pinned SASS is CUDA 12.9's")
    obj, _ = compile_source(tmp_path, src)
    sass = subprocess.check_output([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "-sass", obj], text=True)
    got = {}
    for sec in sass.split("Function : ")[1:]:
        lines = sec.splitlines()
        body = "\n".join(x for x in lines[1:] if x.strip() and "Fatbin" not in x and "code for" not in x)
        got[lines[0].strip()] = hashlib.sha256(body.encode()).hexdigest()
    return got
