"""How the tests compile: libcrb's CUDA sources as the build compiles them, and the small host programs they run.

compile_source builds cpprobotics_b200/csrc/<src> with the build's own command line (__graft_entry__.NVCC and
NVCC_FLAGS), at most once per process, into a directory removed at exit; ptxas_functions and kernel_sass_hashes read
that one compile.  build_ref_program and run_layout_probe hold the host recipes of the C++ programs under tests/cpp
and of the C programs that print include/crb.h's layout."""
import functools
import hashlib
import os
import re
import subprocess
import tempfile
from typing import NamedTuple, Optional

import pytest

import __graft_entry__ as G
from cpprobotics_b200 import _lib

INCLUDE = os.path.join(G.ROOT, "include")
CPP_DIR = os.path.join(G.ROOT, "tests", "cpp")
LIBDIR = os.path.dirname(_lib.LIB_PATH)
_OBJ_DIR = tempfile.TemporaryDirectory(prefix="crb-nvcc-")   # removed when the interpreter exits


@functools.lru_cache(maxsize=None)
def _nvcc(src):
    obj = os.path.join(_OBJ_DIR.name, src + ".o")
    log = subprocess.run([G.NVCC] + G.NVCC_FLAGS + ["-c", os.path.join(G.CSRC, src), "-o", obj],
                         capture_output=True, text=True, check=True).stderr
    return obj, log


def compile_source(src):
    """(object path, ptxas -v report) of csrc/<src>, compiled once per process; skips without nvcc."""
    if not os.path.exists(G.NVCC):
        pytest.skip("no nvcc")
    return _nvcc(src)


class PtxasFunction(NamedTuple):
    name: str                  # mangled
    entry: bool                # a kernel, not an out-of-line device function
    registers: Optional[int]   # kernels only: ptxas reports registers per entry function
    stack: int                 # stack frame bytes
    spill_stores: int
    spill_loads: int


_ENTRY = re.compile(r"Compiling entry function '([^']+)'")
_PROPS = re.compile(r"Function properties for (\S+)$")
_FRAME = re.compile(r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads$")
_REGS = re.compile(r"Used (\d+) registers")


def parse_ptxas(report):
    """One record per 'Function properties for <name>' in a ptxas -v report, in report order, each read from its own
    properties line.  An out-of-line function appears once under every kernel that calls it."""
    lines = report.splitlines()
    entry, out = None, []
    for i, ln in enumerate(lines):
        m = _ENTRY.search(ln)
        if m:
            entry = m.group(1)
            continue
        m = _PROPS.search(ln)
        if not m:
            continue
        name = m.group(1)
        frame = _FRAME.match(lines[i + 1])
        assert frame, lines[i:i + 2]
        regs = None
        if name == entry:   # a kernel's register line follows its properties
            used = _REGS.search(lines[i + 2])
            assert used, lines[i:i + 3]
            regs = int(used.group(1))
        out.append(PtxasFunction(name, name == entry, regs, *map(int, frame.groups())))
        entry = None
    return out


def ptxas_functions(src):
    """parse_ptxas of csrc/<src>'s compile."""
    return parse_ptxas(compile_source(src)[1])


def ptxas_kernels(src):
    """{mangled kernel name: its PtxasFunction} for every kernel of csrc/<src>."""
    return {f.name: f for f in ptxas_functions(src) if f.entry}


def kernel_sass_hashes(src):
    """{mangled kernel name: sha256 of its SASS} for every kernel of csrc/<src>.  A kernel's hash covers its
    instructions and the device functions it calls, without the fatbin and section header lines of cuobjdump -sass.
    The pinned values are CUDA 12.9's, so this skips with any other nvcc."""
    ver = subprocess.run([G.NVCC, "--version"], capture_output=True, text=True).stdout if os.path.exists(G.NVCC) else ""
    if "release 12.9" not in ver:
        pytest.skip("the pinned SASS is CUDA 12.9's")
    obj, _ = compile_source(src)
    sass = subprocess.check_output([os.path.join(os.path.dirname(G.NVCC), "cuobjdump"), "-sass", obj], text=True)
    got = {}
    for sec in sass.split("Function : ")[1:]:
        lines = sec.splitlines()
        body = "\n".join(x for x in lines[1:] if x.strip() and "Fatbin" not in x and "code for" not in x)
        got[lines[0].strip()] = hashlib.sha256(body.encode()).hexdigest()
    return got


def build_ref_program(tmp_path, cpp, extra_flags=(), werror=True):
    """Build tests/cpp/<cpp> as a CppRobotics user would against include/ and libcrb.so; returns the executable."""
    exe = str(tmp_path / os.path.splitext(cpp)[0])
    subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall"] + (["-Werror"] if werror else []) + list(extra_flags)
                          + ["-I", INCLUDE, os.path.join(CPP_DIR, cpp), "-L", LIBDIR, "-lcrb",
                             f"-Wl,-rpath,{LIBDIR}", "-o", exe])
    return exe


STRICT_C99 = ("-std=c99", "-Wall", "-Werror")


def run_layout_probe(tmp_path, c_source, cflags=(), link_crb=False):
    """Build a C program that prints integers about include/crb.h (sizes, offsets, constants), with gcc and `cflags`,
    run it and return the integers."""
    src, exe = tmp_path / "sz.c", str(tmp_path / "sz")
    src.write_text(c_source)
    link = ["-L", LIBDIR, "-lcrb", f"-Wl,-rpath,{LIBDIR}"] if link_crb else []
    subprocess.check_call(["gcc"] + list(cflags) + ["-I", INCLUDE, str(src), "-o", exe] + link)
    return [int(v) for v in subprocess.check_output([exe]).split()]
