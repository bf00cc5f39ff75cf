"""CPU: oracle/Makefile on a copy of oracle/ and include/ (never on the tree's own oracle/, whose libraries other tests
have loaded): one make builds every checker and, where the reference tree is present, every reference library; a
second make compiles nothing; and without the reference tree the reference libraries already there are left alone."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = ["liboracle.so"] + [f"liboracle_{n}.so" for n in ("fast", "O0", "dwa", "mptg", "slp", "grid", "rrt", "lqrt")]
REF_LIBS = [f"libref_{n}.so" for n in ("ekf", "pf", "mpc", "lqr4", "lqr5", "dwa", "mptg", "slp", "astar", "dijkstra",
                                       "rrt", "lqrt4", "lqrt5")]
SKIP_LINE = "skipping oracle/_ref"


def _copy(dst):
    shutil.copytree(os.path.join(ROOT, "oracle"), dst / "oracle",
                    ignore=shutil.ignore_patterns("lib", "_ref", "__pycache__"))
    shutil.copytree(os.path.join(ROOT, "include"), dst / "include")
    return dst / "oracle"


def _make(d, *args):
    r = subprocess.run(["make", "-C", str(d), "-j4", *args], capture_output=True, text=True)
    return r.returncode, r.stdout + r.stderr


@pytest.fixture(scope="module", params=["reference", "no_reference"])
def built(request, tmp_path_factory):
    """A copy built once, with the default REF or with REF an empty directory; returns (oracle dir, REF args, output)."""
    base = tmp_path_factory.mktemp("oracle_build")
    d = _copy(base)
    ref = []
    if request.param == "no_reference":
        (base / "empty").mkdir()
        ref = [f"REF={base / 'empty'}"]
    rc, out = _make(d, *ref)
    assert rc == 0, out
    return d, ref, out


def test_one_make_builds_every_library(built):
    d, ref, out = built
    assert sorted(os.listdir(d / "lib")) == sorted(LIBS)
    if ref:
        assert out.count(SKIP_LINE) == 1 and not (d / "_ref").exists(), out
    elif SKIP_LINE in out:
        pytest.skip("no reference tree: the reference libraries are not built")
    else:
        assert sorted(os.listdir(d / "_ref")) == sorted(REF_LIBS)


def test_a_second_make_compiles_nothing(built):
    d, ref, _ = built
    rc, out = _make(d, *ref, "-q")
    assert rc == 0, out
    rc, out = _make(d, *ref, "-n")
    assert rc == 0 and not re.search(r"\b(gcc|g\+\+)\b", out), out


def test_without_the_reference_tree_existing_reference_libraries_are_untouched(tmp_path):
    d = _copy(tmp_path)
    empty = tmp_path / "empty"
    empty.mkdir()
    (d / "_ref").mkdir()
    dummy = d / "_ref" / "libref_ekf.so"
    dummy.write_bytes(b"built where the reference tree is")
    mtime = dummy.stat().st_mtime_ns
    for force in ([], ["-B"]):
        rc, out = _make(d, f"REF={empty}", *force)
        assert rc == 0, out
        assert out.count(SKIP_LINE) == 1, out
        assert os.listdir(d / "_ref") == ["libref_ekf.so"]
        assert dummy.read_bytes() == b"built where the reference tree is" and dummy.stat().st_mtime_ns == mtime
    assert sorted(os.listdir(d / "lib")) == sorted(LIBS)
