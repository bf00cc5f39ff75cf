import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine with one)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure libcrb.so and liboracle.so exist (the driver runs build() first; this covers a bare
    `pytest` in a fresh checkout).  On the GPU box the prebuilt files travel with the snapshot."""
    import __graft_entry__ as g
    from cpprobotics_b200 import _lib
    from oracle import oracle as O
    if not os.path.exists(_lib.LIB_PATH):
        g.build_libcrb()
    if not os.path.exists(O.LIB_PATH):
        g.build_oracle()


@pytest.fixture(scope="session")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from cpprobotics_b200 import Engine
    e = Engine(0)
    yield e
    e.close()
