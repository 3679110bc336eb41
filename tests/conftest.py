import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle_api import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def hostemu():
    import ctypes
    from hotstuff_b200 import build
    lib = ctypes.CDLL(build.build_hostemu())
    lib.emu_verify_generic.restype = ctypes.c_uint
    lib.emu_verify_committee.restype = ctypes.c_uint
    lib.emu_verify_committee_tree.restype = ctypes.c_uint
    return lib


@pytest.fixture(scope="session")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from hotstuff_b200 import build, Engine
    build.build_engine()
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "vectors.json")) as f:
        return json.load(f)
