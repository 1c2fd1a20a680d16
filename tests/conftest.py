import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine with one)")


def _port():
    from oracle import build_port
    build_port.build()
    from oracle.api import Oracle
    return Oracle("port")


@pytest.fixture(scope="session")
def port():
    """plain-C restatement of the reference (always available: compiled on demand with gcc)"""
    return _port()


@pytest.fixture(scope="session")
def ref(request):
    """the unmodified reference built by oracle/build_ref.py; where oracle/_ref is absent, its recorded answers (tests/ref_replay.py)"""
    from oracle.api import Oracle, available
    from ref_replay import RecordingOracle, ReplayOracle
    if not available("ref"):
        return ReplayOracle()
    if os.environ.get("B200CV_RECORD_REF"):
        rec = RecordingOracle(Oracle("ref"))
        request.addfinalizer(rec.save)
        return rec
    return Oracle("ref")


@pytest.fixture(scope="session")
def oracle():
    """the strongest oracle present: the real reference if built, else the port"""
    from oracle.api import Oracle, available
    return Oracle("ref") if available("ref") else _port()


@pytest.fixture(scope="session")
def cvb():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import opencv_b200 as m
    m.init(0)
    return m


@pytest.fixture()
def rng():
    return np.random.default_rng(0xB200)
