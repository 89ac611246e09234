import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PKG = "3d-lidar-multi-object-tracking_b200"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def pkg():
    return importlib.import_module(PKG)


@pytest.fixture(scope="session")
def synth():
    return importlib.import_module(PKG + ".synth")


@pytest.fixture(scope="session")
def ref_intended():
    from oracle import ref
    if not ref.have_ref("intended"):
        pytest.skip("oracle/_ref not built (needs /root/reference; run `make -C oracle ref`)")
    return ref.RefOracle("intended")


@pytest.fixture(scope="session")
def ref_o2():
    from oracle import ref
    if not ref.have_ref("o2"):
        pytest.skip("oracle/_ref not built")
    return ref.RefOracle("o2")


@pytest.fixture(scope="session")
def lm(pkg):
    """One liblmot context on cuda:0 for the whole GPU test session."""
    ctx = pkg.Lmot(device=0)
    yield ctx
    ctx.close()
