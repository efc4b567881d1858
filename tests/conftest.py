import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ws():
    import websplat_b200
    return websplat_b200


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def ctx(ws):
    return ws.Context(0)
