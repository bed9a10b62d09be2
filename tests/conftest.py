import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_cuda():
    try:
        from rebel_b200 import capi
        return capi.lib().cfrb_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # GPU tests are selected with -m gpu on a GPU machine.  When somebody runs the whole suite on a CPU-only
    # machine they are skipped (not silently passed); on a GPU machine a missing CUDA library is a hard failure.
    if _has_cuda():
        return
    import shutil
    if shutil.which("nvidia-smi") and os.system("nvidia-smi -L >/dev/null 2>&1") == 0:
        return  # a GPU is there but the library did not load: let the tests fail loudly
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def port():
    from oracle.oracle import Oracle
    return Oracle("port")


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return np.load(os.path.join(GOLDEN, name))
    return load


_W = {}


@pytest.fixture(scope="session")
def net_weights():
    """Flat Net2 weights re-created from seed 0 (pinned by the checksum stored in the fixtures)."""
    def get(D, F):
        if (D, F) not in _W:
            from rebel_b200.models import flatten_state_dict, make_selfplay_net
            _W[(D, F)] = flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())
        return _W[(D, F)]
    return get
