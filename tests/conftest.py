import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden():
    """Committed fixtures: reference test streams + oracle-decoded PCM (tests/golden/make_golden.py)."""
    import numpy as np
    path = os.path.join(ROOT, "tests", "golden", "fixtures.npz")
    return np.load(path, allow_pickle=False)


@pytest.fixture(scope="session", params=["seq", "warp", "generic"])
def ctx(request):
    """Every device path: the fast path (lane-per-frame entropy + lane-per-subframe prediction, with its
    fallback), the earlier warp-per-frame fast path, and the generic kernel alone."""
    import claxon_b200 as cb
    c = cb.Context(device=0, generic_only=(request.param == "generic"), warp_per_frame=(request.param == "warp"),
                   lane_per_frame=(request.param == "seq"))
    yield c
    c.close()
