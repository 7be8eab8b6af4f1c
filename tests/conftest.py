import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle_py as orc
    orc.build()
    orc.lib()
    return orc


@pytest.fixture(scope="session")
def engine():
    """The CUDA engine through the C ABI.  No fallback: a missing library or device is an error."""
    import __graft_entry__ as ge
    from dvo_slam_b200.engine import Engine
    if not os.path.exists(ge.LIB):
        ge.build_cuda()
    eng = Engine(device=0)
    yield eng
    eng.close()


@pytest.fixture(scope="session")
def small_scene():
    """160x120 scene (fr1 intrinsics / 4), 3 usable levels -- the oracle finishes a match in milliseconds."""
    from dvo_slam_b200 import synth
    return synth.SceneConfig(width=160, height=120, intrinsics=tuple(v / 4 for v in synth.FR1_INTRINSICS))
