import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90)")


@pytest.fixture(scope="session")
def kat():
    """The reference's golden vectors (contraction_test_data.json), see tests/golden/make_golden.py."""
    with open(os.path.join(ROOT, "tests", "golden", "contraction_kat.json")) as f:
        raw = json.load(f)
    out = {}
    for name, t in raw["tensors"].items():
        arr = (np.array(t["re"]) + 1j * np.array(t["im"])).reshape(t["shape"])
        out[name] = {"legs": t["legs"], "shape": t["shape"], "data": arr}
    return out


@pytest.fixture(scope="session")
def built_lib():
    """Builds (if needed) and loads libtncb200; CPU-safe."""
    import __graft_entry__ as ge
    ge.build()
    from tnc_b200._lib import lib
    return lib()


@pytest.fixture(scope="session")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()
