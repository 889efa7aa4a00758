import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def gpu():
    """Initialise libggml_b200 on cuda:0.  No fallback: fails loudly if the library or the GPU is missing."""
    import ggllm_cpp_b200.binding as b
    b.init(0)
    return b


@pytest.fixture(scope="session")
def orc():
    import pyoracle as po
    return po.orc()
