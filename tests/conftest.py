import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    return pyoracle.Oracle()


@pytest.fixture(scope="session")
def ref_cpu():
    from tests.refreplay import reference
    ref = reference("cpu")
    if ref is None:
        pytest.skip("oracle/_ref not built and no recorded reference outputs")
    return ref


@pytest.fixture(scope="session")
def ref_avx2():
    from tests.refreplay import reference
    ref = reference("avx2")
    if ref is None:
        pytest.skip("oracle/_ref not built and no recorded reference outputs")
    return ref
