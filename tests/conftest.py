import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "python-audio-separator_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def lib_built():
    """Build libb200sep.so if it is missing or stale (nvcc cross-compiles without a GPU)."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("b200_build", os.path.join(ROOT, "python-audio-separator_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build(verbose=False)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
