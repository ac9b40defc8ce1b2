import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "reference_kats.json")) as f:
        return json.load(f)


def pytest_collection_modifyitems(config, items):
    """A wedged kernel must not hang the whole GPU run: every GPU test gets a hard limit (thread method:
    a blocked CUDA call cannot be interrupted by a signal, the process is ended instead)."""
    try:
        import pytest_timeout  # noqa: F401
    except ImportError:
        return
    for item in items:
        if item.get_closest_marker("gpu") and not item.get_closest_marker("timeout"):
            item.add_marker(pytest.mark.timeout(600, method="thread"))
