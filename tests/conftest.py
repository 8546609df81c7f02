import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")
    config.addinivalue_line("markers", "gpu_extra: extra GPU property tests, opt-in: B200_RUN_EXTRA=1 pytest -m gpu_extra")


@pytest.fixture(scope="session")
def goldens():
    import json

    with open(os.path.join(ROOT, "tests", "golden", "reference_goldens.json")) as f:
        return json.load(f)
