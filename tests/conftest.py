import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def pytest_sessionfinish(session, exitstatus):
    """Dump the parity records the tests collected (parity_utils.RECORDS): measured exact-match rates, margins, errors."""
    try:
        import parity_utils
        parity_utils.dump_records(os.path.join(ROOT, "gpurun_out", "parity_records.json"))
    except Exception:
        pass
