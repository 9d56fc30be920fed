import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box with -m gpu)")
    config.addinivalue_line("markers", "slow: multi-minute CPU test (full-width 1.5-2.6 B parameter UNets through the ops "
                                       "emulator); skipped unless CA_RUN_SLOW=1")


def pytest_collection_modifyitems(config, items):
    if os.environ.get("CA_RUN_SLOW") == "1":
        return
    skip = pytest.mark.skip(reason="slow CPU test: set CA_RUN_SLOW=1 to run")
    for item in items:
        if "slow" in item.keywords:
            item.add_marker(skip)
