import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


try:  # property tests run the same examples on every machine: a red suite then always means a regression, not a new draw
    from hypothesis import settings as _hyp_settings

    _hyp_settings.register_profile("pinned", derandomize=True, deadline=None, database=None)
    _hyp_settings.load_profile("pinned")
except ImportError:
    pass
