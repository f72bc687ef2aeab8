import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # tests/sql_golden.py (shared by the CPU and GPU suites)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle binding (test infrastructure; builds oracle/libmzoracle.so on demand)."""
    from oracle import binding

    binding.lib()
    return binding
