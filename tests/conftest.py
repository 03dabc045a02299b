import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Build (or reuse) the native libraries once per session."""
    import __graft_entry__ as g
    need = [("acados_b200", "csrc", "libcuipm.so"), ("oracle", "liboracle_ipm.so"), ("oracle", "libcondense_emul.so")]
    if not all(os.path.exists(os.path.join(ROOT, *p)) for p in need):
        g.build()
    return True
