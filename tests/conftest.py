import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle.oracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference compiled into oracle/_ref (skips where it is neither built nor buildable)."""
    from oracle import oracle as O
    if not O.ref_available() and not Path("/root/reference/src/ggml.c").exists():
        pytest.skip("oracle/_ref not built and /root/reference absent")
    return O.Ref()
