import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    import json
    return json.loads((ROOT / "tests" / "golden" / "reference_golden.json").read_text())


@pytest.fixture(scope="session")
def client():
    """One ComputeClient on cuda:0 through the C ABI; fails loudly (never skips) if the native path is unavailable."""
    from cubecl_b200 import ComputeClient
    c = ComputeClient.load(0)
    yield c
    c.sync()
    for other in list(ComputeClient._clients.values()):   # leave every device idle and released before the process exits
        other.close()
