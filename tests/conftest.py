import json
import sys
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parent.parent
GOLDEN = REPO / "tests" / "golden"
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built_lib():
    """Build (or reuse) the in-tree shared object; never silently skipped."""
    from kakveda_b200 import build

    return build.build()


def load_golden(name: str):
    return json.loads((GOLDEN / name).read_text(encoding="utf-8"))


@pytest.fixture(scope="session")
def golden():
    return load_golden
