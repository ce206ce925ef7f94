import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def checker_libs():
    """Build the checker libraries (oracle restatement; oracle/_ref where the reference is mounted)."""
    import checker
    checker.build_oracle()
    return checker


@pytest.fixture(scope="session")
def gpu_decoder_factory():
    """Decoder factory for -m gpu tests; fails loudly (never falls back) without the CUDA library."""
    from dump1090_b200 import api

    made = []

    def make(**cfg):
        d = api.Decoder(**cfg)
        made.append(d)
        return d

    yield make
    for d in made:
        d.close()
