import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def orc():
    from tests.checker import get_checker, have
    if not have("orc"):
        import subprocess
        subprocess.check_call(["make", "-s", "-C", str(ROOT / "oracle"), "-f", "Makefile", "oracle"])
    return get_checker("orc")


@pytest.fixture(scope="session")
def ref():
    """The reference's own translation units (oracle/_ref); absent only if the
    prebuilt .so did not travel."""
    from tests.checker import get_checker, have
    if not have("ref"):
        pytest.skip("oracle/_ref/libopenpano_ref.so not built (needs the reference sources)")
    return get_checker("ref")


@pytest.fixture(scope="session")
def engine():
    from openpano_b200.capi import Engine
    eng = Engine(0)
    yield eng
    eng.close()
