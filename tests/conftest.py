import importlib
import sys
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parent.parent
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))
if str(REPO / "tests") not in sys.path:
    sys.path.insert(0, str(REPO / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90); select with -m gpu")


@pytest.fixture(scope="session")
def garecon():
    return importlib.import_module("aws-global-accelerator-controller_b200")


@pytest.fixture(scope="session")
def oracle():
    ob = importlib.import_module("oracle.binding")
    ob.build()
    return ob


@pytest.fixture(scope="session")
def engine(garecon):
    """One CUDA engine for the whole GPU session (cluster name "default")."""
    import __graft_entry__ as ge
    ge.ensure_built()
    e = garecon.Engine(cluster_name="default", device=0)
    yield e
    e.close()
