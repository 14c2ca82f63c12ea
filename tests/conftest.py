import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")
    config.addinivalue_line("markers", "sweep: exhaustive device-vs-oracle Unicode sweeps (also marked gpu; -m sweep selects "
                                       "them alone)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    o.lib()
    return o


@pytest.fixture(scope="session")
def ingest():
    """A default handle (block_size 128, seed 1024) — GPU tests only."""
    import xllm_service_b200 as x
    h = x.Ingest(block_size=128, xxh3_seed=1024, device=0)
    yield h
    h.close()
