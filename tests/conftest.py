import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def pkg():
    """The product package with libcdprobe.so built in-tree (nvcc cross-compiles without a GPU)."""
    import cdprobe_pkg

    mod = cdprobe_pkg.load()
    mod.build.build()
    mod.abi.load_library()
    return mod


@pytest.fixture(scope="session")
def oracle():
    """CPU oracle (test infrastructure; see oracle/cdoracle.h)."""
    from oracle import oracle as o

    o.build()
    o.lib()
    return o


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "golden.json")) as f:
        return json.load(f)


def gpu_count() -> int:
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0
