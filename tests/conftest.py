"""pytest configuration: registers the `gpu` marker (tests that need a real H100)."""
import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def rpx_lib():
    """The built engine library (builds it in-tree if it is missing)."""
    from reprover_b200 import _build, _native

    if not _native.library_path().exists():
        _build.build_engine()
    return _native.load()


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("a `gpu`-marked test ran without a CUDA device (select with -m gpu on an H100 machine)")
    return torch.device("cuda:0")


@pytest.fixture(scope="session")
def out_dir():
    d = ROOT / "gpurun_out"
    d.mkdir(exist_ok=True)
    return d
