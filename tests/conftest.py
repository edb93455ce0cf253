import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: `pytest -m gpu`)")


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a CUDA device: on a box without one (this container) a plain `pytest tests/` skips them
    instead of failing at the first driver call."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (run on an H100 with `-m gpu`)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def pytest_sessionstart(session):
    """The engine library is a build artefact (git-ignored). If a checkout has not been built yet, build it once
    (nvcc cross-compiles sm_90a without a GPU) so that the ABI tests exercise the real thing."""
    import subprocess
    lib = os.path.join(ROOT, "sparse_coding_b200", "libsce.so")
    if not os.path.exists(lib):
        subprocess.run(["make", "-C", ROOT, "all"], check=True, stdout=subprocess.DEVNULL)


@pytest.fixture(scope="session")
def golden():
    import torch

    def load(name):
        return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)

    return load
