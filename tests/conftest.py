import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the in-tree library is a build artefact (git-ignored): build it when a fresh checkout has none.  A failing
    # build is reported as such -- there is no fallback for the tests to hide behind.
    lib = os.path.join(ROOT, "audiomuse-ai_b200", "libaudiomuse_b200.so")
    if not os.path.exists(lib):
        import __graft_entry__
        __graft_entry__.build()


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
