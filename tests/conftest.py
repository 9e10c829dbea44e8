import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_cuda = torch.cuda.is_available()
    except Exception:
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def _reference(request, name):
    # the reference's kernels, or their recorded outputs (tests/refreplay.py)
    import refreplay
    from oracle.build_ref import built, load_ref
    mod = load_ref("_ref_" + name) if (refreplay.RECORD or built("_ref_" + name)) else None
    if refreplay.RECORD:
        request.addfinalizer(refreplay.save_all)
    # recordings are keyed by test file name and test name (with parameters): independent of the directory pytest runs from
    return refreplay.Replay(name, mod, f"{os.path.basename(str(request.node.fspath))}::{request.node.name}")


@pytest.fixture
def ref_raymarching(request):
    return _reference(request, "raymarching")


@pytest.fixture
def ref_gridencoder(request):
    return _reference(request, "gridencoder")


@pytest.fixture
def ref_shencoder(request):
    return _reference(request, "shencoder")
