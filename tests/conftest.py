import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `pytest -m gpu`)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        n = 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and n == 0:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and n < 2:
            item.add_marker(skip_multi)


@pytest.fixture
def workdir(tmp_path, monkeypatch):
    """Run inside a scratch cwd: the trainer writes tensorboard/, checkpoints/, results.csv there."""
    monkeypatch.chdir(tmp_path)
    return tmp_path
