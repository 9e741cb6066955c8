import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# Property tests draw the SAME examples on every run and on every box (and keep no example database): a green
# suite here is a green suite at the round-end run, not a new random sample.
try:
    from hypothesis import settings as _hyp_settings

    _hyp_settings.register_profile("repo", derandomize=True, deadline=None, database=None)
    _hyp_settings.load_profile("repo")
except ImportError:  # hypothesis is optional for the non-property tests
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    # -m gpu tests must never silently pass on a box without a GPU
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
