import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    config.addinivalue_line("markers", "tf32: run the decoder MLP on the tensor-core TF32 path (default in tests: strict-FP32 path)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _decoder_math_mode(request, monkeypatch):
    """Parity tests with tight tolerances run the decoder MLP on the strict-FP32 CUDA-core path; tests marked `tf32`
    exercise the production tensor-core TF32 path with the (looser) tolerances SURVEY.md Appendix C assigns to it."""
    if "tf32" in request.keywords:
        monkeypatch.delenv("GA_DECODER_FP32", raising=False)
    else:
        monkeypatch.setenv("GA_DECODER_FP32", "1")
