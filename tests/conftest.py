import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXT_DIR = os.path.join(ROOT, "stable-diffusion-webui-distributed_b200")
HOSTSTUB = os.path.join(ROOT, "tests", "hoststub")   # stand-in for sdwui's `modules` / `gradio` (test infrastructure)
for p in (ROOT, EXT_DIR, HOSTSTUB):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")
    try:   # fp32 references are IEEE fp32 on the GPU too (cuDNN's default lets fp32 convolutions use TF32 tensor cores)
        import torch
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    except Exception:  # pragma: no cover
        pass


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
