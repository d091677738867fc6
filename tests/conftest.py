import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (needs an H100)")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords or "multigpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def tiny_config():
    from bert_pytorch_b200 import BertConfig
    return BertConfig(vocab_size_or_config_json_file=512, hidden_size=64, num_hidden_layers=2,
                      num_attention_heads=4, intermediate_size=128, max_position_embeddings=64)


@pytest.fixture(autouse=True)
def _reset_process_wide_kernel_state(request):
    """The extension keeps one process-wide pointer to the device step counter that CUDA-graph replays mix into the
    dropout seed (bindings.cpp: set_seed_step).  A test that captured graphs leaves it set; tests that regenerate
    Philox masks on the host assume the plain seed -- detach it before every GPU test."""
    if "gpu" in request.keywords:
        import torch
        if torch.cuda.is_available():
            from bert_pytorch_b200 import ops
            if ops.available():
                ops.extension().set_seed_step(None)
    yield
