"""The in-tree extension must export every entry point the Python layer calls (a renamed or forgotten binding would only
show up on a GPU box otherwise).  Importing ``_C.so`` needs no device: it is skipped when the file has not been built."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "bert_pytorch_b200")


def _called_names():
    names = set()
    for dirpath, _, files in os.walk(PKG):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                names |= set(re.findall(r"extension\(\)\.([A-Za-z_][A-Za-z0-9_]*)\(", src))
    for f in os.listdir(os.path.join(ROOT, "tools")):
        if f.endswith(".py"):
            src = open(os.path.join(ROOT, "tools", f)).read()
            names |= set(re.findall(r"\bC\.([a-z_][A-Za-z0-9_]*)\(", src)) if "load_extension()" in src else set()
    return names


def test_every_binding_the_python_layer_calls_exists():
    from bert_pytorch_b200.ops import _loader
    if not os.path.exists(_loader.extension_path()):
        pytest.skip("extension not built (python -m bert_pytorch_b200.ops.build)")
    mod = _loader.load_extension()
    called = _called_names()
    assert len(called) > 25, called                      # the scan itself found the API
    missing = sorted(n for n in called if not hasattr(mod, n))
    assert not missing, missing


def test_build_script_lists_every_cuda_source():
    from bert_pytorch_b200.ops import build
    on_disk = sorted(f for f in os.listdir(build.CSRC) if f.endswith(".cu"))
    assert sorted(build.CUDA_SOURCES) == on_disk


def test_tile_variant_heuristic_sends_the_bert_large_shapes_to_the_cta_pair_kernel():
    """(The name dates from a 2-CTA kernel; the wide variant is the 128 x 256 tile now.)
    ops.api.pick_block_n: every GEMM of a BERT-large layer (and the vocabulary projection) runs on 128 x 256 tiles;
    the fine-tuning heads (N padded to 8) run on 128 x 128 tiles, one-row-block problems on whichever fills more SMs."""
    from bert_pytorch_b200.ops import api
    for M, N in ((12288, 1024), (12288, 3072), (12288, 4096), (1920, 30528), (8192, 1024), (4096, 1024)):
        assert api.pick_block_n(M, N) == 256, (M, N)
    assert api.pick_block_n(12288, 8) == 128            # QA / token-classification heads
    assert api.pick_block_n(96, 1024) in (128, 256)     # pooler: one 128-row block, whichever fills more SMs
    assert api.pick_block_n(128, 4096) in (128, 256)
    assert api.pick_block_n(1024, 1024) in (128, 256)
    # the narrow variant only when it wastes (clearly) fewer SM slots in the last wave
    assert api._pick_block_n(128, api.NUM_SMS * 128) == 128
