"""Hand written sm_90a kernels and their bindings.

``available()`` is true when a CUDA device is present *and* the in-tree extension
``_C.so`` (built by :mod:`bert_pytorch_b200.ops.build`, sources in ``csrc/``) loads.  On a GPU
box a missing/broken extension is a hard error -- the fused engine must never fall back
silently to eager PyTorch (set ``B200_ALLOW_EAGER=1`` to opt into the oracle path, e.g. to
bisect a numerics issue).
"""
from __future__ import annotations

import os

import torch

_C = None
_ERR = None
_TRIED = False


def _load():
    global _C, _ERR, _TRIED
    if _TRIED:
        return _C
    _TRIED = True
    try:
        from . import _loader
        _C = _loader.load_extension()
    except Exception as e:  # noqa: BLE001
        _ERR = e
        _C = None
    return _C


def extension():
    """The loaded extension module; raises if it is not usable."""
    c = _load()
    if c is None:
        raise RuntimeError(f"bert_pytorch_b200 CUDA extension is not available: {_ERR!r}. "
                           "Build it with `python -m bert_pytorch_b200.ops.build`.")
    return c


def available() -> bool:
    if not torch.cuda.is_available():
        return False
    if os.environ.get("B200_ALLOW_EAGER") == "1" and os.environ.get("B200_FORCE_EAGER") == "1":
        return False
    if _load() is None:
        if os.environ.get("B200_ALLOW_EAGER") == "1":
            return False
        raise RuntimeError(
            f"CUDA device present but the sm_90a extension failed to load: {_ERR!r}. Refusing to "
            "fall back to eager PyTorch silently (export B200_ALLOW_EAGER=1 to allow it).")
    return True


_SUBMODULES = ("api", "native_host", "build", "_loader")


def __getattr__(name):
    # lazily expose submodules and the python wrappers (ops.gemm, ops.layer_norm, ...)
    import importlib
    if name in _SUBMODULES:
        return importlib.import_module(f"{__name__}.{name}")
    if name.startswith("__"):
        raise AttributeError(name)
    api = importlib.import_module(f"{__name__}.api")
    if hasattr(api, name):
        return getattr(api, name)
    raise AttributeError(name)
