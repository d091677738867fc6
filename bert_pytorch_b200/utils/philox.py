"""Host-side (numpy) evaluation of the kernels' dropout masks.

Every dropout site of the sm_90a kernels draws its keep decisions from Philox4x32-7 keyed by ``seed`` with the
counter ``(element_index >> 3, stream, 0x5EED)`` -- 128 random bits per group of 8 consecutive elements, 16 bits per
element, kept iff ``bits >= round(p * 65536)`` (ops/csrc/common.cuh: ``Philox::gen`` / ``dropout_keep8`` / ``philox7``).
Reproducing that here lets a test feed the SAME masks to an fp32 autograd oracle and compare gradients tensor by
tensor (VERDICT r1 #8b) instead of only checking statistics.

Element indices: GEMM epilogue dropout ``row * N + col``; attention probabilities ``((b * heads + h) * S + q) * S + k``;
embedding / LayerNorm output dropout ``row * H + col``.  Streams: ``layer * 8 + site`` with site 1 = attention
probabilities, 2 = attention output, 3 = FFN output; the embedding site is ``1023 * 8``.
"""
from __future__ import annotations

import numpy as np

_KA, _KB, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_7(seed: int, idx: np.ndarray, stream: int) -> np.ndarray:
    """[..., 4] uint32 words for the 64-bit counters ``idx`` (same values as ``Philox::gen(seed, idx, stream)``)."""
    idx = np.asarray(idx, dtype=np.uint64)
    x = idx & _M32
    y = idx >> np.uint64(32)
    z = np.full_like(x, np.uint64(stream & 0xFFFFFFFF))
    w = np.full_like(x, np.uint64(0x5EED))
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(7):
        p0 = np.uint64(_KA) * x
        p1 = np.uint64(_KB) * z
        nx = ((p1 >> np.uint64(32)) ^ y ^ np.uint64(k0)) & _M32
        nz = ((p0 >> np.uint64(32)) ^ w ^ np.uint64(k1)) & _M32
        y, w, x, z = p1 & _M32, p0 & _M32, nx, nz
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack([x, y, z, w], axis=-1).astype(np.uint32)


def keep_mask(seed: int, stream: int, numel: int, p_drop: float, first_index: int = 0) -> np.ndarray:
    """Boolean keep decisions of ``numel`` consecutive elements starting at ``first_index`` (multiple of 8)."""
    if p_drop <= 0.0:
        return np.ones(numel, dtype=bool)
    assert first_index % 8 == 0
    thresh = int(p_drop * 65536.0 + 0.5)
    groups = (numel + 7) // 8
    words = philox4x32_7(seed, np.arange(groups, dtype=np.uint64) + np.uint64(first_index // 8), stream)   # [G, 4]
    lo = (words & np.uint32(0xFFFF)).astype(np.uint32)
    hi = (words >> np.uint32(16)).astype(np.uint32)
    fields = np.stack([lo, hi], axis=-1).reshape(groups, 8)       # element t: word t // 2, low half for even t
    return (fields >= thresh).reshape(-1)[:numel]


def keep_scale(p_drop: float) -> float:
    """The kernels' rescale factor of kept elements: 65536 / (65536 - round(p * 65536))."""
    if p_drop <= 0.0:
        return 1.0
    thresh = int(p_drop * 65536.0 + 0.5)
    return 65536.0 / (65536.0 - thresh)


def keep_bits(seed: int, stream: int, rows: int, cols: int, p_drop: float) -> np.ndarray:
    """uint8 [rows, cols // 8]: the packed keep bits of a ``[rows, cols]`` dropout site exactly as ``dropout_mask_kernel``
    writes them (ops/csrc/norm_embed.cu; ``ops.api.dropout_mask``): bit ``t`` of byte ``j`` of a row = element
    ``8 j + t`` kept.  The GEMM epilogue (``mask_in``) and the LayerNorm backward (``keep_mask``) consume this layout."""
    assert cols % 8 == 0
    keep = keep_mask(seed, stream, rows * cols, p_drop).reshape(rows, cols // 8, 8)
    return np.packbits(keep, axis=-1, bitorder="little").reshape(rows, cols // 8)
