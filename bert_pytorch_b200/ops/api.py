"""Python wrappers over the sm_90a extension (``_C.so``).

Thin: allocate outputs, pick tile/split heuristics, translate enums.  No autograd here -- the
fused engine (models/fused.py) calls forward and backward kernels explicitly.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import extension

# GEMM enums (csrc/gemm_sm90.h)
NT, NN, TN = 0, 1, 2
EPI_NONE, EPI_BIAS, EPI_BIAS_DROP_RES, EPI_ADD, EPI_ACCUM_F32, EPI_BIAS_TANH, EPI_F32, EPI_BIAS_GELU_DG, EPI_MUL = (
    0, 1, 3, 4, 6, 7, 8, 9, 10)

NUM_SMS = 132           # H100 SXM; only the tile heuristics below use it (the kernels ask the device)
KERNEL_LAUNCHES = 0     # every wrapper bumps this: bench.py reports it as ``gpu_launches``


def deterministic() -> bool:
    """Deterministic mode: the wrappers below take fixed-order forms of every floating-point sum whose order would
    otherwise depend on CTA scheduling (split-K weight gradients, bias gradients, attention dQ, the embedding scatter,
    the losses, the optimizer norms), so that the same program on the same inputs, GPU and build gives the same bits.
    On with ``B200_DETERMINISTIC=1`` or ``torch.use_deterministic_algorithms(True)``."""
    return os.environ.get("B200_DETERMINISTIC", "0") == "1" or torch.are_deterministic_algorithms_enabled()


def use_deterministic() -> None:
    """What the runners' ``--deterministic`` does, before CUDA starts: torch's flag (which also switches this module
    into deterministic mode) and the cuBLAS workspace setting it needs for the torch ops around the engine (fine-tuning
    heads, cross-entropy).  torch's fill of uninitialised memory stays off: every engine output and workspace is written
    in full before it is read, so the fill would only cost a memset per allocation."""
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False


def pick_block_n(M: int, N: int, epi: int = EPI_NONE) -> int:
    """The tile width :func:`gemm` chooses for an [M, N] output with epilogue ``epi`` (128 x 256 or 128 x 128
    tiles)."""
    return _pick_block_n(M, N, epi)


def _count(n: int = 1) -> None:
    global KERNEL_LAUNCHES
    KERNEL_LAUNCHES += n


# bias + GELU + GELU' is long enough that on 128 x 128 tiles, where the kernel runs it ping-pong under the other
# warpgroup's MMAs, it measured 6 % faster on H100 at the BERT-large FFN-1 shape than on the 128 x 256 tile whose two
# warpgroups run the epilogue together.  The epilogues that read a residual or saved factor stage it through shared
# memory and measured 1-12 % faster on 128 x 256 tiles (tools/gemm_bench.py --epi).
_HEAVY_EPI = (EPI_BIAS_GELU_DG,)


def _pick_block_n(M: int, N: int, epi: int = EPI_NONE) -> int:
    """128 for N <= 128 and for bias + GELU + GELU'; otherwise 256 (128 x 256 tiles: half the A-operand traffic per
    FLOP) unless the narrow tiles waste clearly fewer SM slots in the last wave."""
    if N <= 128 or epi in _HEAVY_EPI:
        return 128
    m_blocks = (M + 127) // 128
    t256 = m_blocks * ((N + 255) // 256)
    t128 = m_blocks * ((N + 127) // 128)

    def eff(tiles: int) -> float:
        waves = math.ceil(tiles / NUM_SMS)
        return tiles / (waves * NUM_SMS) if tiles else 0.0
    return 256 if eff(t256) >= eff(t128) - 0.08 else 128


def gemm(a: torch.Tensor, b: torch.Tensor, *, layout: int = NT, epi: int = EPI_NONE,
         out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
         res: Optional[torch.Tensor] = None, aux_out: Optional[torch.Tensor] = None, k_splits: int = 1,
         block_n: Optional[int] = None, alpha: float = 1.0, p_drop: float = 0.0, seed: int = 0,
         stream: int = 0, scale_a: Optional[torch.Tensor] = None, scale_b: Optional[torch.Tensor] = None,
         a_e5m2: bool = False, b_e5m2: bool = False, push: bool = False,
         colsum: Optional[torch.Tensor] = None, mask_out: Optional[torch.Tensor] = None,
         mask_in: Optional[torch.Tensor] = None) -> torch.Tensor:
    """wgmma GEMM with a fused epilogue (see csrc/gemm_sm90.cu).  ``a``/``b`` are 2-D bf16, or -- with
    ``scale_a``/``scale_b`` (device inv-scale scalars from an :class:`Fp8Meta`) -- 1-byte fp8 tensors.
    ``colsum`` (fp32 [N], EPI_NONE / EPI_ADD / EPI_MUL): accumulates the column sums of the bf16 output (a bias
    gradient that would otherwise need its own pass over the tensor).  ``mask_out`` (uint8 [M, N / 8],
    EPI_BIAS_DROP_RES): receives the dropout keep bits, which :func:`layer_norm_bwd` can read
    back (``keep_mask``) instead of regenerating them.
    Deterministic mode: EPI_ACCUM_F32 runs without split-K (:func:`wgrad_accumulate` splits in order itself), and
    ``colsum`` is a separate fixed-order column sum of the output (the same bf16 values the epilogue would have
    summed)."""
    det = deterministic()
    if det:
        k_splits = 1 if epi == EPI_ACCUM_F32 else k_splits
        colsum, det_colsum = None, colsum
    if layout == NT:
        M, N = a.size(0), b.size(0)
    elif layout == NN:
        M, N = a.size(0), b.size(1)
    else:
        M, N = a.size(1), b.size(1)
    if out is None:
        dt = torch.float32 if epi in (EPI_ACCUM_F32, EPI_F32) else torch.bfloat16
        out = torch.empty(M, N, dtype=dt, device=a.device)
    if block_n is None:
        block_n = _pick_block_n(M, N, epi)
    extension().gemm(a, b, out, layout, epi, bias, res, aux_out, k_splits, block_n, alpha, p_drop, seed, stream,
                     scale_a, scale_b, a_e5m2, b_e5m2, push, colsum, mask_out, mask_in)
    _count()
    if det and det_colsum is not None:
        colsum_accumulate(out, det_colsum)
    return out


class Fp8Meta:
    """Device-resident per-tensor scaling records ``{amax, scale, inv_scale, _}`` for the fp8 GEMM path
    (delayed scaling: quantise with the scale derived from the previous step's amax; csrc/fp8.cu)."""

    def __init__(self, sites: Sequence[str], e5m2: Sequence[bool], device, margin: float = 1.0):
        self.index = {name: i for i, name in enumerate(sites)}
        self.e5m2 = list(bool(x) for x in e5m2)
        self.table = torch.zeros(len(sites), 4, dtype=torch.float32, device=device)
        self.table[:, 1:3] = 1.0
        self.flags = torch.tensor([1 if x else 0 for x in self.e5m2], dtype=torch.int32, device=device)
        self.margin = float(margin)

    def record(self, site) -> torch.Tensor:
        return self.table[self.index[site] if isinstance(site, str) else site]

    def inv_scale(self, site) -> torch.Tensor:
        return self.record(site)[2:3]

    def is_e5m2(self, site) -> bool:
        return self.e5m2[self.index[site] if isinstance(site, str) else site]

    def quantize(self, x: torch.Tensor, site, out: Optional[torch.Tensor] = None, calibrate: bool = False) -> torch.Tensor:
        """bf16 -> fp8 bytes with the site's current scale; records amax for the next ``update``.  With
        ``calibrate`` the scale is first derived from this very tensor (current scaling, one extra pass)."""
        ext = extension()
        rec = self.record(site)
        e5 = self.is_e5m2(site)
        if calibrate:
            ext.fp8_amax(x, rec)
            i = self.index[site] if isinstance(site, str) else site
            ext.fp8_update(self.table[i:i + 1], self.flags[i:i + 1], self.margin)
            _count(2)
        if out is None:
            out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
        ext.fp8_quantize(x, out, rec, e5)
        _count()
        return out

    def update(self) -> None:
        """new scales from the amaxes seen since the last update (one tiny launch for all sites)"""
        extension().fp8_update(self.table, self.flags, self.margin)
        _count()


def wgrad_splits(n_out: int, k_out: int, reduce_len: int, block_n: int = 256) -> int:
    """Split-K factor for dW[n_out, k_out]: as many K ranges as keep the work units (tiles x splits) within one unit
    per SM of the persistent grid.  More splits only add fp32 reduction traffic once every SM has a unit, and a
    fraction of a second unit per SM leaves the others idle for a whole unit."""
    tiles = ((n_out + 127) // 128) * ((k_out + block_n - 1) // block_n)
    kb = max(1, (reduce_len + 63) // 64)
    want = max(1, NUM_SMS // max(tiles, 1))
    return max(1, min(want, kb // 4 if kb >= 8 else 1, 32))


def wgrad_accumulate(dy: torch.Tensor, x: torch.Tensor, grad: torch.Tensor, alpha: float = 1.0, push: bool = False,
                     **fp8) -> None:
    """grad[N,K] (fp32, arena view) += dy[M,N]^T @ x[M,K]  (``fp8``: scale_a / scale_b / a_e5m2 for 1-byte operands)."""
    n_out, k_out = grad.shape
    bn = 256 if k_out >= 256 else _pick_block_n(n_out, k_out)
    splits = wgrad_splits(n_out, k_out, dy.size(0) // (2 if fp8 else 1), bn)
    if splits > 1 and deterministic():
        if extension().grad_peers_world() > 1:
            # the gradient arenas are registered with the peer-memory backend: peers add into this arena and the GEMMs
            # push tiles to their owners, which a plain read-modify-write of the partials would race with
            raise RuntimeError("deterministic mode covers one GPU; it cannot run with the peer-memory gradient backend "
                               "(--backend fused)")
        # the split-K partition done in order: each range of 128-row blocks of the reduction is stored plainly to its
        # own fp32 partial, and the partials are added to the gradient in range order.  (Not one split: an fp8 wgmma
        # accumulates with less than fp32 precision, so the whole reduction in one pass would lose accuracy.)
        M = dy.size(0)
        step = -(-M // (splits * 128)) * 128
        parts = torch.empty(-(-M // step), n_out, k_out, dtype=torch.float32, device=grad.device)
        for s in range(parts.size(0)):
            gemm(dy[s * step:(s + 1) * step], x[s * step:(s + 1) * step], layout=TN, epi=EPI_F32, out=parts[s],
                 block_n=bn, alpha=alpha, **fp8)
        extension().ordered_sum(parts, grad)
        _count()
        return
    # ``push``: with the peer-memory backend in push mode the tiles go to the owner rank's arena (GEMM -> reduce-scatter)
    gemm(dy, x, layout=TN, epi=EPI_ACCUM_F32, out=grad, block_n=bn, alpha=alpha, k_splits=splits, push=push, **fp8)


def _fp8_side(fp8, like: torch.Tensor):
    """``fp8`` = (Fp8Meta, site) -> (q tensor, meta record, e5m2) for a kernel's fused fp8 copy of its output."""
    if fp8 is None:
        return None, None, False
    meta, site = fp8
    return torch.empty(like.shape, dtype=torch.uint8, device=like.device), meta.record(site), meta.is_e5m2(site)


def layer_norm_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, eps: float = 1e-12,
                   save_stats: bool = True, fp8=None):
    """``fp8=(meta, site)``: also emit the fp8 copy of y (delayed scaling) -> returns (y, mean, rstd, q)."""
    y = torch.empty_like(x)
    M = x.numel() // x.size(-1)
    mean = torch.empty(M, dtype=torch.float32, device=x.device) if save_stats else None
    rstd = torch.empty(M, dtype=torch.float32, device=x.device) if save_stats else None
    q, rec, e5 = _fp8_side(fp8, x)
    extension().layer_norm_fwd(x, gamma, beta, y, mean, rstd, eps, q, rec, e5)
    _count()
    return (y, mean, rstd) if fp8 is None else (y, mean, rstd, q)


_LN_WS: Dict[Tuple[int, int], torch.Tensor] = {}


def _ln_workspace(M: int, H: int, device: torch.device) -> torch.Tensor:
    """One workspace per (device, H), sized for the largest grid the LN backward launches (the grid stops growing at a
    few CTAs per SM), so that any row count fits -- the unpadded engine sees a new M every batch.  Entries are never
    replaced: captured CUDA graphs keep their pointers."""
    key = (device.index or 0, H)
    ws = _LN_WS.get(key)
    if ws is None:
        ws = torch.empty(extension().ln_bwd_workspace(1 << 30, H), dtype=torch.float32, device=device)
        _LN_WS[key] = ws
    return ws


NO_STREAM = 0xFFFFFFFF


def dropout_mask(M: int, N: int, p_drop: float, seed: int, stream: int, device) -> torch.Tensor:
    """uint8 [M, N / 8] keep bits of the dropout stream ``(seed, stream)`` over an [M, N] tensor -- the decisions the
    kernels would draw themselves.  Feed it to ``gemm(..., mask_in=)`` (EPI_BIAS_DROP_RES) and to
    ``layer_norm_bwd(..., keep_mask=)``: Philox then runs once per element, in a kernel that keeps the whole machine
    busy, instead of in the latency-bound GEMM epilogue and again in the LayerNorm backward."""
    out = torch.empty(M, N // 8, dtype=torch.uint8, device=device)
    extension().dropout_mask(out, p_drop, seed, stream)
    _count()
    return out


def layer_norm_bwd(dy: torch.Tensor, x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, gamma: torch.Tensor, *,
                   dgamma: Optional[torch.Tensor], dbeta: Optional[torch.Tensor], dbias: Optional[torch.Tensor] = None,
                   want_dropped: bool = False, p_drop: float = 0.0, seed: int = 0, drop_stream: int = 0,
                   in_stream: int = NO_STREAM, fp8=None, keep_mask: Optional[torch.Tensor] = None):
    """Returns (dx, dx_dropped or None).  ``dgamma``/``dbeta``/``dbias`` are *accumulated into*.
    ``keep_mask`` (uint8 [M, H / 8]): the keep bits of the ``drop_stream`` dropout as written by the producing GEMM
    (``gemm(mask_out=...)``); without it the decisions are regenerated from the Philox stream (same bits).
    ``fp8=(meta, site)`` (with ``want_dropped``): also the fp8 copy of dx_dropped -> (dx, dxd, q)."""
    dx = torch.empty_like(x)
    dxd = torch.empty_like(x) if want_dropped else None
    M, H = x.numel() // x.size(-1), x.size(-1)
    q, rec, e5 = _fp8_side(fp8 if want_dropped else None, x)
    extension().layer_norm_bwd(dy, x, mean, rstd, gamma, dx, dxd, dgamma, dbeta, dbias, _ln_workspace(M, H, x.device),
                               p_drop, seed, drop_stream, in_stream, q, rec, e5, keep_mask, deterministic())
    _count(2)
    return (dx, dxd) if fp8 is None else (dx, dxd, q)


def colsum_accumulate(x: torch.Tensor, out: torch.Tensor) -> None:
    """out[N] (fp32) += x[M,N].sum(0)"""
    det = deterministic()
    extension().colsum(x, out, det)
    _count(2 if det else 1)


def gelu_fwd(x: torch.Tensor, fp8=None):
    y = torch.empty_like(x)
    q, rec, e5 = _fp8_side(fp8, x)
    extension().gelu_fwd(x, y, q, rec, e5)
    _count()
    return y if fp8 is None else (y, q)


def dgelu_bwd(dy: torch.Tensor, x: torch.Tensor, dbias: Optional[torch.Tensor] = None, fp8=None):
    """dy * gelu'(x); ``dbias`` (fp32 [N]) accumulates the column sums of the result (of its fp32 values, before the
    bf16 rounding; deterministic mode: per-block sums finished in a fixed order)."""
    dx = torch.empty_like(dy)
    q, rec, e5 = _fp8_side(fp8, dy)
    det = deterministic() and dbias is not None
    extension().dgelu_bwd(dy, x, dx, dbias, q, rec, e5, det)
    _count(2 if det else 1)
    return dx if fp8 is None else (dx, q)


def embedding_fwd(ids, seg, word, pos, type_emb, gamma, beta, S: int, *, eps=1e-12, p_drop=0.0, seed=0, stream=0,
                  pos_ids: Optional[torch.Tensor] = None):
    """``pos_ids`` (int32, one per id): the position row of every token, for packed rows of an unpadded batch;
    without it token ``i`` sits at position ``i % S``."""
    M, H = ids.numel(), word.size(1)
    e = torch.empty(M, H, dtype=torch.bfloat16, device=ids.device)
    y = torch.empty_like(e)
    mean = torch.empty(M, dtype=torch.float32, device=ids.device)
    rstd = torch.empty_like(mean)
    extension().embedding_fwd(ids, seg, word, pos, type_emb, gamma, beta, e, y, mean, rstd, S, eps, p_drop, seed, stream,
                              pos_ids)
    _count()
    return y, e, mean, rstd


def embedding_bwd_scatter(de, ids, seg, gword, gpos, gtype, S: int, *, pos_ids: Optional[torch.Tensor] = None) -> None:
    """Deterministic mode: the rows are sorted by table row and every table row is summed by one owner in token order
    (32768 token rows at a time, the chunks added in order)."""
    det = deterministic()
    extension().embedding_bwd_scatter(de, ids, seg, gword, gpos, gtype, S, pos_ids, det)
    _count(9 if det else 2)


def mlm_compact(labels: torch.Tensor, max_pred: int, row_map: Optional[torch.Tensor] = None):
    """``row_map`` (int32 [B * S], from :func:`pack_tokens`): ``idx`` holds packed rows instead of ``b * S + s``, and a
    label whose token is masked is dropped (not counted)."""
    B = labels.size(0)
    idx = torch.empty(B * max_pred, dtype=torch.int32, device=labels.device)
    tgt = torch.empty_like(idx)
    count = torch.empty(1, dtype=torch.int32, device=labels.device)
    if row_map is None:
        extension().mlm_compact(labels, max_pred, idx, tgt, count)
    else:
        extension().mlm_compact(labels, max_pred, idx, tgt, count, row_map)
    _count()
    return idx, tgt, count


def pack_tokens(input_mask: torch.Tensor, input_ids: torch.Tensor, segment_ids: Optional[torch.Tensor], T_cap: int,
                D: int):
    """Packs the unmasked tokens of a [B, S] batch into ``T_cap`` rows on the device, with no host sync (it runs inside
    a captured graph).  Returns int32 ``(ids, seg, pos_ids, cu_seqlens, cls_rows, row_map)``:

    * ``ids``, ``seg``, ``pos_ids`` [T_cap]: token id, segment and position of every unmasked token in ``b * S + s``
      order, then the pad tail (id 0, segment 0, position inside its dummy sequence);
    * ``cu_seqlens`` [B + D + 1]: the B sequences, then D dummy sequences of at most S rows over the pad tail;
    * ``cls_rows`` [B]: first packed row of every sequence; ``row_map`` [B * S]: packed row of every token, -1 if masked.

    A row without any unmasked token packs as S tokens (the padded attention computes it with every key valid).
    ``D * S`` must cover the pad tail ``T_cap - T`` (:func:`bert_pytorch_b200.models.fused.token_bucket`)."""
    B, S = input_mask.shape
    dev = input_mask.device

    def i32(t):
        return t.reshape(B, S).to(torch.int32).contiguous()
    ids = torch.empty(T_cap, dtype=torch.int32, device=dev)
    seg, pos = torch.empty_like(ids), torch.empty_like(ids)
    cu = torch.empty(B + D + 1, dtype=torch.int32, device=dev)
    cls = torch.empty(B, dtype=torch.int32, device=dev)
    row_map = torch.empty(B * S, dtype=torch.int32, device=dev)
    extension().pack_tokens(i32(input_mask), i32(input_ids), None if segment_ids is None else i32(segment_ids),
                            T_cap, D, ids, seg, pos, cu, cls, row_map)
    _count()
    return ids, seg, pos, cu, cls, row_map


def gather_rows(src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    dst = torch.empty(idx.numel(), src.size(-1), dtype=src.dtype, device=src.device)
    extension().gather_rows(src, idx, dst)
    _count()
    return dst


def scatter_rows(src: torch.Tensor, idx: torch.Tensor, dst: torch.Tensor) -> None:
    extension().scatter_rows(src, idx, dst)
    _count()


def nsp_head_(pooled: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, labels: torch.Tensor, grad_scale: float,
              loss_out: torch.Tensor, dw: torch.Tensor, db: torch.Tensor) -> torch.Tensor:
    """NSP classifier [B,H] x [H,2] + cross-entropy (ignore_index -1) + backward in one launch: ``loss_out`` += mean CE,
    ``dw`` / ``db`` (fp32) accumulate the classifier gradients, returns dz = d loss / d (pooler pre-activation) [B,H]
    bf16 (tanh' of the pooler folded in)."""
    dz = torch.empty_like(pooled)
    det = deterministic()
    extension().nsp_head(pooled, w, bias, labels, grad_scale, loss_out, dz, dw, db, det)
    _count(4 if det else 1)
    return dz


CLS_CLASSES = (2, 3)    # the instantiated class counts of cls_head (the GLUE classification tasks)


def _check_classes(w: torch.Tensor) -> None:
    if w.dim() != 2 or w.size(0) not in CLS_CLASSES:
        raise ValueError(f"cls_head: {w.size(0) if w.dim() == 2 else '?'} classes; the kernel is built for "
                         f"C in {CLS_CLASSES}")


def cls_head_(pooled: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, labels: torch.Tensor, grad_scale: float,
              loss_out: torch.Tensor, dw: torch.Tensor, db: torch.Tensor, p_drop: float = 0.0, seed: int = 0,
              stream: int = 0) -> torch.Tensor:
    """Sequence-classification head after the pooler in one launch: dropout ``p_drop`` on the pooled bf16 [B, H]
    (Philox ``(seed, stream)``, element ``b * H + i``), logits = dropped @ ``w``^T + ``bias`` (``w`` bf16 [C, H], C = 2
    or 3; fp32 ``bias``), and mean cross-entropy over the rows whose int64 label lies in [0, C).  ``loss_out`` += the
    mean, ``dw`` / ``db`` (fp32) accumulate the classifier gradients (atomics, or per-row partials added in order in
    deterministic mode); returns dz = d loss / d (pooler pre-activation) [B, H] bf16 (dropout and tanh' folded in).
    With no valid row the loss and every gradient are zero."""
    _check_classes(w)
    dz = torch.empty_like(pooled)
    det = deterministic()
    extension().cls_head(pooled, w, bias, labels, grad_scale, seed, stream, p_drop, loss_out, dz, dw, db, det)
    _count(4 if det else 1)
    return dz


def cls_logits(pooled: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """Evaluation form of :func:`cls_head_`: fp32 logits [B, C] of the pooled bf16 [B, H], without dropout."""
    _check_classes(w)
    out = torch.empty(pooled.size(0), w.size(0), dtype=torch.float32, device=pooled.device)
    extension().cls_logits(pooled, w, bias, out)
    _count()
    return out


TOKEN_HEAD_MAX_N = 64   # the widest per-token head the token_* kernels serve (QA: 2, NER: len(labels) + 1)


def _i32(t: torch.Tensor) -> torch.Tensor:
    return t.reshape(-1).to(torch.int32).contiguous()


def token_logits(seq: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, p_drop: float = 0.0, seed: int = 0,
                 stream: int = 0, row_map: Optional[torch.Tensor] = None,
                 mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Per-token head forward: fp32 logits [M, N] = dropout(``seq``) @ ``w``^T + ``bias`` for the bf16 [M, H] sequence
    output (H % 8 == 0) and a bf16 [N, H] weight, 1 <= N <= 64.  Dropout ``p_drop`` draws Philox ``(seed, stream)`` at
    element ``row * H + i`` (:func:`bert_pytorch_b200.utils.philox.keep_bits`).  With ``row_map`` (int32 [B * S] from
    :func:`pack_tokens`, ``seq`` the packed rows) and the batch's attention ``mask`` the result is unpacked to
    [B * S, N], ``bias`` at the masked positions."""
    out = torch.empty(seq.size(0) if seq.dim() == 2 else 0, w.size(0) if w.dim() == 2 else 0, dtype=torch.float32,
                      device=seq.device)
    extension().token_logits(seq, w, bias, p_drop, seed, stream, out)
    _count()
    if row_map is None:
        return out
    full = torch.empty(row_map.numel(), out.size(1), dtype=torch.float32, device=seq.device)
    extension().token_unpack(out, row_map, _i32(mask), bias, full)
    _count()
    return full


def token_ce_(logits: torch.Tensor, labels: torch.Tensor, grad_scale: float, loss_out: torch.Tensor,
              mask: Optional[torch.Tensor] = None, row_map: Optional[torch.Tensor] = None) -> None:
    """NER loss, in place: ``logits`` (fp32 [R, N]) <- d loss / d logits times ``grad_scale``, ``loss_out`` += the mean
    cross-entropy over the counted positions: ``mask == 1`` (every position without a mask) and ``0 <= label < N``
    (-100, -1 and labels >= N are ignored).  With ``row_map`` (from :func:`pack_tokens`) position p reads packed row
    ``row_map[p]``; rows that no counted position maps to get a zero gradient.  The count stays on the device; with no
    counted position the loss and every gradient are 0.  Deterministic mode: per-CTA loss sums added by ordered_sum."""
    det = deterministic()
    extension().token_ce(logits, _i32(labels), None if mask is None else _i32(mask),
                         None if row_map is None else _i32(row_map), grad_scale, loss_out, det)
    _count(3 if det else 2)


def span_ce_(logits: torch.Tensor, start_positions: torch.Tensor, end_positions: torch.Tensor, grad_scale: float,
             loss_out: torch.Tensor) -> None:
    """SQuAD loss, in place on the padded fp32 logits [B * S, 2] (start, end): per sequence a softmax over its S
    positions for each column; positions are clamped to [0, S] and S is ignored.  ``loss_out`` += (mean start CE + mean
    end CE) / 2, each mean over its own non-ignored sequences (0 without any); ``logits`` <- d loss / d logits times
    ``grad_scale``."""
    B = start_positions.numel()
    if B == 0 or logits.dim() != 2 or logits.size(0) % B != 0:
        raise ValueError(f"span_ce_: logits {tuple(logits.shape)} is not [B * S, 2] for B = {B}")
    det = deterministic()
    extension().span_ce(logits, _i32(start_positions), _i32(end_positions), logits.size(0) // B, grad_scale, loss_out,
                        det)
    _count(2 if det else 1)


def token_head_bwd(dlogits: torch.Tensor, seq: torch.Tensor, w: torch.Tensor, dw: torch.Tensor, db: torch.Tensor,
                   p_drop: float = 0.0, seed: int = 0, stream: int = 0) -> torch.Tensor:
    """Per-token head backward: returns d_seq bf16 [M, H] = (``dlogits`` @ ``w``) * keep / (1 - p), and accumulates
    ``dw`` (fp32 [N, H]) += dlogits^T @ dropout(seq) and ``db`` (fp32 [N]) += the column sums of dlogits -- per CTA over
    fixed 512-row partitions, then one atomic per CTA and element, or (deterministic mode) the partitions' partials
    added in order by ordered_sum.  The keep bits are :func:`token_logits`' for the same ``(seed, stream)``."""
    dseq = torch.empty_like(seq)
    det = deterministic()
    extension().token_head_bwd(dlogits, seq, w, dw, db, p_drop, seed, stream, dseq, det)
    _count(3 if det else 1)
    return dseq


def softmax_ce_(logits: torch.Tensor, targets: torch.Tensor, count: torch.Tensor, grad_scale: float,
                loss_out: torch.Tensor) -> None:
    """In place: logits <- d loss / d logits (scaled); loss_out += mean CE over valid targets."""
    det = deterministic()
    extension().softmax_ce(logits, targets, count, grad_scale, loss_out, det)
    _count(2 if det else 1)


def _eval_sums(acc: Optional[torch.Tensor], sums: torch.Tensor) -> None:
    if acc is not None:
        if acc.dtype != torch.float64 or acc.numel() != 3:
            raise ValueError("the metric accumulator must be an fp64 tensor of 3 elements")
        acc += sums


def mlm_eval(logits: torch.Tensor, targets: torch.Tensor, acc: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Masked-LM metrics of bf16 logits [R, V] (only read) against int32 ``targets`` [R] (< 0: ignored).  Returns the
    rows fp32 [R, 3] = {loss, correct, valid}: ``logsumexp(row) - row[t]`` (the forward half of :func:`softmax_ce_`,
    same arithmetic), ``argmax(row) == t`` with the lowest index winning a tie (``torch.argmax``'s rule), and 1; an
    ignored row is {0, 0, 0}.  ``acc`` (fp64 [3]) += their column sums, added in a fixed order without atomics in every
    mode: {loss sum, correct count, row count}."""
    R = logits.size(0)
    rows = torch.empty(R, 3, dtype=torch.float32, device=logits.device)
    sums = torch.zeros(3, dtype=torch.float32, device=logits.device)
    extension().mlm_eval(logits, targets, rows, sums)
    _count(2)
    _eval_sums(acc, sums)
    return rows


def nsp_eval(pooled: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, labels: torch.Tensor,
             acc: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Next-sentence metrics of the pooled bf16 [B, H] through the classifier ``w`` bf16 [2, H] + fp32 ``bias``
    against int64 ``labels`` [B] (< 0: ignored): rows fp32 [B, 3] = {cross-entropy, prediction == label, 1}, where the
    prediction is class 1 only when its logit is strictly larger.  ``acc`` (fp64 [3]) += their column sums, as
    :func:`mlm_eval`."""
    B = pooled.size(0)
    rows = torch.empty(B, 3, dtype=torch.float32, device=pooled.device)
    sums = torch.zeros(3, dtype=torch.float32, device=pooled.device)
    extension().nsp_eval(pooled, w, bias, labels, rows, sums)
    _count(2)
    _eval_sums(acc, sums)
    return rows


def _attn_shape(qkv: torch.Tensor, seqlens, cu_seqlens, S):
    """(B, S, rows, H) of the padded form (qkv [B, S, 3H], ``seqlens`` int32 [B]) or of the varlen form (qkv packed
    [T, 3H], ``cu_seqlens`` int32 [B + 1], ``S`` the padded length)."""
    if cu_seqlens is None:
        B, S, H3 = qkv.shape
        return B, S, B * S, H3 // 3
    if seqlens is not None or S is None:
        raise ValueError("the varlen form takes cu_seqlens and S, and no seqlens")
    return cu_seqlens.numel() - 1, int(S), qkv.size(0), qkv.size(-1) // 3


def attention_fwd(qkv: torch.Tensor, seqlens: Optional[torch.Tensor], heads: int, *, p_drop=0.0, seed=0, stream=0,
                  fp8=None, cu_seqlens: Optional[torch.Tensor] = None, S: Optional[int] = None):
    """Padded form: qkv [B, S, 3H], valid keys of sequence b = its first ``seqlens[b]`` (clamped to S; 0, an all-zero
    mask row, means all S keys, as under the model's additive mask) -> ctx [B, S, H].
    Varlen form (``cu_seqlens``, ``S``, ``seqlens=None``): qkv packed [T, 3H], sequence b = rows cu_seqlens[b] ..
    cu_seqlens[b + 1] -> ctx [T, H]; ``S`` is the padded length (at most 512, a multiple of 8), which sizes the grid
    and lse, and strides the dropout counter, so the keep decisions are the padded call's.  lse is [B, heads, S] in
    both forms.  ``fp8=(meta, site)`` (padded form only): the kernel also writes the fp8 copy of the context ->
    (ctx, lse, q)."""
    B, S, rows, H = _attn_shape(qkv, seqlens, cu_seqlens, S)
    ctx = torch.empty(*qkv.shape[:-1], H, dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty(B, heads, S, dtype=torch.float32, device=qkv.device)
    q, rec, e5 = _fp8_side(fp8, ctx)
    extension().attention_fwd(qkv, seqlens, ctx, lse, heads, 1.0 / math.sqrt(H // heads), p_drop, seed, stream, q, rec, e5,
                              cu_seqlens, S)
    _count()
    return (ctx, lse) if fp8 is None else (ctx, lse, q)


def attention_bwd(qkv, seqlens, ctx, dctx, lse, heads: int, *, p_drop=0.0, seed=0, stream=0, fp8=None,
                  cu_seqlens: Optional[torch.Tensor] = None, S: Optional[int] = None,
                  dbias: Optional[torch.Tensor] = None, _general: bool = False):
    """Both forms as :func:`attention_fwd`.  ``fp8=(meta, site)``: the kernels also write the fp8 copy of dqkv ->
    (dqkv, q).  ``dbias`` (fp32 [3H], the QKV bias gradient) += the column sums of dqkv (:func:`colsum_accumulate`).
    S <= 128 runs the one-pass kernel (no delta or dQ accumulation buffers); ``_general`` runs the multi-block path
    there too (for tests that compare the two)."""
    B, S, rows, H = _attn_shape(qkv, seqlens, cu_seqlens, S)
    dqkv = torch.empty_like(qkv)
    det = deterministic()
    onepass = S <= 128 and not _general
    delta = dq_acc = None
    if not onepass:
        delta = torch.empty(B, heads, S, dtype=torch.float32, device=qkv.device)
        # deterministic mode with more than one 128-key block: one dQ slice per key block, summed in key-block order
        slices = (S + 127) // 128 if det and S > 128 else 1
        dq_acc = torch.empty(slices, rows, H, dtype=torch.float32, device=qkv.device)
    q, rec, e5 = _fp8_side(fp8, dqkv)
    extension().attention_bwd(qkv, seqlens, ctx, dctx, lse, dqkv, delta, dq_acc, heads, 1.0 / math.sqrt(H // heads), p_drop,
                              seed, stream, q, rec, e5, cu_seqlens, S, det, _general)
    _count(1 if onepass else 2)
    if dbias is not None:
        colsum_accumulate(dqkv.view(-1, 3 * H), dbias)
    return dqkv if fp8 is None else (dqkv, q)


# ---------------------------------------------------------------------------
# multi-tensor ops over arbitrary tensor lists
# ---------------------------------------------------------------------------
CHUNK = 65536
_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_TABLE_CACHE: Dict[Tuple, Tuple[torch.Tensor, ...]] = {}


def _chunk_table(numels: Sequence[int], device: torch.device, offsets: Optional[Sequence[int]] = None):
    """chunk -> (tensor, start, len).  With ``offsets`` the starts are absolute arena positions."""
    ct, cs, cl = [], [], []
    for t, n in enumerate(numels):
        base = offsets[t] if offsets is not None else 0
        for s in range(0, n, CHUNK):
            ct.append(t); cs.append(base + s); cl.append(min(CHUNK, n - s))
    return (torch.tensor(ct, dtype=torch.int32, device=device), torch.tensor(cs, dtype=torch.int64, device=device),
            torch.tensor(cl, dtype=torch.int32, device=device))


def _list_tables(tensors: List[torch.Tensor]):
    key = tuple((t.data_ptr(), t.numel()) for t in tensors)
    hit = _TABLE_CACHE.get(key)
    if hit is None:
        dev = tensors[0].device
        ptrs = torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=dev)
        hit = (ptrs,) + _chunk_table([t.numel() for t in tensors], dev)
        if len(_TABLE_CACHE) > 64:
            _TABLE_CACHE.clear()
        _TABLE_CACHE[key] = hit
    return hit


def multi_tensor_l2norm(tensors: List[torch.Tensor], per_tensor: bool = False):
    dev = tensors[0].device
    total = torch.zeros(1, dtype=torch.float32, device=dev)
    per = torch.zeros(len(tensors), dtype=torch.float32, device=dev) if per_tensor else None
    det = deterministic()
    by_dtype: Dict[torch.dtype, List[int]] = {}
    for i, t in enumerate(tensors):
        if not t.is_contiguous():
            raise ValueError("multi_tensor_l2norm needs contiguous tensors")
        by_dtype.setdefault(t.dtype, []).append(i)
    for dt, idxs in by_dtype.items():
        group = [tensors[i] for i in idxs]
        ptrs, ct, cs, cl = _list_tables(group)
        sub = torch.zeros(len(group), dtype=torch.float32, device=dev) if per_tensor else None
        extension().mt_l2norm(_DT[dt], ptrs, ct, cs, cl, sub, total, det)
        _count(1 + (per_tensor + 1 if det else 0))
        if per_tensor:
            per[torch.tensor(idxs, device=dev)] = sub
    return total.sqrt().squeeze(0), (per.sqrt() if per_tensor else torch.zeros(0, device=dev))


def multi_tensor_scale(src: List[torch.Tensor], dst: List[torch.Tensor], scale) -> torch.Tensor:
    dev = src[0].device
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    groups: Dict[Tuple[torch.dtype, torch.dtype], List[int]] = {}
    for i, (s, d) in enumerate(zip(src, dst)):
        groups.setdefault((s.dtype, d.dtype), []).append(i)
    sd = scale.to(device=dev, dtype=torch.float32).reshape(1) if torch.is_tensor(scale) else None
    sh = 1.0 if torch.is_tensor(scale) else float(scale)
    for (sdt, ddt), idxs in groups.items():
        ins, outs = [src[i] for i in idxs], [dst[i] for i in idxs]
        ip, ct, cs, cl = _list_tables(ins)
        op = _list_tables(outs)[0]
        extension().mt_scale(_DT[sdt], _DT[ddt], ip, op, ct, cs, cl, sd, sh, overflow)
        _count()
    return overflow.squeeze(0)


# ---------------------------------------------------------------------------
# arena optimizers
# ---------------------------------------------------------------------------

def _arena_tables(arena):
    t = getattr(arena, "_opt_tables", None)
    if t is None:
        dev = arena.device
        ct, cs, cl = _chunk_table([s.numel for s in arena.slots], dev, [s.offset for s in arena.slots])
        t = dict(ct=ct, cs=cs, cl=cl,
                 decay=torch.tensor([1 if s.decay else 0 for s in arena.slots], dtype=torch.int32, device=dev),
                 stats=torch.zeros(1, dtype=torch.float32, device=dev),
                 norms=torch.zeros(2 * len(arena.slots), dtype=torch.float32, device=dev))
        arena._opt_tables = t
    return t


def flat_unscale_(flat_grad: torch.Tensor, inv_scale: torch.Tensor, found_inf: torch.Tensor) -> None:
    extension().flat_unscale(flat_grad, inv_scale.reshape(1), found_inf.reshape(1))
    _count()


def _uniform(optimizer, key):
    vals = {repr(g[key]) for g in optimizer.param_groups}
    if len(vals) != 1:
        raise NotImplementedError(f"fused arena optimizer needs the same '{key}' in every param group")
    return optimizer.param_groups[0][key]


def _uniform_decay(optimizer) -> float:
    """The weight decay of the decaying slots.  The fused kernels take one value and a per-slot decay flag (set by
    ``ParamArena.bind_optimizer`` from ``weight_decay != 0``), so the groups may mix 0 with one non-zero value only."""
    wds = {float(g["weight_decay"]) for g in optimizer.param_groups} - {0.0}
    if len(wds) > 1:
        raise NotImplementedError(f"fused arena optimizer needs one non-zero 'weight_decay' across the param groups, "
                                  f"got {sorted(wds)}")
    return wds.pop() if wds else 0.0


def arena_lamb_step(arena, optimizer, inv_scale=None, found_inf=None) -> None:
    """One LAMB step over the arena (3 launches + 2 memsets).  Weight decay is per slot (decay flag x
    the single non-zero group value), every other hyper-parameter must agree across groups -- which is
    how every runner builds its groups (run_pretraining.py:279-296)."""
    T = _arena_tables(arena)
    lr = _uniform(optimizer, "lr")
    b1, b2 = _uniform(optimizer, "betas")
    eps = _uniform(optimizer, "eps")
    wd = _uniform_decay(optimizer)
    step = int(optimizer.param_groups[0].get("step", 0)) + 1
    ext = extension()
    inv = inv_scale.reshape(1) if inv_scale is not None else None
    fi = found_inf.reshape(1) if found_inf is not None else None
    det = deterministic()
    ext.flat_sumsq(arena.flat_grad, inv, T["stats"], fi, det)
    ext.arena_lamb(arena.flat_grad, arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow, T["ct"],
                   T["cs"], T["cl"], T["decay"], T["stats"], T["norms"], inv, fi, float(lr), float(b1), float(b2),
                   float(eps), float(wd), step, bool(_uniform(optimizer, "bias_correction")),
                   bool(_uniform(optimizer, "grad_averaging")), float(_uniform(optimizer, "max_grad_norm") or 0.0),
                   bool(optimizer.adam_w_mode), bool(optimizer.use_nvlamb), det)
    _count(5 if det else 3)
    # apex semantics: the step counter only advances when the update was applied.  Keeping that exact
    # would need a host sync on found_inf; with a scaler we advance optimistically only when no scaler
    # is in play, otherwise we read the flag (fp16 path only -- bf16 never has a scaler).
    if fi is None or float(fi) == 0.0:
        for g in optimizer.param_groups:
            g["step"] = step
    optimizer.last_grad_norm = T["stats"].sqrt()


def arena_adam_step(arena, optimizer, inv_scale=None, found_inf=None) -> None:
    T = _arena_tables(arena)
    lr = _uniform(optimizer, "lr")
    b1, b2 = _uniform(optimizer, "betas")
    eps = _uniform(optimizer, "eps")
    wd = _uniform_decay(optimizer)
    step = int(optimizer.param_groups[0].get("step", 0)) + 1
    inv = inv_scale.reshape(1) if inv_scale is not None else None
    fi = found_inf.reshape(1) if found_inf is not None else None
    if inv is not None and fi is not None:
        # the Adam kernel only reads found_inf (LAMB's norm pass sets it): unscale and check the gradients first
        extension().flat_unscale(arena.flat_grad, inv, fi)
        _count()
        inv = None
    extension().arena_adam(arena.flat_grad, arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow,
                           T["ct"], T["cs"], T["cl"], T["decay"], inv, fi, float(lr), float(b1), float(b2), float(eps),
                           float(wd), step, bool(_uniform(optimizer, "bias_correction")), bool(optimizer.adam_w_mode))
    _count()
    if fi is None or float(fi) == 0.0:
        for g in optimizer.param_groups:
            g["step"] = step
