"""Fused sm_90a execution engine for the BERT encoder and the pre-training heads.

The ``nn.Module`` tree in :mod:`.modeling` only *holds* the parameters (as views into the
:class:`~.arena.ParamArena`); on an H100 the math runs here as an explicit forward/backward
*kernel program* -- no autograd graph, no per-op Python dispatch beyond one launch per fused block:

  embeddings   gather x3 + add + LayerNorm + dropout                       1 kernel   (K1-K3)
  per layer    QKV GEMM [M,H]x[H,3H] + bias                                 wgmma    (K5, K6 gone)
               flash attention (scale, key-padding, softmax, dropout, PV)   wgmma    (K7-K12)
               out-proj GEMM + bias + dropout + residual                    wgmma    (K13-K14)
               LayerNorm                                                     1 kernel   (K15)
               FFN-1 GEMM + bias + GELU (and GELU' for the backward) epilogue  wgmma    (K16)
               FFN-2 GEMM + bias + dropout + residual                        wgmma    (K17-K18)
               LayerNorm                                                     1 kernel
  MLM head     compact masked positions -> gather -> transform GEMM+GELU -> LN -> decoder GEMM + bias
               -> softmax-CE fwd+bwd in place (only max_pred rows/sequence, K21-K24; fixes Q15)
  backward     the mirror image: LN-bwd kernels emit the residual gradient *and* the dropout-masked
               gradient plus all dgamma/dbeta/dbias column sums; dgrad GEMMs fuse the residual-gradient
               add or the multiplication by GELU' (+ the FFN-1 bias gradient); wgrad GEMMs (both operands MN-major,
               split-K) accumulate in fp32 straight into the gradient arena -- or, on the last micro-step
               with the peer-memory backend, straight into the OWNER rank's arena over NVLink.

Dropout masks are a counter-based function of (seed, stream id, element index) so backward regenerates
them (nothing stored, and recompute is deterministic -- SURVEY.md K27).
Activations are saved rather than recomputed by default: an H100 has 80 GB (phase-1 micro-batch 96x128 needs
~10 GB); ``--checkpoint_activations`` replays ceil(sqrt(L))-layer segments instead.
Options: fp8 GEMM operands (``enable_fp8`` / ``B200_FP8=1`` / ``--fp8``), whole-micro-step CUDA-graph replay
(``FusedPretrainer``, on by default, ``B200_GRAPH=0`` disables), K-FAC taps.

Unpadded mode (``BertModel.unpad``, fine-tuning and inference through :meth:`FusedEncoderEngine.encode`): the
unmasked tokens of the [B, S] batch are packed into T rows (:func:`pack_rows`) and every kernel runs on those rows
only -- embeddings with explicit position ids, GEMMs / LayerNorms / dropout with M = T, variable-length attention
over ``cu_seqlens``.  The output is scattered back into a zeroed [B*S, H] tensor.
Pre-training (``FusedPretrainer`` with ``BertModel.unpad``, ``--unpad``) packs on the device instead (:func:`pack_device`,
no host sync) into a static row count T_cap from :func:`token_bucket`, so that each bucket replays its own CUDA graph;
the rows past the real tokens are [PAD] tokens in dummy sequences of their own, finite and with zero gradient.
"""
from __future__ import annotations

import gc
import math
import os
import warnings
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from .. import ops
from ..ops import api as K
from .arena import ParamArena

# dropout stream ids: stream = layer * 8 + site
SITE_EMB, SITE_ATTN_PROB, SITE_ATTN_OUT, SITE_FFN_OUT = 0, 1, 2, 3
_EMB_LAYER = 1023
# dropout on the pooled row of the sequence classifier (FusedClassifier): site 4 of the embedding's layer slot.  No
# encoder layer uses site 4 and the embedding uses site 0, so the stream collides with none of theirs at any depth.
SITE_CLS = 4
# dropout on the sequence output under the per-token heads (FusedTokenClassifier): site 5 of the same slot, used by no
# encoder layer, the embedding or the sequence classifier
SITE_TOKEN = 5


def _stream(layer: int, site: int) -> int:
    return layer * 8 + site


CLS_STREAM = _stream(_EMB_LAYER, SITE_CLS)
TOKEN_STREAM = _stream(_EMB_LAYER, SITE_TOKEN)


def _as_tuple(x):
    return x if isinstance(x, tuple) else (x,)


@dataclass
class _LayerSaved:
    x: torch.Tensor = None
    qkv: torch.Tensor = None
    ctx: torch.Tensor = None
    lse: torch.Tensor = None
    pre1: torch.Tensor = None
    mean1: torch.Tensor = None
    rstd1: torch.Tensor = None
    x1: torch.Tensor = None
    y1: torch.Tensor = None
    act: torch.Tensor = None
    pre2: torch.Tensor = None
    mask1: torch.Tensor = None      # dropout keep bits of the two hidden-dropout sites (uint8 [M, H / 8]), written by the
    mask2: torch.Tensor = None      # GEMM epilogues, read back by the LayerNorm backward kernels
    mean2: torch.Tensor = None
    rstd2: torch.Tensor = None
    x_op: torch.Tensor = None      # operands of the four weight-gradient GEMMs (bf16 tensors or their fp8 copies)
    ctx_op: torch.Tensor = None
    x1_op: torch.Tensor = None
    act_op: torch.Tensor = None


@dataclass
class Packing:
    """The unmasked tokens of a [B, S] batch packed back to back (one record per call, shared by every layer)."""
    rows: Optional[torch.Tensor]  # int32 [T]: index b * S + s of every unmasked token, in order (pack_rows only)
    cu_seqlens: torch.Tensor    # int32 [B + 1]: sequence b is packed rows cu_seqlens[b] .. cu_seqlens[b + 1]
    pos_ids: torch.Tensor       # int32 [T]: position s of every packed row
    T: int
    S: int
    # device packing of pre-training (pack_device): T is the bucket capacity T_cap, cu_seqlens has B + D + 1 entries
    # (D dummy sequences over the pad tail), and the token ids / segments come packed already
    ids: Optional[torch.Tensor] = None       # int32 [T]
    seg: Optional[torch.Tensor] = None       # int32 [T]
    cls_rows: Optional[torch.Tensor] = None  # int32 [B]: first packed row of every sequence
    row_map: Optional[torch.Tensor] = None   # int32 [B * S]: packed row of token (b, s), -1 where masked


def pack_rows(attention_mask: torch.Tensor) -> Packing:
    """Packing of any 0/1 ``attention_mask`` [B, S] (holes included).  ``torch.nonzero`` costs one host sync."""
    B, S = attention_mask.shape
    keep = attention_mask != 0
    rows = torch.nonzero(keep.reshape(-1)).squeeze(1)
    cu = torch.zeros(B + 1, dtype=torch.int32, device=attention_mask.device)
    cu[1:] = torch.cumsum(keep.sum(dim=1, dtype=torch.int32), 0, dtype=torch.int32)
    return Packing(rows=rows.to(torch.int32), cu_seqlens=cu, pos_ids=(rows % S).to(torch.int32),
                   T=rows.numel(), S=S)


# ---- unpadded pre-training: static token buckets -------------------------------------------------------------------
MAX_TOKEN_BUCKETS = 16


def token_bucket(T: int, B: int, S: int):
    """(T_cap, D) of a micro-batch with T packed tokens: the row capacity of its CUDA graph and the number of dummy
    sequences that cover the pad tail ``T_cap - T``.  The bucket step is ``g = 128 * ceil(B*S / (128 * 16))`` rows: at
    most 16 buckets (16 graphs per batch shape), each a whole number of 128-row GEMM tiles, and a pad tail below one
    step (< 1/16 of the batch).  ``T_cap = min(B*S, ceil(T / g) * g)``; ``D = ceil(g / S)`` dummies of at most S rows
    always cover the tail, since it is shorter than g."""
    M = B * S
    if not 1 <= T <= M:
        raise ValueError(f"token count {T} outside [1, {M}] for a [{B}, {S}] batch")
    g = 128 * -(-M // (128 * MAX_TOKEN_BUCKETS))
    return min(M, -(-T // g) * g), -(-g // S)


def packed_tokens(mask: torch.Tensor) -> int:
    """Number of packed rows of a [B, S] attention mask: its unmasked tokens, where a row without any counts S (the
    padded attention computes such a row with every key valid).  One host read on a device tensor; none on the pinned
    host batch."""
    S = mask.size(-1)
    n = (mask.reshape(-1, S) != 0).sum(dim=1)
    return int(torch.where(n > 0, n, torch.full_like(n, S)).sum())


def pack_device(input_mask, input_ids, segment_ids, T_cap: int, D: int) -> Packing:
    """:func:`~bert_pytorch_b200.ops.api.pack_tokens` as a :class:`Packing` (no host sync: capturable)."""
    ids, seg, pos, cu, cls, row_map = K.pack_tokens(input_mask, input_ids, segment_ids, T_cap, D)
    return Packing(rows=None, cu_seqlens=cu, pos_ids=pos, T=T_cap, S=input_mask.size(1), ids=ids, seg=seg,
                   cls_rows=cls, row_map=row_map)


@dataclass
class _Saved:
    B: int = 0
    S: int = 0
    pk: Optional[Packing] = None
    seed: int = 0
    p_hidden: float = 0.0
    p_attn: float = 0.0
    ids: torch.Tensor = None
    seg: torch.Tensor = None
    seqlens: torch.Tensor = None
    emb_sum: torch.Tensor = None
    emb_mean: torch.Tensor = None
    emb_rstd: torch.Tensor = None
    layers: List[_LayerSaved] = field(default_factory=list)
    boundaries: Dict[int, torch.Tensor] = field(default_factory=dict)   # segment inputs under --checkpoint_activations
    seg_len: int = 0


class FusedEncoderEngine:
    """Bound to one ``BertModel``; reads weights from the arena's bf16 shadow and LN parameters from the
    fp32 master copy, writes gradients into the fp32 gradient arena."""

    def __init__(self, bert):
        self.bert = bert
        cfg = bert.config
        self.H, self.heads, self.L = cfg.hidden_size, cfg.num_attention_heads, cfg.num_hidden_layers
        self.I = cfg.intermediate_size
        if cfg.hidden_act != "gelu":
            raise NotImplementedError("the fused engine implements the erf-GELU FFN only")
        if self.H % 64 != 0 or (self.H // self.heads) != 64:
            # the attention kernel is specialised for head_dim 64 (every shipped config)
            raise NotImplementedError("fused attention needs head_dim == 64")
        ref = getattr(bert, "_arena_ref", None)
        arena = ref() if ref is not None else None
        if arena is None:
            arena = ParamArena(bert)
            self._own_arena = arena          # keep alive
        self.arena = arena
        self.prefix = self._find_prefix()
        self.p_hidden = float(cfg.hidden_dropout_prob)
        self.p_attn = float(cfg.attention_probs_dropout_prob)
        self.has_type = bert.embeddings.has_token_type
        self._seed_base = int(torch.initial_seed()) & 0x7FFFFFFF
        self._calls = 0
        self._hook = torch.zeros(1, device=arena.device, requires_grad=True)
        # fp8 GEMM operands (B200_FP8=1 or enable_fp8()): activations / weights as e4m3, gradients as e5m2,
        # per-tensor delayed scaling; LN / GELU / attention / residual stream / master weights unchanged
        self.fp8 = False
        self.meta = None
        if os.environ.get("B200_FP8", "0") == "1":
            self.enable_fp8()
        # weight-gradient GEMMs on a second (lower priority) stream: they are off the critical path of the
        # backward pass, so the bandwidth-bound kernels of the chain (LN / dGELU / attention backward) can share
        # the machine with them (+2.5 % on the phase-1 step at 1 and 2 GPUs).  B200_WGRAD_STREAM=0 / ``wgrad_side =
        # False`` keeps everything on one stream.
        self.wgrad_side = os.environ.get("B200_WGRAD_STREAM", "1") != "0"
        self._wstream = None
        self._wkeep: list = []

    # -- parameter lookup --------------------------------------------------------------------
    def _find_prefix(self) -> str:
        """Name prefix of this BertModel's parameters inside the arena ('' or 'bert.')."""
        for cand in ("bert.", ""):
            if (cand + "embeddings.word_embeddings.weight") in self.arena.by_name:
                return cand
        raise RuntimeError("the arena does not contain this encoder's parameters")

    def w(self, name: str) -> torch.Tensor:      # bf16 shadow weight
        return self.arena.shadow(self.prefix + name)

    def p(self, name: str) -> torch.Tensor:      # fp32 master parameter
        return self.arena.view(self.prefix + name)

    def g(self, name: str) -> torch.Tensor:      # fp32 gradient slot
        return self.arena.grad(self.prefix + name)

    def _qkv(self, l: int, flat: torch.Tensor, kind: str) -> torch.Tensor:
        base = f"{self.prefix}encoder.layer.{l}.attention.self."
        if kind == "weight":
            return self.arena.span(base + "query.weight", base + "value.weight", flat, (3 * self.H, self.H))
        return self.arena.span(base + "query.bias", base + "value.bias", flat, (3 * self.H,))

    # -- fp8 ------------------------------------------------------------------------------------------
    _FP8_ACT = ("x", "ctx", "x1", "act")
    _FP8_W = ("wqkv", "wo", "w1", "w2")
    _FP8_GRAD = ("d_y2", "d_y1", "d_yo", "d_qkv")

    def enable_fp8(self, margin: float = 1.0) -> None:
        sites, e5 = [], []
        for l in range(self.L):
            for n in self._FP8_ACT + self._FP8_W:
                sites.append(f"{l}.{n}"); e5.append(False)
            for n in self._FP8_GRAD:
                sites.append(f"{l}.{n}"); e5.append(True)
        self.meta = K.Fp8Meta(sites, e5, self.arena.device, margin=margin)
        self.fp8 = True
        self._fp8_calibrated = False
        self._w8: Dict[str, tuple] = {}

    def _weight8(self, l: int, which: str, w_bf16: torch.Tensor) -> torch.Tensor:
        """e4m3 copy of a weight, re-quantised (current scaling) only when the arena's weights changed --
        once per optimizer step, i.e. amortised over the accumulation steps."""
        key = f"{l}.{which}"
        ent = self._w8.get(key)
        if ent is None or ent[1] != self.arena.version:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("fp8 weight copies are stale inside a CUDA-graph capture: call prepare_step() first")
            q = self.meta.quantize(w_bf16.contiguous(), key, out=ent[0] if ent is not None else None, calibrate=True)
            ent = (q, self.arena.version)          # same storage every time: captured graphs keep reading it
            self._w8[key] = ent
        return ent[0]

    def gemm_reduced_parameters(self) -> List[str]:
        """Arena names of the parameters whose whole gradient comes out of fp32-accumulate GEMMs of this engine
        (candidates for the GEMM -> reduce-scatter fusion of the peer-memory backend)."""
        out = []
        for l in range(self.L):
            pre = f"{self.prefix}encoder.layer.{l}."
            out += [pre + "attention.self.query.weight", pre + "attention.self.key.weight",
                    pre + "attention.self.value.weight", pre + "attention.output.dense.weight",
                    pre + "intermediate.dense_act.weight", pre + "output.dense.weight"]
        return out

    def prepare_step(self) -> None:
        """Host-side work that must not happen inside a captured graph: refresh the fp8 weight copies when the
        optimizer has changed the weights (once per optimizer step)."""
        if not self.fp8:
            return
        A = self.arena
        for l in range(self.L):
            pre = f"encoder.layer.{l}."
            self._weight8(l, "wqkv", self._qkv(l, A.flat_shadow, "weight"))
            self._weight8(l, "wo", self.w(pre + "attention.output.dense.weight"))
            self._weight8(l, "w1", self.w(pre + "intermediate.dense_act.weight"))
            self._weight8(l, "w2", self.w(pre + "output.dense.weight"))

    def _side(self, site: str):
        """(meta, site) for a producer kernel's fused fp8 copy -- only once the scales are calibrated (delayed
        scaling needs last step's amax; the first micro-step quantises in a separate pass)."""
        return (self.meta, site) if (self.fp8 and self._fp8_calibrated) else None

    def _lin(self, l: int, act_site: str, w_site: str, x: torch.Tensor, w: torch.Tensor, xq=None, **kw):
        """y = x @ w^T through the bf16 or the fp8 operand path; returns (y, saved operand for wgrad).
        ``xq``: fp8 copy of x already emitted by the kernel that produced x."""
        if not self.fp8:
            return K.gemm(x, w, **kw), x
        qx = xq if xq is not None else self.meta.quantize(x, f"{l}.{act_site}", calibrate=not self._fp8_calibrated)
        qw = self._weight8(l, w_site, w)
        y = K.gemm(qx, qw, scale_a=self.meta.inv_scale(f"{l}.{act_site}"), scale_b=self.meta.inv_scale(f"{l}.{w_site}"), **kw)
        return y, qx

    def _wgrad(self, dy: torch.Tensor, x: torch.Tensor, wgrad: torch.Tensor, **kw) -> None:
        """wgrad += dy^T @ x, on the side stream when enabled: fork after the producer of ``dy`` (the caller launches
        the dgrad GEMM afterwards).  The operands stay referenced until the main stream has waited for the side
        stream again (two layers later, or the join at the end of :meth:`backward`), so the caching allocator cannot
        hand their memory to a main-stream kernel while the side stream still reads it."""
        if not (self.wgrad_side and dy.is_cuda):
            K.wgrad_accumulate(dy, x, wgrad, push=True, **kw)
            return
        if self._wstream is None:
            self._wstream = torch.cuda.Stream(device=dy.device)
        self._wstream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._wstream):
            K.wgrad_accumulate(dy, x, wgrad, push=True, **kw)
        if not self._wkeep or self._wkeep[-1][0] is not None:
            self._wkeep.append([None, []])
        self._wkeep[-1][1].append((dy, x))

    def _wgrad_layer_done(self) -> None:
        """End of one layer's backward: mark the layer's group of side-stream GEMMs with an event and retire the
        groups that are two layers old (their GEMMs finished long ago: the wait is free, the operands can go)."""
        if not self._wkeep or self._wkeep[-1][0] is not None:
            return
        ev = torch.cuda.Event()
        ev.record(self._wstream)
        self._wkeep[-1][0] = ev
        while len(self._wkeep) > 2:
            torch.cuda.current_stream().wait_event(self._wkeep.pop(0)[0])

    def _join_wgrads(self) -> None:
        if self._wkeep:
            torch.cuda.current_stream().wait_stream(self._wstream)
            self._wkeep.clear()

    def _lin_bwd(self, l: int, g_site: str, act_site: str, w_site: str, dy: torch.Tensor, x_saved: torch.Tensor,
                 w: torch.Tensor, wgrad: torch.Tensor, dyq=None, **kw) -> torch.Tensor:
        """dx = dy @ w (with the epilogue in ``kw``) and wgrad += dy^T @ x."""
        if not self.fp8:
            if self.wgrad_side:
                self._wgrad(dy, x_saved, wgrad)
                return K.gemm(dy, w, layout=K.NN, **kw)
            dx = K.gemm(dy, w, layout=K.NN, **kw)
            K.wgrad_accumulate(dy, x_saved, wgrad, push=True)
            return dx
        m = self.meta
        qdy = dyq if dyq is not None else m.quantize(dy, f"{l}.{g_site}", calibrate=not self._fp8_calibrated)
        sg, sw, sx = m.inv_scale(f"{l}.{g_site}"), m.inv_scale(f"{l}.{w_site}"), m.inv_scale(f"{l}.{act_site}")
        if self.wgrad_side:
            self._wgrad(qdy, x_saved, wgrad, scale_a=sg, scale_b=sx, a_e5m2=True)
            return K.gemm(qdy, self._weight8(l, w_site, w), layout=K.NN, scale_a=sg, scale_b=sw, a_e5m2=True, **kw)
        dx = K.gemm(qdy, self._weight8(l, w_site, w), layout=K.NN, scale_a=sg, scale_b=sw, a_e5m2=True, **kw)
        K.wgrad_accumulate(qdy, x_saved, wgrad, push=True, scale_a=sg, scale_b=sx, a_e5m2=True)
        return dx

    def next_seed(self) -> int:
        self._calls += 1
        return (self._seed_base * 1000003 + self._calls) & 0x7FFFFFFFFFFF

    # -- forward --------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, input_ids, token_type_ids, attention_mask, training: bool, seed: Optional[int] = None,
                dropout: Optional[bool] = None, pack: Optional[Packing] = None):
        """Returns (sequence_output [B*S, H] bf16, saved-or-None).  ``training`` saves activations for
        ``backward``; ``dropout`` (default: same as ``training``) applies the dropout sites.  With ``pack``
        (:func:`pack_rows` of the mask, at least one token) only the packed rows are computed: the sequence output is
        [T, H] and the dropout elements are counted by packed row."""
        B, S = input_ids.shape
        H, A = self.H, self.arena
        dropout = training if dropout is None else dropout
        ph = self.p_hidden if dropout else 0.0
        pa = self.p_attn if dropout else 0.0
        seed = self.next_seed() if seed is None else seed
        ids = input_ids.reshape(-1).to(torch.int32).contiguous()
        seg = None
        if self.has_type:
            seg = (token_type_ids if token_type_ids is not None else torch.zeros_like(input_ids)
                   ).reshape(-1).to(torch.int32).contiguous()
        if pack is not None and pack.ids is not None:   # packed on the device already (pack_device)
            ids, seg, seqlens = pack.ids, pack.seg if seg is not None else None, None
        elif pack is not None:
            ids = ids.index_select(0, pack.rows)
            seg = seg.index_select(0, pack.rows) if seg is not None else None
            seqlens = None
        else:
            seqlens = attention_mask.to(torch.int32).sum(dim=1, dtype=torch.int32).contiguous()
        sv = _Saved(B=B, S=S, pk=pack, seed=seed, p_hidden=ph, p_attn=pa, ids=ids, seg=seg, seqlens=seqlens) if training else None

        x, e, mean, rstd = K.embedding_fwd(
            ids, seg, self.w("embeddings.word_embeddings.weight"), self.w("embeddings.position_embeddings.weight"),
            self.w("embeddings.token_type_embeddings.weight") if self.has_type else None,
            self.p("embeddings.LayerNorm.weight"), self.p("embeddings.LayerNorm.bias"), S,
            p_drop=ph, seed=seed, stream=_stream(_EMB_LAYER, SITE_EMB), pos_ids=pack.pos_ids if pack is not None else None)
        if training:
            sv.emb_sum, sv.emb_mean, sv.emb_rstd = e, mean, rstd

        ckpt = training and bool(getattr(self.bert.encoder, "_checkpoint_activations", False))
        seg_len = int(math.ceil(math.sqrt(self.L))) if ckpt else 0
        for l in range(self.L):
            if ckpt and l % seg_len == 0:
                sv.boundaries[l] = x             # --checkpoint_activations: keep segment inputs only (K27)
            x, ls, xq = self._layer_forward(l, x, seqlens, B, S, ph, pa, seed, save=training and not ckpt,
                                            xq=None if (l == 0 or (ckpt and l % seg_len == 0)) else xq, pk=pack)
            if ls is not None:
                sv.layers.append(ls)
        if ckpt:
            sv.seg_len = seg_len
        return x, sv

    def _layer_forward(self, l: int, x, seqlens, B: int, S: int, ph: float, pa: float, seed: int, save: bool, xq=None,
                       pk: Optional[Packing] = None):
        """One post-LN transformer layer (reference: src/modeling.py:482-499) as 9 kernel launches.  ``x``: [B*S, H],
        or [T, H] packed rows with ``pk``."""
        A, H, M = self.arena, self.H, x.size(0)
        pre = f"encoder.layer.{l}."
        ls = _LayerSaved() if save else None
        qkv, x_op = self._lin(l, "x", "wqkv", x, self._qkv(l, A.flat_shadow, "weight"), xq=xq, epi=K.EPI_BIAS,
                              bias=self._qkv(l, A.flat_shadow, "bias"))
        if pk is not None:
            ctx, lse = K.attention_fwd(qkv, None, self.heads, p_drop=pa, seed=seed, stream=_stream(l, SITE_ATTN_PROB),
                                       cu_seqlens=pk.cu_seqlens, S=S)
            ctx_q = None
        else:
            ctx, lse, *q = K.attention_fwd(qkv.view(B, S, 3 * H), seqlens, self.heads, p_drop=pa, seed=seed,
                                           stream=_stream(l, SITE_ATTN_PROB), fp8=self._side(f"{l}.ctx"))
            ctx = ctx.view(M, H)
            ctx_q = q[0].view(M, H) if q else None
        # keep bits of the hidden dropout leave the GEMM epilogue (1 bit per element) so that the LayerNorm backward does
        # not have to run Philox again -- bf16 path only
        keep_bits = save and ph > 0 and not self.fp8 and H % 128 == 0
        # ... and are GENERATED by their own kernel (K.dropout_mask: every warp of the machine on Philox) rather than by
        # the GEMM's epilogue warps while the tensor cores idle
        mask1 = K.dropout_mask(M, H, ph, seed, _stream(l, SITE_ATTN_OUT), x.device) if keep_bits else None
        mask2 = K.dropout_mask(M, H, ph, seed, _stream(l, SITE_FFN_OUT), x.device) if keep_bits else None
        pre1, ctx_op = self._lin(l, "ctx", "wo", ctx, self.w(pre + "attention.output.dense.weight"), xq=ctx_q,
                                 epi=K.EPI_BIAS_DROP_RES, bias=self.w(pre + "attention.output.dense.bias"), res=x,
                                 p_drop=ph, seed=seed, stream=_stream(l, SITE_ATTN_OUT),
                                 **({"mask_in": mask1} if keep_bits else {}))
        # producers emit the fp8 copy of their output for the next GEMM (no separate quantise pass)
        x1, mean1, rstd1, *q = K.layer_norm_fwd(pre1, self.p(pre + "attention.output.LayerNorm.weight"),
                                                self.p(pre + "attention.output.LayerNorm.bias"), save_stats=save,
                                                fp8=self._side(f"{l}.x1"))
        if not self.fp8:
            # K16: GELU *and* GELU' leave the FFN-1 GEMM through its epilogue (y1 holds gelu'(x), which is all the
            # backward pass needs: the FFN-2 dgrad epilogue multiplies by it) -- no activation pass over HBM at all
            y1 = torch.empty(M, self.I, dtype=torch.bfloat16, device=x1.device)
            act, x1_op = self._lin(l, "x1", "w1", x1, self.w(pre + "intermediate.dense_act.weight"),
                                   epi=K.EPI_BIAS_GELU_DG, bias=self.w(pre + "intermediate.dense_act.bias"), aux_out=y1)
            q = []
        else:
            # fp8 operands: GELU stays a bandwidth kernel that also emits the e4m3 copy of the activation
            y1, x1_op = self._lin(l, "x1", "w1", x1, self.w(pre + "intermediate.dense_act.weight"), xq=q[0] if q else None,
                                  epi=K.EPI_BIAS, bias=self.w(pre + "intermediate.dense_act.bias"))
            side = self._side(f"{l}.act")
            act, *q = K.gelu_fwd(y1, fp8=side) if side else (K.gelu_fwd(y1),)
        pre2, act_op = self._lin(l, "act", "w2", act, self.w(pre + "output.dense.weight"), xq=q[0] if q else None,
                                 epi=K.EPI_BIAS_DROP_RES, bias=self.w(pre + "output.dense.bias"), res=x1, p_drop=ph,
                                 seed=seed, stream=_stream(l, SITE_FFN_OUT), **({"mask_in": mask2} if keep_bits else {}))
        x2, mean2, rstd2, *q = K.layer_norm_fwd(pre2, self.p(pre + "output.LayerNorm.weight"),
                                                self.p(pre + "output.LayerNorm.bias"), save_stats=save,
                                                fp8=self._side(f"{l + 1}.x") if l + 1 < self.L else None)
        x2q = q[0] if q else None
        if save:
            ls.x, ls.qkv, ls.ctx, ls.lse = x, qkv, ctx, lse
            ls.pre1, ls.mean1, ls.rstd1, ls.x1 = pre1, mean1, rstd1, x1
            ls.y1, ls.act, ls.pre2, ls.mean2, ls.rstd2 = y1, act, pre2, mean2, rstd2
            ls.mask1, ls.mask2 = mask1, mask2
            ls.x_op, ls.ctx_op, ls.x1_op, ls.act_op = x_op, ctx_op, x1_op, act_op   # wgrad operands (fp8 or bf16)
        return x2, ls, x2q

    # -- backward -------------------------------------------------------------------------------
    @torch.no_grad()
    def backward(self, sv: _Saved, d_out: torch.Tensor) -> None:
        """``d_out``: [B*S, H] bf16 gradient of the sequence output ([T, H] packed rows when the forward ran with a
        packing).  Accumulates every parameter gradient of the encoder into the arena."""
        A, H = self.arena, self.H
        ph, pa, seed = sv.p_hidden, sv.p_attn, sv.seed
        d = d_out
        kfac = getattr(self.bert, "_kfac", None)      # K-FAC taps: the saved activations double as its statistics
        if kfac is not None and not getattr(kfac, "capture", True):
            kfac = None                               # this micro-step does not feed the factors (KFAC.wants_data)
        if sv.seg_len:                                    # recompute each segment from its saved input, then walk it back
            for lo in reversed(range(0, self.L, sv.seg_len)):
                hi = min(self.L, lo + sv.seg_len)
                x, saved, xq = sv.boundaries.pop(lo), [], None
                for l in range(lo, hi):                   # same seed -> same Philox dropout masks as the first pass
                    x, ls, xq = self._layer_forward(l, x, sv.seqlens, sv.B, sv.S, ph, pa, seed, save=True, xq=xq, pk=sv.pk)
                    saved.append(ls)
                for l in reversed(range(lo, hi)):
                    d = self._layer_backward(l, saved[l - lo], d, sv, kfac)
                del saved
        else:
            for l in reversed(range(self.L)):
                d = self._layer_backward(l, sv.layers[l], d, sv, kfac)
                sv.layers[l] = None                       # activations of finished layers go back to the allocator
        # ---- embeddings: output dropout -> LN -> scatter into the three tables
        d_e, _ = K.layer_norm_bwd(
            d, sv.emb_sum, sv.emb_mean, sv.emb_rstd, self.p("embeddings.LayerNorm.weight"),
            dgamma=self.g("embeddings.LayerNorm.weight"), dbeta=self.g("embeddings.LayerNorm.bias"),
            p_drop=ph, seed=seed, in_stream=_stream(_EMB_LAYER, SITE_EMB) if ph > 0 else K.NO_STREAM)
        K.embedding_bwd_scatter(d_e, sv.ids, sv.seg, self.g("embeddings.word_embeddings.weight"),
                                self.g("embeddings.position_embeddings.weight"),
                                self.g("embeddings.token_type_embeddings.weight") if self.has_type else None, sv.S,
                                pos_ids=sv.pk.pos_ids if sv.pk is not None else None)
        self._join_wgrads()
        if self.fp8:                       # delayed scaling: next micro-step quantises with this one's amaxes
            self.meta.update()
            self._fp8_calibrated = True

    def _layer_backward(self, l: int, ls: _LayerSaved, d: torch.Tensor, sv: _Saved, kfac) -> torch.Tensor:
        A, H, M = self.arena, self.H, d.size(0)
        ph, pa, seed = sv.p_hidden, sv.p_attn, sv.seed
        pre = f"encoder.layer.{l}."
        # ---- LN2 -> (residual grad, dropped grad of the FFN-2 output)
        d_pre2, d_y2, *q = K.layer_norm_bwd(
            d, ls.pre2, ls.mean2, ls.rstd2, self.p(pre + "output.LayerNorm.weight"),
            dgamma=self.g(pre + "output.LayerNorm.weight"), dbeta=self.g(pre + "output.LayerNorm.bias"),
            dbias=self.g(pre + "output.dense.bias"), want_dropped=True, p_drop=ph, seed=seed,
            drop_stream=_stream(l, SITE_FFN_OUT), fp8=self._side(f"{l}.d_y2"), keep_mask=ls.mask2)
        if kfac is not None:
            kfac.tap(self.prefix + pre + "output.dense", ls.act, d_y2)
        # ---- FFN-2 / GELU'
        if not self.fp8:
            # dgrad epilogue: d_y1 = (d_y2 W2) * gelu'(x) with the FFN-1 bias gradient (column sums) reduced from the
            # staged tile -- the dGELU pass and its bias-gradient pass are gone
            d_y1 = self._lin_bwd(l, "d_y2", "act", "w2", d_y2, ls.act_op, self.w(pre + "output.dense.weight"),
                                 self.g(pre + "output.dense.weight"), epi=K.EPI_MUL, res=ls.y1,
                                 colsum=self.g(pre + "intermediate.dense_act.bias"))
            q = []
        else:
            d_act = self._lin_bwd(l, "d_y2", "act", "w2", d_y2, ls.act_op, self.w(pre + "output.dense.weight"),
                                  self.g(pre + "output.dense.weight"), dyq=q[0] if q else None)
            side = self._side(f"{l}.d_y1")
            d_y1, *q = (K.dgelu_bwd(d_act, ls.y1, self.g(pre + "intermediate.dense_act.bias"), fp8=side) if side
                        else (K.dgelu_bwd(d_act, ls.y1, self.g(pre + "intermediate.dense_act.bias")),))
        d_x1 = self._lin_bwd(l, "d_y1", "x1", "w1", d_y1, ls.x1_op, self.w(pre + "intermediate.dense_act.weight"),
                             self.g(pre + "intermediate.dense_act.weight"), dyq=q[0] if q else None,
                             epi=K.EPI_ADD, res=d_pre2)
        # ---- LN1
        d_pre1, d_yo, *q = K.layer_norm_bwd(
            d_x1, ls.pre1, ls.mean1, ls.rstd1, self.p(pre + "attention.output.LayerNorm.weight"),
            dgamma=self.g(pre + "attention.output.LayerNorm.weight"),
            dbeta=self.g(pre + "attention.output.LayerNorm.bias"),
            dbias=self.g(pre + "attention.output.dense.bias"), want_dropped=True, p_drop=ph, seed=seed,
            drop_stream=_stream(l, SITE_ATTN_OUT), fp8=self._side(f"{l}.d_yo"), keep_mask=ls.mask1)
        if kfac is not None:
            kfac.tap(self.prefix + pre + "attention.output.dense", ls.ctx, d_yo)
        # ---- attention output projection
        d_ctx = self._lin_bwd(l, "d_yo", "ctx", "wo", d_yo, ls.ctx_op, self.w(pre + "attention.output.dense.weight"),
                              self.g(pre + "attention.output.dense.weight"), dyq=q[0] if q else None)
        # ---- attention core
        dqkv_q = None
        d_bqkv = self._qkv(l, A.flat_grad, "bias")           # the attention backward adds the QKV bias gradient
        if sv.pk is not None:
            d_qkv = K.attention_bwd(ls.qkv, None, ls.ctx, d_ctx, ls.lse, self.heads, p_drop=pa, seed=seed,
                                    stream=_stream(l, SITE_ATTN_PROB), cu_seqlens=sv.pk.cu_seqlens, S=sv.S, dbias=d_bqkv)
        else:
            d_qkv, *q = _as_tuple(K.attention_bwd(ls.qkv.view(sv.B, sv.S, 3 * H), sv.seqlens, ls.ctx.view(sv.B, sv.S, H),
                                                  d_ctx.view(sv.B, sv.S, H), ls.lse, self.heads, p_drop=pa, seed=seed,
                                                  stream=_stream(l, SITE_ATTN_PROB), fp8=self._side(f"{l}.d_qkv"),
                                                  dbias=d_bqkv))
            d_qkv = d_qkv.view(M, 3 * H)
            dqkv_q = q[0].view(M, 3 * H) if q else None
        if kfac is not None:
            for j, nm in enumerate(("query", "key", "value")):
                kfac.tap(self.prefix + pre + "attention.self." + nm, ls.x, d_qkv[:, j * H:(j + 1) * H])
        # ---- QKV projection
        d = self._lin_bwd(l, "d_qkv", "x", "wqkv", d_qkv, ls.x_op, self._qkv(l, A.flat_shadow, "weight"),
                          self._qkv(l, A.flat_grad, "weight"), dyq=dqkv_q, epi=K.EPI_ADD, res=d_pre1)
        self._wgrad_layer_done()
        return d

    # -- autograd bridge for models with ordinary torch heads (finetuning, inference) ------------------
    def _packing(self, attention_mask) -> Optional[Packing]:
        """The packing of this batch when ``BertModel.unpad`` is set and the unpadded path can serve the engine's
        configuration (fp8 operands run padded), else None."""
        if not getattr(self.bert, "unpad", False):
            return None
        if self.fp8:
            if not getattr(self, "_unpad_warned", False):
                warnings.warn("BertModel.unpad: fp8 operands have no unpadded path; running padded")
                self._unpad_warned = True
            return None
        return pack_rows(attention_mask)

    def encode(self, input_ids, token_type_ids, attention_mask) -> torch.Tensor:
        B, S = input_ids.shape
        training = self.bert.training and torch.is_grad_enabled()
        pack = self._packing(attention_mask)
        if pack is not None and pack.T == 0:          # nothing to compute: the output at masked positions is zero
            out = torch.zeros(B, S, self.H, dtype=torch.bfloat16, device=input_ids.device)
        elif not training:
            seq, _ = self.forward(input_ids, token_type_ids, attention_mask, training=False, pack=pack)
            out = _unpack(seq, pack, B * S).view(B, S, self.H)
        else:
            out = _EncoderFn.apply(self._hook, self, input_ids, token_type_ids, attention_mask, pack)
        if torch.is_autocast_enabled():
            return out.to(torch.get_autocast_dtype("cuda"))
        return out.float()


def _unpack(seq: torch.Tensor, pack: Optional[Packing], rows: int) -> torch.Tensor:
    """Packed rows [T, H] -> [rows, H] with zeros at the masked positions (identity without a packing)."""
    if pack is None:
        return seq
    out = torch.zeros(rows, seq.size(1), dtype=seq.dtype, device=seq.device)
    K.scatter_rows(seq, pack.rows, out)
    return out


class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, engine, input_ids, token_type_ids, attention_mask, pack=None):
        seq, sv = engine.forward(input_ids, token_type_ids, attention_mask, training=True, pack=pack)
        ctx.engine, ctx.sv = engine, sv
        return _unpack(seq, pack, input_ids.numel()).view(input_ids.size(0), input_ids.size(1), engine.H)

    @staticmethod
    def backward(ctx, d_seq):
        engine, sv = ctx.engine, ctx.sv
        d = d_seq.reshape(-1, engine.H).to(torch.bfloat16).contiguous()
        if sv.pk is not None:                       # the gradient of the packed rows; masked positions had no effect
            d = K.gather_rows(d, sv.pk.rows)
        engine.backward(sv, d)
        ctx.sv = None
        return torch.zeros(1, device=d_seq.device), None, None, None, None, None


class _HeadLinearFn(torch.autograd.Function):
    """y = x W^T + b for the small-N fine-tuning heads (QA: N = 2, token / sequence classifiers: N = num_labels,
    multiple choice: N = 1; reference src/modeling.py:1127-1128, 1188-1189, 1256-1257, 1323-1326) on the wgmma GEMM:
    N is padded to 8 output columns, forward NT with fp32 store, dgrad NN, wgrad TN with fp32 store -- the SQuAD / NER
    steps then contain no library GEMM (VERDICT r1: K28 / K29 ran as torch ops = cuBLAS behind the bridge)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        shape = x.shape
        xb = x.reshape(-1, shape[-1])
        xb = (xb if xb.dtype == torch.bfloat16 else xb.to(torch.bfloat16)).contiguous()
        n, H = weight.shape
        npad = (n + 7) // 8 * 8
        wp = torch.zeros(npad, H, dtype=torch.bfloat16, device=x.device)
        wp[:n] = weight.detach().to(torch.bfloat16)
        y = K.gemm(xb, wp, epi=K.EPI_F32, block_n=128)[:, :n]
        if bias is not None:
            y = y + bias.detach().float()
        ctx.save_for_backward(xb, wp)
        ctx.meta = (shape, n, x.dtype, bias is not None, weight.dtype)
        return y.to(x.dtype if x.dtype != torch.float32 else torch.float32).view(*shape[:-1], n)

    @staticmethod
    def backward(ctx, gy):
        xb, wp = ctx.saved_tensors
        shape, n, xdtype, has_bias, wdtype = ctx.meta
        go = gy.reshape(-1, n).float()
        gop = torch.zeros(go.size(0), wp.size(0), dtype=torch.bfloat16, device=go.device)
        gop[:, :n] = go
        dx = K.gemm(gop, wp, layout=K.NN).to(xdtype).view(*shape)
        dw = K.gemm(gop, xb, layout=K.TN, epi=K.EPI_F32, block_n=128)[:n].to(wdtype)
        db = go.sum(0) if has_bias else None
        return dx, dw, db


def head_linear(linear: torch.nn.Linear, x: torch.Tensor) -> torch.Tensor:
    """``linear(x)`` through :class:`_HeadLinearFn` when the sm_90a extension can serve it (CUDA, H % 8 == 0, at most
    64 outputs, at least 128 rows -- smaller problems are launch bound either way), else the module itself."""
    H = x.size(-1)
    rows = x.numel() // max(H, 1)
    if x.is_cuda and ops.available() and H % 8 == 0 and linear.out_features <= 64 and rows >= 128:
        return _HeadLinearFn.apply(x, linear.weight, linear.bias)
    return linear(x)


class _GraphedProgram:
    """What the fused programs share: the token bucket of an unpadded batch, the steps every program starts with
    (packing, encoder forward, [CLS] rows, pooler), the CUDA-graph key, and the policy that runs a kernel program
    eagerly for its first ``graph_warmup`` calls per input signature, then captures it once and replays it as one CUDA
    graph, every capture in one memory pool."""

    def __init__(self, model):
        self.model = model
        self.engine: FusedEncoderEngine = model.bert.fused_engine()
        self.arena = self.engine.arena
        # CUDA graphs: the micro-step is ~600 launches of static shape; replaying it as one graph removes the
        # launch gaps (~6 % of the phase-1 step).  B200_GRAPH=0 keeps the eager program.
        self.use_graphs = os.environ.get("B200_GRAPH", "1") != "0"
        self.graph_warmup = 2                 # eager calls per input signature before capturing
        self._graphs: Dict[tuple, dict] = {}
        self._seed_step: Optional[torch.Tensor] = None
        self._cap_stream = None               # high-priority capture stream (wgrad side-stream mode)
        self._cls: Dict[tuple, torch.Tensor] = {}    # [CLS] row indices of the padded batch shapes

    def _graph_ok(self) -> bool:
        kf = getattr(self.model.bert, "_kfac", None)
        if not self.use_graphs or (kf is not None and getattr(kf, "capture", True)):
            return False                      # tapped micro-steps keep Python-side state
        return self.arena.device.type == "cuda"

    def _bucket(self, input_mask, tokens: Optional[int], kfac: bool = True):
        """(T_cap, D) of this micro-step when it runs unpadded (``BertModel.unpad``), else None.  fp8 operands have no
        unpadded path (warned once), and K-FAC micro-steps that feed the factors run padded so that their statistics
        are the padded ones (``kfac=False``: an evaluation, which feeds nothing).  Without ``tokens`` the count is read
        back from the device (one host sync)."""
        if not getattr(self.model.bert, "unpad", False):
            return None
        if self.engine.fp8:
            if not getattr(self, "_unpad_warned", False):
                warnings.warn("BertModel.unpad: fp8 operands have no unpadded pre-training path or classification "
                              "program; running padded")
                self._unpad_warned = True
            return None
        kf = getattr(self.model.bert, "_kfac", None)
        if kfac and kf is not None and getattr(kf, "capture", True):
            return None
        B, S = input_mask.shape
        return token_bucket(packed_tokens(input_mask) if tokens is None else int(tokens), B, S)

    def _encode(self, input_ids, segment_ids, input_mask, bucket, train: bool, seed: Optional[int] = None):
        """The start of every program: the device packing of the batch into ``bucket`` (padded without one), then the
        encoder forward -- ``train``: saving activations, with dropout as ``model.training`` says; otherwise without
        dropout.  Returns (sequence output, saved-or-None, packing-or-None, its row count M)."""
        B, S = input_ids.shape
        pk = pack_device(input_mask, input_ids, segment_ids, *bucket) if bucket is not None else None
        M = pk.T if pk is not None else B * S
        # an evaluation passes an explicit seed: the engine's call counter, which numbers the training dropout seeds,
        # stays where it is
        seq, sv = self.engine.forward(input_ids, segment_ids, input_mask, training=train, seed=seed if train else 0,
                                      dropout=train and self.model.training, pack=pk)
        return seq, sv, pk, M

    def _cls_rows(self, pk: Optional[Packing], B: int, S: int, device) -> torch.Tensor:
        """Rows of the [CLS] tokens in the sequence output: the first packed row of every sequence, or b * S.  The
        padded indices are one tensor per (B, S), never replaced or evicted: captured graphs keep reading them."""
        if pk is not None:
            return pk.cls_rows
        idx = self._cls.get((B, S))
        if idx is None:
            idx = self._cls[(B, S)] = torch.arange(B, device=device, dtype=torch.int32) * S
        return idx

    def _pooled(self, seq, cls_idx):
        """(the [CLS] rows [B, H] bf16, the pooler output): a gather, then a GEMM with the bias + tanh epilogue."""
        eng, A = self.engine, self.arena
        cls_tok = K.gather_rows(seq, cls_idx)
        pooled = K.gemm(cls_tok, A.shadow(eng.prefix + "pooler.dense_act.weight"), epi=K.EPI_BIAS_TANH,
                        bias=A.shadow(eng.prefix + "pooler.dense_act.bias"))
        return cls_tok, pooled

    def _graph_key(self, kind: str, args, bucket, train: bool, *extra) -> tuple:
        """CUDA-graph key of one call: ``kind``, the batch shape, the dtype of every argument (None where absent), the
        fp8 mode; for a training program its mode, activation checkpointing, the weight-gradient stream and ``extra``;
        then the deterministic mode and, last, the token bucket."""
        eng = self.engine
        key = (kind, tuple(args[0].shape), tuple(None if t is None else t.dtype for t in args), eng.fp8)
        if train:
            key += (self.model.training, bool(getattr(self.model.bert.encoder, "_checkpoint_activations", False)),
                    bool(eng.wgrad_side), *extra)
        return key + (K.deterministic(), bucket)

    def _graphed(self, key: tuple, args, run, train: bool, grad_scale: float = 1.0, what: str = "micro-step"):
        """``run(*args)`` -- eager for the first ``graph_warmup`` calls of ``key``, then captured once and replayed with
        ``args`` copied into the graph's static inputs.  Returns the program's output (the graph's own tensor when
        replayed: valid until the next replay).

        ``train``: the program draws dropout and writes gradients.  The capture runs it as ``run(*static,
        seed=engine._seed_base)`` after advancing the device step counter, so that every replay draws fresh masks; the
        fp8 weight copies are refreshed before every call, and ``grad_scale``, a launch constant, is part of the capture.
        Otherwise (an evaluation) the step counter does not move."""
        ent = self._graphs.setdefault(key, {"calls": 0})
        ent["calls"] += 1
        eng = self.engine
        if train and "graph" in ent and ent["grad_scale"] != float(grad_scale):
            # the loss scale is a launch constant: a GradScaler update invalidates the capture (rare); drop it
            # (and its private memory pool) and capture again right away
            for k in ("graph", "static", "out"):
                ent.pop(k)
        if "graph" not in ent:
            if ent["calls"] <= self.graph_warmup or (eng.fp8 and not eng._fp8_calibrated):
                return run(*args)
            if train and self._seed_step is None:
                self._seed_step = torch.zeros(1, dtype=torch.int64, device=self.arena.device)
                ops.extension().set_seed_step(self._seed_step)
            static = [None if t is None else t.clone() for t in args]
            if train:
                eng.prepare_step()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = K.KERNEL_LAUNCHES
            pool = next((e["graph"].pool() for e in self._graphs.values() if "graph" in e), None)
            # replays never overlap: all captures share one memory pool; thread_local: a data-loader thread that pins
            # or allocates memory while we capture must not abort the capture
            extra = {}
            if train and eng.wgrad_side:      # capture on a high-priority stream: the dgrad chain wins SMs over the wgrads
                if self._cap_stream is None:
                    self._cap_stream = torch.cuda.Stream(device=self.arena.device, priority=-1)
                extra["stream"] = self._cap_stream
            # no cyclic garbage collection inside the capture: it could destroy the CUDA graphs and events of programs
            # that are no longer referenced (a model and its engine form reference cycles), and a CUDA call of this
            # thread that is not capturable invalidates the capture
            gc_on = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.graph(graph, pool=pool, capture_error_mode="thread_local", **extra):
                    if train:
                        self._seed_step.add_(1)
                        out = run(*static, seed=eng._seed_base)
                    else:                     # no dropout, and training's step counter must not move
                        out = run(*static)
            except Exception as e:            # e.g. an allocator / stream condition this build of torch cannot capture
                warnings.warn(f"CUDA-graph capture of the {what} failed ({type(e).__name__}: {e}); "
                              "continuing with the eager kernel program")
                K.KERNEL_LAUNCHES = n0
                self.use_graphs = False
                torch.cuda.synchronize()      # nothing of the captured program ran: the accumulated gradients are intact
                return run(*args)
            finally:
                if gc_on:
                    gc.enable()
            ent.update(graph=graph, static=static, out=out, launches=K.KERNEL_LAUNCHES - n0, grad_scale=float(grad_scale))
            K.KERNEL_LAUNCHES = n0            # the capture itself ran nothing
        for dst, src in zip(ent["static"], args):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        if train:
            eng.prepare_step()
        ent["graph"].replay()
        K._count(ent["launches"])
        return ent["out"]

    def _eval_graphs_ok(self) -> bool:
        return self.use_graphs and self.arena.device.type == "cuda"

    def _keeping_fp8_table(self, fn):
        """``fn()`` with the fp8 scaling table restored afterwards (the weight copies are refreshed first, as the next
        micro-step would): an evaluation must not move the training's delayed scaling."""
        eng = self.engine
        table = None
        if eng.fp8:
            eng.prepare_step()
            table = eng.meta.table.clone()
        try:
            return fn()
        finally:
            if table is not None:
                eng.meta.table.copy_(table)


class FusedPretrainer(_GraphedProgram):
    """Forward + backward of ``BertForPreTraining`` + criterion as one kernel program.

    ``forward_backward`` returns the (unscaled) loss of the micro-batch as a device scalar and leaves the
    gradients -- multiplied by ``grad_scale`` (= loss_scale / accumulation_steps) -- accumulated in the arena.
    """

    def __init__(self, model):
        super().__init__(model)
        cfg = model.config
        self.V, self.H = cfg.vocab_size, cfg.hidden_size
        self.has_nsp = model.cls.has_nsp and model.bert.pooler is not None
        self.max_pred = int(getattr(cfg, "max_predictions_per_seq", 0)) or None
        self._loss = None
        self.grad_push = False                # set by the runtime around the last micro-step (PeerComm.begin_push)

    def _max_pred(self, labels: torch.Tensor) -> int:
        # capacity of masked positions per sequence; fixed per run so shapes stay static
        if self.max_pred is None:
            # no --max_predictions_per_seq: the capacity is the sequence length (any batch fits; the static-shape head
            # then costs S rows per sequence, so runners should always pass the flag -- data/dataset.py validates
            # pre-masked shards against it)
            self.max_pred = (labels.size(1) + 7) // 8 * 8
        return self.max_pred

    @torch.no_grad()
    def forward_backward(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels,
                         grad_scale: float = 1.0, tokens: Optional[int] = None) -> torch.Tensor:
        """One micro-step.  After ``graph_warmup`` eager calls with the same input signature the whole kernel
        program (forward, loss, backward: ~600 launches) is captured once and replayed as ONE CUDA graph; the
        dropout seed advances through a device-side step counter inside the graph.

        Unpadded (``BertModel.unpad``): the program packs the batch on the device into the token bucket of ``tokens``
        (:func:`packed_tokens` of the mask, a host int; counted on the device when omitted) and computes T_cap rows
        instead of B * S.  The bucket is part of the graph key: one graph per bucket, all in one memory pool."""
        bucket = self._bucket(input_mask, tokens)
        if not self._graph_ok():
            return self._program(input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels, grad_scale,
                                 bucket=bucket)
        args = (input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels)
        key = self._graph_key("train", args, bucket, True, bool(self.grad_push))
        return self._graphed(key, args, lambda *a, seed=None: self._program(*a, grad_scale, seed=seed, bucket=bucket),
                             train=True, grad_scale=grad_scale)

    @torch.no_grad()
    def _program(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels,
                 grad_scale: float = 1.0, seed: Optional[int] = None, bucket=None) -> torch.Tensor:
        """The kernel program of one micro-step; ``bucket`` = (T_cap, D) runs it on the packed tokens of the batch
        (T_cap rows: the real tokens, then a pad tail of inert [PAD] rows in D dummy sequences)."""
        eng, A, H = self.engine, self.arena, self.H
        B, S = input_ids.shape
        seq, sv, pk, M = self._encode(input_ids, segment_ids, input_mask, bucket, train=True, seed=seed)
        labels = masked_lm_labels.to(torch.int32).contiguous()
        mp = self._max_pred(labels)
        idx, tgt, count = K.mlm_compact(labels, mp, row_map=pk.row_map if pk is not None else None)
        loss = torch.zeros(1, dtype=torch.float32, device=seq.device)

        # ---- MLM head forward (masked rows only)
        logits, (rows, t_pre, t_act, t_ln, t_mean, t_rstd) = self._mlm_forward(seq, idx, save_stats=True)
        K.softmax_ce_(logits, tgt, count, grad_scale, loss)            # logits <- dlogits

        # ---- MLM head backward
        emb_w = eng.w("embeddings.word_embeddings.weight")            # tied decoder weight [V, H]
        K.colsum_accumulate(logits, A.grad("cls.predictions.bias"))
        d_t_ln = K.gemm(logits, emb_w, layout=K.NN)
        K.wgrad_accumulate(logits, t_ln, eng.g("embeddings.word_embeddings.weight"))
        d_t_act, _ = K.layer_norm_bwd(d_t_ln, t_act, t_mean, t_rstd, A.view("cls.predictions.transform.LayerNorm.weight"),
                                      dgamma=A.grad("cls.predictions.transform.LayerNorm.weight"),
                                      dbeta=A.grad("cls.predictions.transform.LayerNorm.bias"))
        d_t_pre = K.dgelu_bwd(d_t_act, t_pre, A.grad("cls.predictions.transform.dense_act.bias"))
        K.wgrad_accumulate(d_t_pre, rows, A.grad("cls.predictions.transform.dense_act.weight"))
        d_rows = K.gemm(d_t_pre, A.shadow("cls.predictions.transform.dense_act.weight"), layout=K.NN)
        d_seq = torch.zeros(M, H, dtype=torch.bfloat16, device=seq.device)
        K.scatter_rows(d_rows, idx, d_seq)

        # ---- NSP head on our own kernels as well (K19 / K20 / K25): pooler = wgmma GEMM with the bias+tanh epilogue
        #      on the [CLS] rows, classifier + CE + their backward = one small kernel, pooler backward = the usual
        #      dgrad / wgrad GEMMs (M = B rows)
        if self.has_nsp and next_sentence_labels is not None:
            pool, nsp = self.model.bert.pooler.dense_act, self.model.cls.seq_relationship
            cls_idx = self._cls_rows(pk, B, S, seq.device)
            cls_tok, pooled = self._pooled(seq, cls_idx)
            d_z = K.nsp_head_(pooled, A.shadow("cls.seq_relationship.weight"), nsp.bias, next_sentence_labels.long().view(-1),
                              grad_scale, loss, nsp.weight.grad, nsp.bias.grad)
            kf = getattr(self.model.bert, "_kfac", None)
            if kf is not None and not getattr(kf, "capture", True):
                kf = None
            if kf is not None:                     # the NSP classifier is an nn.Linear: K-FAC preconditions it; its output
                with torch.no_grad():              # gradient is rebuilt here (K-FAC mode only, plain torch on [B, 2])
                    lg = pooled.float() @ A.shadow("cls.seq_relationship.weight").float().t() + nsp.bias
                    y = next_sentence_labels.long().view(-1)
                    valid = (y >= 0).float()
                    d_lg = (torch.softmax(lg, -1) - F.one_hot(y.clamp(min=0), 2).float()) \
                        * (valid / valid.sum().clamp_(min=1.0) * grad_scale).unsqueeze(1)
                kf.tap("cls.seq_relationship", pooled, d_lg)
            K.wgrad_accumulate(d_z, cls_tok, pool.weight.grad)
            K.colsum_accumulate(d_z, pool.bias.grad)
            d_cls = K.gemm(d_z, A.shadow(eng.prefix + "pooler.dense_act.weight"), layout=K.NN)
            if pk is not None and K.deterministic():
                # torch's deterministic index_add_ sorts its indices; the rows are distinct, so gather, add and scatter
                # back instead: the same bf16 add, on the engine's kernels
                K.scatter_rows(K.gather_rows(d_seq, pk.cls_rows) + d_cls, pk.cls_rows, d_seq)
            elif pk is not None:                   # the same bf16 add at the (distinct) first packed rows
                d_seq.index_add_(0, pk.cls_rows.long(), d_cls)
            else:
                d_seq.view(B, S, H)[:, 0] += d_cls

        eng.backward(sv, d_seq)
        return loss.squeeze(0) if loss.dim() else loss

    def _mlm_forward(self, seq, idx, save_stats: bool):
        """The MLM head on the masked rows ``idx`` of the sequence output: gather -> transform GEMM + bias -> GELU ->
        LayerNorm (with its row statistics when ``save_stats``) -> tied decoder GEMM + bias.  Returns (logits [rows,
        V], (rows, t_pre, t_act, t_ln, t_mean, t_rstd)), the intermediates the backward reads."""
        A = self.arena
        rows = K.gather_rows(seq, idx)
        t_pre = K.gemm(rows, A.shadow("cls.predictions.transform.dense_act.weight"), epi=K.EPI_BIAS,
                       bias=A.shadow("cls.predictions.transform.dense_act.bias"))
        t_act = K.gelu_fwd(t_pre)
        t_ln, t_mean, t_rstd = K.layer_norm_fwd(t_act, A.view("cls.predictions.transform.LayerNorm.weight"),
                                                A.view("cls.predictions.transform.LayerNorm.bias"), save_stats=save_stats)
        logits = K.gemm(t_ln, self.engine.w("embeddings.word_embeddings.weight"), epi=K.EPI_BIAS,
                        bias=A.shadow("cls.predictions.bias"))
        return logits, (rows, t_pre, t_act, t_ln, t_mean, t_rstd)

    # -- evaluation ------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def evaluate(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels, acc: torch.Tensor,
                 tokens: Optional[int] = None) -> torch.Tensor:
        """Adds the metric sums of one batch into ``acc`` (fp64 [6] on the device): ``[mlm_loss_sum, mlm_correct,
        mlm_count, nsp_loss_sum, nsp_correct, nsp_count]`` (the NSP half stays zero without an NSP head or labels).
        Forward only, without dropout, and every sum in a fixed order (no atomics): the same batch gives the same bits in
        the default and the deterministic mode, padded or unpadded, eager or replayed.

        The training state comes out as it went in: no activation is saved, no gradient is written, the dropout seed
        counters (``_seed_step``, the engine's call count) and ``model.training`` do not move, and the fp8 scaling table
        is restored after the batch (the weight copies are refreshed first, as the next micro-step would).  Unpadded
        (``BertModel.unpad``) the batch is packed into the token bucket of ``tokens`` as in training.  CUDA graphs: the
        training policy (``graph_warmup`` eager calls per signature, then one capture), with keys of their own in the
        training graphs' memory pool."""
        if acc.dtype != torch.float64 or acc.numel() != 6:
            raise ValueError("evaluate: acc must be an fp64 tensor of 6 elements")
        bucket = self._bucket(input_mask, tokens, kfac=False)
        args = (input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels)
        acc += self._keeping_fp8_table(lambda: self._eval_replay(args, bucket))
        return acc

    def _eval_replay(self, args, bucket) -> torch.Tensor:
        """The evaluation program of ``args``, eager or as a replayed CUDA graph; returns its fp64 [6] sums."""
        run = lambda *a: self._eval_program(*a, bucket=bucket)      # noqa: E731
        if not self._eval_graphs_ok():
            return run(*args)
        return self._graphed(self._graph_key("eval", args, bucket, False), args, run, train=False, what="evaluation")

    @torch.no_grad()
    def _eval_program(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels,
                      bucket=None) -> torch.Tensor:
        """Encoder forward without dropout, the MLM head on the masked rows and the NSP head on the [CLS] rows, then the
        metric kernels.  Returns fp64 [6]: the MLM sums {loss, correct, count}, then the NSP sums."""
        B, S = input_ids.shape
        seq, _, pk, _ = self._encode(input_ids, segment_ids, input_mask, bucket, train=False)
        labels = masked_lm_labels.to(torch.int32).contiguous()
        idx, tgt, _ = K.mlm_compact(labels, self._max_pred(labels), row_map=pk.row_map if pk is not None else None)
        part = torch.zeros(6, dtype=torch.float64, device=seq.device)

        logits, _ = self._mlm_forward(seq, idx, save_stats=False)
        K.mlm_eval(logits, tgt, part[0:3])

        if self.has_nsp and next_sentence_labels is not None:
            _, pooled = self._pooled(seq, self._cls_rows(pk, B, S, seq.device))
            K.nsp_eval(pooled, self.arena.shadow("cls.seq_relationship.weight"), self.model.cls.seq_relationship.bias,
                       next_sentence_labels.long().view(-1).contiguous(), part[3:6])
        return part


class FusedClassifier(_GraphedProgram):
    """Fine-tuning and evaluation of ``BertForSequenceClassification`` (GLUE) as one kernel program each.

    Training (``train_step``): [device packing] -> encoder forward -> gather of the [CLS] rows -> pooler GEMM with the
    bias + tanh epilogue -> ``cls_head`` (dropout, classifier, cross-entropy and their backward in one launch) -> pooler
    wgrad / bias / dgrad -> the [CLS]-row gradient into a zero sequence gradient -> encoder backward.  The classifier
    dropout draws from stream :data:`CLS_STREAM` with the encoder's seed, so a replayed graph draws new masks as the
    device step counter advances.  Evaluation (``predict``): the forward without dropout, ending in fp32 logits.  Both
    follow the pre-training policy for buckets and graphs: one graph per (batch shape, bucket, mode), all in one pool.
    Rows whose label is -1 are inert: a batch filled up to the static batch size with such rows (one unmasked token,
    label -1) replays the same graph and its mean loss is over the real rows only."""

    def __init__(self, model):
        super().__init__(model)
        if model.bert.pooler is None:
            raise ValueError("FusedClassifier: the model has no pooler (config.next_sentence is false)")
        if model.num_labels not in K.CLS_CLASSES:
            raise ValueError(f"FusedClassifier: {model.num_labels} labels; the classifier kernel is built for "
                             f"{K.CLS_CLASSES} classes")
        self.H = model.config.hidden_size

    @torch.no_grad()
    def train_step(self, input_ids, segment_ids, input_mask, labels, grad_scale: float = 1.0,
                   tokens: Optional[int] = None) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the mean cross-entropy over the rows whose label is not -1
        (a device scalar) and accumulates the gradients, times ``grad_scale``, in the arena.  Unpadded
        (``BertModel.unpad``) the batch is packed into the token bucket of ``tokens`` (its unmasked token count, a host
        int; read back from the device when omitted)."""
        bucket = self._bucket(input_mask, tokens)
        run = lambda *a, seed=None: self._program(*a, grad_scale, seed=seed, bucket=bucket)   # noqa: E731
        args = (input_ids, segment_ids, input_mask, labels)
        if not self._graph_ok():
            return run(*args)
        return self._graphed(self._graph_key("cls", args, bucket, True), args, run, train=True, grad_scale=grad_scale)

    @torch.no_grad()
    def _program(self, input_ids, segment_ids, input_mask, labels, grad_scale: float = 1.0, seed: Optional[int] = None,
                 bucket=None) -> torch.Tensor:
        eng, A, H = self.engine, self.arena, self.H
        B, S = input_ids.shape
        seq, sv, pk, M = self._encode(input_ids, segment_ids, input_mask, bucket, train=True, seed=seed)
        cls_idx = self._cls_rows(pk, B, S, seq.device)
        cls_tok, pooled = self._pooled(seq, cls_idx)
        loss = torch.zeros(1, dtype=torch.float32, device=seq.device)
        pool, clf = self.model.bert.pooler.dense_act, self.model.classifier
        d_z = K.cls_head_(pooled, A.shadow("classifier.weight"), clf.bias, labels.long().view(-1).contiguous(),
                          grad_scale, loss, clf.weight.grad, clf.bias.grad, p_drop=sv.p_hidden, seed=sv.seed,
                          stream=CLS_STREAM)
        pw = A.shadow(eng.prefix + "pooler.dense_act.weight")
        K.wgrad_accumulate(d_z, cls_tok, pool.weight.grad)
        K.colsum_accumulate(d_z, pool.bias.grad)
        d_cls = K.gemm(d_z, pw, layout=K.NN)
        # the sequence gradient is zero but at the (distinct) [CLS] rows: a scatter is the whole add, in every mode
        d_seq = torch.zeros(M, H, dtype=torch.bfloat16, device=seq.device)
        K.scatter_rows(d_cls, cls_idx, d_seq)
        eng.backward(sv, d_seq)
        return loss.squeeze(0)

    @torch.no_grad()
    def predict(self, input_ids, segment_ids, input_mask, tokens: Optional[int] = None) -> torch.Tensor:
        """fp32 logits [B, C] of one batch: the forward without dropout.  Leaves the training state as it was: no
        activation saved, no gradient written, the seed counters, ``model.training`` and the fp8 scaling table unmoved.
        Graphs under keys of their own, in the training graphs' pool."""
        bucket = self._bucket(input_mask, tokens, kfac=False)
        args = (input_ids, segment_ids, input_mask)
        run = lambda *a: self._eval_program(*a, bucket=bucket)                                 # noqa: E731

        def go():
            if not self._eval_graphs_ok():
                return run(*args)
            key = self._graph_key("cls-eval", args, bucket, False)
            return self._graphed(key, args, run, train=False, what="evaluation").clone()
        return self._keeping_fp8_table(go)

    @torch.no_grad()
    def _eval_program(self, input_ids, segment_ids, input_mask, bucket=None) -> torch.Tensor:
        B, S = input_ids.shape
        seq, _, pk, _ = self._encode(input_ids, segment_ids, input_mask, bucket, train=False)
        _, pooled = self._pooled(seq, self._cls_rows(pk, B, S, seq.device))
        return K.cls_logits(pooled, self.arena.shadow("classifier.weight"), self.model.classifier.bias)


class _TokenHeadProgram(_GraphedProgram):
    """What the per-token head programs share: the head's bf16 weight, fp32 bias and gradient slots, its evaluation
    program (the forward without dropout, ending in fp32 logits [B, S, N] -- ``bias`` at the masked positions of an
    unpadded batch), and ``predict`` under graph keys of kind ``eval_kind``."""

    eval_kind = ""

    def __init__(self, model, head: torch.nn.Linear, head_name: str):
        super().__init__(model)
        if head.out_features > K.TOKEN_HEAD_MAX_N:
            raise ValueError(f"{type(self).__name__}: {head.out_features} outputs; the per-token head kernels serve "
                             f"at most {K.TOKEN_HEAD_MAX_N}")
        self.head, self.head_name = head, head_name

    def _w(self) -> torch.Tensor:
        return self.arena.shadow(self.head_name + ".weight")

    @torch.no_grad()
    def _predict(self, input_ids, segment_ids, input_mask, tokens: Optional[int] = None) -> torch.Tensor:
        bucket = self._bucket(input_mask, tokens, kfac=False)
        args = (input_ids, segment_ids, input_mask)
        run = lambda *a: self._eval_program(*a, bucket=bucket)                                 # noqa: E731

        def go():
            if not self._eval_graphs_ok():
                return run(*args)
            key = self._graph_key(self.eval_kind, args, bucket, False)
            return self._graphed(key, args, run, train=False, what="evaluation").clone()
        return self._keeping_fp8_table(go)

    @torch.no_grad()
    def _eval_program(self, input_ids, segment_ids, input_mask, bucket=None) -> torch.Tensor:
        B, S = input_ids.shape
        seq, _, pk, _ = self._encode(input_ids, segment_ids, input_mask, bucket, train=False)
        logits = K.token_logits(seq, self._w(), self.head.bias, row_map=pk.row_map if pk is not None else None,
                                mask=input_mask)
        return logits.view(B, S, -1)


class FusedQuestionAnswering(_TokenHeadProgram):
    """SQuAD fine-tuning and prediction of ``BertForQuestionAnswering`` as one kernel program each.

    Training (``train_step``): encoder forward -> ``token_logits`` (N = 2, no dropout, as in the reference) ->
    ``span_ce_`` (start / end cross-entropy in place) -> ``token_head_bwd`` -> encoder backward.  Training always runs
    padded, whatever ``BertModel.unpad`` says: the span softmax normalises over every position, and the encoder outputs
    of the padded positions cannot be had without computing them.  Prediction (``predict``) honours ``unpad``.  A row
    whose start and end positions are S (outside [0, S) after the clamp) is inert: a batch filled up to the static batch
    size with such rows replays the same graph and its loss is that of the real rows."""

    eval_kind = "qa-eval"

    def __init__(self, model):
        super().__init__(model, model.qa_outputs, "qa_outputs")

    @torch.no_grad()
    def train_step(self, input_ids, segment_ids, input_mask, start_positions, end_positions,
                   grad_scale: float = 1.0) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the SQuAD loss (a device scalar) and accumulates the
        gradients, times ``grad_scale``, in the arena."""
        run = lambda *a, seed=None: self._program(*a, grad_scale, seed=seed)                  # noqa: E731
        args = (input_ids, segment_ids, input_mask, start_positions, end_positions)
        if not self._graph_ok():
            return run(*args)
        return self._graphed(self._graph_key("qa", args, None, True), args, run, train=True, grad_scale=grad_scale)

    @torch.no_grad()
    def _program(self, input_ids, segment_ids, input_mask, start_positions, end_positions, grad_scale: float = 1.0,
                 seed: Optional[int] = None) -> torch.Tensor:
        seq, sv, _, _ = self._encode(input_ids, segment_ids, input_mask, None, train=True, seed=seed)
        logits = K.token_logits(seq, self._w(), self.head.bias)
        loss = torch.zeros(1, dtype=torch.float32, device=seq.device)
        K.span_ce_(logits, start_positions, end_positions, grad_scale, loss)            # logits <- dlogits
        d_seq = K.token_head_bwd(logits, seq, self._w(), self.head.weight.grad, self.head.bias.grad)
        self.engine.backward(sv, d_seq)
        return loss.squeeze(0)

    def predict(self, input_ids, segment_ids, input_mask, tokens: Optional[int] = None):
        """fp32 ``(start, end)`` logits, each [B, S], without dropout; unpadded (``BertModel.unpad``, the batch packed
        into the token bucket of ``tokens``) they are exactly ``bias`` at the masked positions.  Leaves the training
        state as it was."""
        out = self._predict(input_ids, segment_ids, input_mask, tokens).permute(2, 0, 1).contiguous()
        return out[0], out[1]


class FusedTokenClassifier(_TokenHeadProgram):
    """NER fine-tuning and prediction of ``BertForTokenClassification`` as one kernel program each.

    Training (``train_step``): [device packing] -> encoder forward -> ``token_logits`` with dropout
    ``hidden_dropout_prob`` on the sequence output (stream :data:`TOKEN_STREAM`, the encoder's seed: a replayed graph
    draws new masks) -> ``token_ce_`` (the masked cross-entropy in place, through the packing's ``row_map``) ->
    ``token_head_bwd`` -> encoder backward.  Prediction (``predict``): fp32 logits [B, S, N].  A position counts iff its
    ``attention_mask`` is 1 and its label lies in [0, N): rows of label -100 are inert, so a short batch filled up with
    them replays the same graph and its loss is that of the real rows."""

    eval_kind = "tok-eval"

    def __init__(self, model):
        super().__init__(model, model.classifier, "classifier")

    @torch.no_grad()
    def train_step(self, input_ids, segment_ids, input_mask, labels, grad_scale: float = 1.0,
                   tokens: Optional[int] = None) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the mean cross-entropy over the counted positions (a
        device scalar) and accumulates the gradients, times ``grad_scale``, in the arena.  Unpadded
        (``BertModel.unpad``) the batch is packed into the token bucket of ``tokens`` (its unmasked token count, a host
        int; read back from the device when omitted)."""
        bucket = self._bucket(input_mask, tokens)
        run = lambda *a, seed=None: self._program(*a, grad_scale, seed=seed, bucket=bucket)   # noqa: E731
        args = (input_ids, segment_ids, input_mask, labels)
        if not self._graph_ok():
            return run(*args)
        return self._graphed(self._graph_key("tok", args, bucket, True), args, run, train=True, grad_scale=grad_scale)

    @torch.no_grad()
    def _program(self, input_ids, segment_ids, input_mask, labels, grad_scale: float = 1.0, seed: Optional[int] = None,
                 bucket=None) -> torch.Tensor:
        seq, sv, pk, _ = self._encode(input_ids, segment_ids, input_mask, bucket, train=True, seed=seed)
        logits = K.token_logits(seq, self._w(), self.head.bias, sv.p_hidden, sv.seed, TOKEN_STREAM)
        loss = torch.zeros(1, dtype=torch.float32, device=seq.device)
        K.token_ce_(logits, labels, grad_scale, loss, mask=input_mask, row_map=pk.row_map if pk is not None else None)
        d_seq = K.token_head_bwd(logits, seq, self._w(), self.head.weight.grad, self.head.bias.grad, sv.p_hidden,
                                 sv.seed, TOKEN_STREAM)
        self.engine.backward(sv, d_seq)
        return loss.squeeze(0)

    def predict(self, input_ids, segment_ids, input_mask, tokens: Optional[int] = None) -> torch.Tensor:
        """fp32 logits [B, S, N] without dropout (``bias`` at the masked positions when unpadded).  Leaves the training
        state as it was."""
        return self._predict(input_ids, segment_ids, input_mask, tokens)
