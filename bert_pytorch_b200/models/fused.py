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
"""
from __future__ import annotations

import math
import os
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


def _stream(layer: int, site: int) -> int:
    return layer * 8 + site


def _as_tuple(x):
    return x if isinstance(x, tuple) else (x,)


def _use_sdpa() -> bool:
    return os.environ.get("B200_ATTN", "native") == "sdpa"


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
    sdpa: tuple = None
    x_op: torch.Tensor = None      # operands of the four weight-gradient GEMMs (bf16 tensors or their fp8 copies)
    ctx_op: torch.Tensor = None
    x1_op: torch.Tensor = None
    act_op: torch.Tensor = None


@dataclass
class _Saved:
    B: int = 0
    S: int = 0
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
            if not _use_sdpa():
                raise NotImplementedError("fused attention needs head_dim == 64 (set B200_ATTN=sdpa otherwise)")
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
        # GELU / GELU' inside the FFN GEMM epilogues (bf16 operand path); B200_FUSED_GELU=0 restores the two
        # bandwidth kernels
        self.fused_gelu = os.environ.get("B200_FUSED_GELU", "1") != "0"
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
                dropout: Optional[bool] = None):
        """Returns (sequence_output [B*S, H] bf16, saved-or-None).  ``training`` saves activations for
        ``backward``; ``dropout`` (default: same as ``training``) applies the dropout sites."""
        B, S = input_ids.shape
        M, H, A = B * S, self.H, self.arena
        dropout = training if dropout is None else dropout
        ph = self.p_hidden if dropout else 0.0
        pa = self.p_attn if dropout else 0.0
        seed = self.next_seed() if seed is None else seed
        ids = input_ids.reshape(-1).to(torch.int32).contiguous()
        seg = None
        if self.has_type:
            seg = (token_type_ids if token_type_ids is not None else torch.zeros_like(input_ids)
                   ).reshape(-1).to(torch.int32).contiguous()
        seqlens = attention_mask.to(torch.int32).sum(dim=1, dtype=torch.int32).contiguous()
        sv = _Saved(B=B, S=S, seed=seed, p_hidden=ph, p_attn=pa, ids=ids, seg=seg, seqlens=seqlens) if training else None

        x, e, mean, rstd = K.embedding_fwd(
            ids, seg, self.w("embeddings.word_embeddings.weight"), self.w("embeddings.position_embeddings.weight"),
            self.w("embeddings.token_type_embeddings.weight") if self.has_type else None,
            self.p("embeddings.LayerNorm.weight"), self.p("embeddings.LayerNorm.bias"), S,
            p_drop=ph, seed=seed, stream=_stream(_EMB_LAYER, SITE_EMB))
        if training:
            sv.emb_sum, sv.emb_mean, sv.emb_rstd = e, mean, rstd

        ckpt = training and bool(getattr(self.bert.encoder, "_checkpoint_activations", False))
        seg_len = int(math.ceil(math.sqrt(self.L))) if ckpt else 0
        if ckpt and _use_sdpa():
            raise NotImplementedError("B200_ATTN=sdpa (library bring-up path) cannot replay its dropout under --checkpoint_activations")
        for l in range(self.L):
            if ckpt and l % seg_len == 0:
                sv.boundaries[l] = x             # --checkpoint_activations: keep segment inputs only (K27)
            x, ls, xq = self._layer_forward(l, x, seqlens, B, S, ph, pa, seed, save=training and not ckpt,
                                            xq=None if (l == 0 or (ckpt and l % seg_len == 0)) else xq)
            if ls is not None:
                sv.layers.append(ls)
        if ckpt:
            sv.seg_len = seg_len
        return x, sv

    def _layer_forward(self, l: int, x, seqlens, B: int, S: int, ph: float, pa: float, seed: int, save: bool, xq=None):
        """One post-LN transformer layer (reference: src/modeling.py:482-499) as 9 kernel launches."""
        A, H, M = self.arena, self.H, B * S
        training = save or pa > 0 or ph > 0
        pre = f"encoder.layer.{l}."
        ls = _LayerSaved() if save else None
        qkv, x_op = self._lin(l, "x", "wqkv", x, self._qkv(l, A.flat_shadow, "weight"), xq=xq, epi=K.EPI_BIAS,
                              bias=self._qkv(l, A.flat_shadow, "bias"))
        if _use_sdpa():
            ctx, lse, sd = self._sdpa_fwd(qkv, seqlens, B, S, pa, training)
            ctx_q = None
            if save:
                ls.sdpa = sd
        else:
            ctx, lse, *q = K.attention_fwd(qkv.view(B, S, 3 * H), seqlens, self.heads, p_drop=pa, seed=seed,
                                           stream=_stream(l, SITE_ATTN_PROB), fp8=self._side(f"{l}.ctx"))
            ctx = ctx.view(M, H)
            ctx_q = q[0].view(M, H) if q else None
        # keep bits of the hidden dropout leave the GEMM epilogue (1 bit per element) so that the LayerNorm backward does
        # not have to run Philox again -- bf16 path only
        keep_bits = (save and ph > 0 and not self.fp8 and H % 128 == 0
                     and os.environ.get("B200_DROP_MASK", "1") != "0")
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
        if self.fused_gelu and not self.fp8:
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
        """``d_out``: [B*S, H] bf16 gradient of the sequence output.  Accumulates every parameter
        gradient of the encoder into the arena."""
        A, H, M = self.arena, self.H, sv.B * sv.S
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
                    x, ls, xq = self._layer_forward(l, x, sv.seqlens, sv.B, sv.S, ph, pa, seed, save=True, xq=xq)
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
                                self.g("embeddings.token_type_embeddings.weight") if self.has_type else None, sv.S)
        self._join_wgrads()
        if self.fp8:                       # delayed scaling: next micro-step quantises with this one's amaxes
            self.meta.update()
            self._fp8_calibrated = True

    def _layer_backward(self, l: int, ls: _LayerSaved, d: torch.Tensor, sv: _Saved, kfac) -> torch.Tensor:
        A, H, M = self.arena, self.H, sv.B * sv.S
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
        if self.fused_gelu and not self.fp8:
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
        if ls.sdpa is not None:
            d_qkv = self._sdpa_bwd(ls.sdpa, d_ctx, sv.B, sv.S)
        else:
            d_qkv, *q = _as_tuple(K.attention_bwd(ls.qkv.view(sv.B, sv.S, 3 * H), sv.seqlens, ls.ctx.view(sv.B, sv.S, H),
                                                  d_ctx.view(sv.B, sv.S, H), ls.lse, self.heads, p_drop=pa, seed=seed,
                                                  stream=_stream(l, SITE_ATTN_PROB), fp8=self._side(f"{l}.d_qkv")))
            d_qkv = d_qkv.view(M, 3 * H)
            dqkv_q = q[0].view(M, 3 * H) if q else None
        if kfac is not None:
            for j, nm in enumerate(("query", "key", "value")):
                kfac.tap(self.prefix + pre + "attention.self." + nm, ls.x, d_qkv[:, j * H:(j + 1) * H])
        # ---- QKV projection
        K.colsum_accumulate(d_qkv, self._qkv(l, A.flat_grad, "bias"))
        d = self._lin_bwd(l, "d_qkv", "x", "wqkv", d_qkv, ls.x_op, self._qkv(l, A.flat_shadow, "weight"),
                          self._qkv(l, A.flat_grad, "weight"), dyq=dqkv_q, epi=K.EPI_ADD, res=d_pre1)
        self._wgrad_layer_done()
        return d

    # -- library attention (bring-up / bisecting aid: B200_ATTN=sdpa) ---------------------------------
    def _sdpa_fwd(self, qkv, seqlens, B, S, p, training):
        H, h = self.H, self.heads
        d = H // h
        t = qkv.view(B, S, 3, h, d)
        q, k, v = (t[:, :, i].transpose(1, 2) for i in range(3))
        mask = (torch.arange(S, device=qkv.device)[None, :] < seqlens[:, None])[:, None, None, :]
        if training:
            with torch.enable_grad():
                q, k, v = (z.detach().requires_grad_(True) for z in (q, k, v))
                o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)
            return o.detach().transpose(1, 2).reshape(B * S, H), None, (q, k, v, o)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        return o.transpose(1, 2).reshape(B * S, H), None, None

    def _sdpa_bwd(self, sd, d_ctx, B, S):
        q, k, v, o = sd
        H, h = self.H, self.heads
        go = d_ctx.view(B, S, h, H // h).transpose(1, 2)
        dq, dk, dv = torch.autograd.grad(o, (q, k, v), go)
        return torch.stack([dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2)], dim=2).reshape(B * S, 3 * H)

    # -- autograd bridge for models with ordinary torch heads (finetuning, inference) ------------------
    def encode(self, input_ids, token_type_ids, attention_mask) -> torch.Tensor:
        B, S = input_ids.shape
        training = self.bert.training and torch.is_grad_enabled()
        if not training:
            seq, _ = self.forward(input_ids, token_type_ids, attention_mask, training=False)
            out = seq.view(B, S, self.H)
        else:
            out = _EncoderFn.apply(self._hook, self, input_ids, token_type_ids, attention_mask)
        if torch.is_autocast_enabled():
            return out.to(torch.get_autocast_dtype("cuda"))
        return out.float()


class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hook, engine, input_ids, token_type_ids, attention_mask):
        seq, sv = engine.forward(input_ids, token_type_ids, attention_mask, training=True)
        ctx.engine, ctx.sv = engine, sv
        return seq.view(input_ids.size(0), input_ids.size(1), engine.H)

    @staticmethod
    def backward(ctx, d_seq):
        engine, sv = ctx.engine, ctx.sv
        engine.backward(sv, d_seq.reshape(-1, engine.H).to(torch.bfloat16).contiguous())
        ctx.sv = None
        return torch.zeros(1, device=d_seq.device), None, None, None, None


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
    if (x.is_cuda and ops.available() and H % 8 == 0 and linear.out_features <= 64 and rows >= 128
            and os.environ.get("B200_HEAD_GEMM", "1") != "0"):
        return _HeadLinearFn.apply(x, linear.weight, linear.bias)
    return linear(x)


class FusedPretrainer:
    """Forward + backward of ``BertForPreTraining`` + criterion as one kernel program.

    ``forward_backward`` returns the (unscaled) loss of the micro-batch as a device scalar and leaves the
    gradients -- multiplied by ``grad_scale`` (= loss_scale / accumulation_steps) -- accumulated in the arena.
    """

    def __init__(self, model):
        self.model = model
        self.engine: FusedEncoderEngine = model.bert.fused_engine()
        self.arena = self.engine.arena
        cfg = model.config
        self.V, self.H = cfg.vocab_size, cfg.hidden_size
        self.has_nsp = model.cls.has_nsp and model.bert.pooler is not None
        self.max_pred = int(getattr(cfg, "max_predictions_per_seq", 0)) or None
        self._loss = None
        # CUDA graphs: the micro-step is ~600 launches of static shape; replaying it as one graph removes the
        # launch gaps (~6 % of the phase-1 step).  B200_GRAPH=0 keeps the eager program.
        self.use_graphs = os.environ.get("B200_GRAPH", "1") != "0"
        self.graph_warmup = 2                 # eager calls per input signature before capturing
        self._graphs: Dict[tuple, dict] = {}
        self._seed_step: Optional[torch.Tensor] = None
        self.grad_push = False                # set by the runtime around the last micro-step (PeerComm.begin_push)
        self._cls_idx = None                  # row indices of the [CLS] tokens (NSP head)
        self._cap_stream = None               # high-priority capture stream (wgrad side-stream mode)
        self._cls_S = 0

    def _max_pred(self, labels: torch.Tensor) -> int:
        # capacity of masked positions per sequence; fixed per run so shapes stay static
        if self.max_pred is None:
            # no --max_predictions_per_seq: the capacity is the sequence length (any batch fits; the static-shape head
            # then costs S rows per sequence, so runners should always pass the flag -- data/dataset.py validates
            # pre-masked shards against it)
            self.max_pred = (labels.size(1) + 7) // 8 * 8
        return self.max_pred

    def _graph_ok(self) -> bool:
        kf = getattr(self.model.bert, "_kfac", None)
        if not self.use_graphs or _use_sdpa() or (kf is not None and getattr(kf, "capture", True)):
            return False                      # tapped micro-steps keep Python-side state; the library attention path owns its RNG
        return self.arena.device.type == "cuda"

    @torch.no_grad()
    def forward_backward(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels,
                         grad_scale: float = 1.0) -> torch.Tensor:
        """One micro-step.  After ``graph_warmup`` eager calls with the same input signature the whole kernel
        program (forward, loss, backward: ~600 launches) is captured once and replayed as ONE CUDA graph; the
        dropout seed advances through a device-side step counter inside the graph."""
        if not self._graph_ok():
            return self._program(input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels, grad_scale)
        args = (input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels)
        key = (tuple(input_ids.shape), self.model.training, next_sentence_labels is not None,
               segment_ids is not None, tuple(str(t.dtype) for t in args if t is not None),
               bool(getattr(self.model.bert.encoder, "_checkpoint_activations", False)), self.engine.fp8,
               bool(self.grad_push), bool(self.engine.wgrad_side))
        ent = self._graphs.setdefault(key, {"calls": 0})
        ent["calls"] += 1
        eng = self.engine
        if "graph" in ent and ent["grad_scale"] != float(grad_scale):
            # the loss scale is a launch constant: a GradScaler update invalidates the capture (rare); drop it
            # (and its private memory pool) and capture again right away
            for k in ("graph", "static", "loss"):
                ent.pop(k)
        if "graph" not in ent:
            if ent["calls"] <= self.graph_warmup or (eng.fp8 and not eng._fp8_calibrated):
                return self._program(*args, grad_scale)
            if self._seed_step is None:
                self._seed_step = torch.zeros(1, dtype=torch.int64, device=self.arena.device)
                ops.extension().set_seed_step(self._seed_step)
            self._max_pred(masked_lm_labels.to(torch.int32))
            static = [None if t is None else t.clone() for t in args]
            eng.prepare_step()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = K.KERNEL_LAUNCHES
            pool = next((e["graph"].pool() for e in self._graphs.values() if "graph" in e), None)
            # replays never overlap: all captures share one memory pool; thread_local: a data-loader thread that pins
            # or allocates memory while we capture must not abort the capture
            extra = {}
            if eng.wgrad_side:                # capture on a high-priority stream: the dgrad chain wins SMs over the wgrads
                if self._cap_stream is None:
                    self._cap_stream = torch.cuda.Stream(device=self.arena.device, priority=-1)
                extra["stream"] = self._cap_stream
            try:
                with torch.cuda.graph(graph, pool=pool, capture_error_mode="thread_local", **extra):
                    self._seed_step.add_(1)
                    loss = self._program(*static, grad_scale, seed=eng._seed_base)
            except Exception as e:            # e.g. an allocator / stream condition this build of torch cannot capture
                import warnings
                warnings.warn(f"CUDA-graph capture of the micro-step failed ({type(e).__name__}: {e}); "
                              "continuing with the eager kernel program")
                K.KERNEL_LAUNCHES = n0
                self.use_graphs = False
                torch.cuda.synchronize()      # nothing of the captured program ran: the accumulated gradients are intact
                return self._program(*args, grad_scale)
            ent.update(graph=graph, static=static, loss=loss, launches=K.KERNEL_LAUNCHES - n0, grad_scale=float(grad_scale))
            K.KERNEL_LAUNCHES = n0            # the capture itself ran nothing
        for dst, src in zip(ent["static"], args):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        eng.prepare_step()
        ent["graph"].replay()
        K._count(ent["launches"])
        return ent["loss"]

    @torch.no_grad()
    def _program(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels,
                 grad_scale: float = 1.0, seed: Optional[int] = None) -> torch.Tensor:
        eng, A, H, V = self.engine, self.arena, self.H, self.V
        B, S = input_ids.shape
        M = B * S
        seq, sv = eng.forward(input_ids, segment_ids, input_mask, training=True, seed=seed, dropout=self.model.training)
        labels = masked_lm_labels.to(torch.int32).contiguous()
        mp = self._max_pred(labels)
        idx, tgt, count = K.mlm_compact(labels, mp)
        loss = torch.zeros(1, dtype=torch.float32, device=seq.device)

        # ---- MLM head forward (masked rows only)
        rows = K.gather_rows(seq, idx)
        t_pre = K.gemm(rows, A.shadow("cls.predictions.transform.dense_act.weight"), epi=K.EPI_BIAS,
                       bias=A.shadow("cls.predictions.transform.dense_act.bias"))
        t_act = K.gelu_fwd(t_pre)
        t_ln, t_mean, t_rstd = K.layer_norm_fwd(t_act, A.view("cls.predictions.transform.LayerNorm.weight"),
                                                A.view("cls.predictions.transform.LayerNorm.bias"))
        emb_w = eng.w("embeddings.word_embeddings.weight")            # tied decoder weight [V, H]
        logits = K.gemm(t_ln, emb_w, epi=K.EPI_BIAS, bias=A.shadow("cls.predictions.bias"))
        K.softmax_ce_(logits, tgt, count, grad_scale, loss)            # logits <- dlogits

        # ---- MLM head backward
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
            pw = A.shadow(eng.prefix + "pooler.dense_act.weight")
            if self._cls_idx is None or self._cls_idx.numel() != B or self._cls_S != S:
                self._cls_idx = (torch.arange(B, device=seq.device, dtype=torch.int32) * S).contiguous()
                self._cls_S = S
            cls_tok = K.gather_rows(seq, self._cls_idx)                                        # [B, H] bf16
            pooled = K.gemm(cls_tok, pw, epi=K.EPI_BIAS_TANH, bias=A.shadow(eng.prefix + "pooler.dense_act.bias"))
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
            d_cls = K.gemm(d_z, pw, layout=K.NN)
            d_seq.view(B, S, H)[:, 0] += d_cls

        eng.backward(sv, d_seq)
        return loss.squeeze(0) if loss.dim() else loss
