"""Flat parameter / gradient arena.

All parameters of a model live in ONE contiguous fp32 buffer (``flat_param``), their
gradients in a second one (``flat_grad``), the LAMB/Adam moments in two more, and -- on
CUDA -- a bf16 shadow copy of the weights that the tensor-core kernels read.  The
``nn.Parameter`` objects keep their reference names (state-dict compatibility, SURVEY.md
2.5.3) but become *views* into the arena, and ``param.grad`` is a persistent view into
``flat_grad``.

Why (H100-first, SURVEY.md 7.1 / 5.8):
  * the optimizer is three launches over contiguous memory instead of 398 tensors,
  * the gradient all-reduce (NCCL baseline or the fused peer-memory kernel) and the
    partitioned LAMB update work on plain ``[offset, offset+n)`` shards,
  * wgrad kernels accumulate straight into the arena (no per-parameter add kernels),
  * Q/K/V weights (and biases) of a layer are adjacent so one ``[3H, H]`` GEMM serves the
    three projections without copies while the state dict still exposes them separately.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

ALIGN = 64  # elements; 256 B in fp32, 128 B in bf16 (TMA needs 16 B)

NO_DECAY_KEYS = ("bias", "gamma", "beta", "LayerNorm")  # run_pretraining.py:279


@dataclass
class Slot:
    name: str
    offset: int
    numel: int
    shape: Tuple[int, ...]
    decay: bool
    group: int = 0     # optimizer param-group index


def _ordered_named_parameters(model: nn.Module) -> List[Tuple[str, nn.Parameter]]:
    """named_parameters() with each layer's q/k/v weights, then q/k/v biases, adjacent."""
    named = list(model.named_parameters())   # tied parameters appear once
    by_name = dict(named)
    out: List[Tuple[str, nn.Parameter]] = []
    done = set()
    for name, p in named:
        if name in done:
            continue
        if name.endswith("attention.self.query.weight"):
            base = name[: -len("query.weight")]
            for suffix in ("query.weight", "key.weight", "value.weight",
                           "query.bias", "key.bias", "value.bias"):
                n = base + suffix
                if n in by_name and n not in done:
                    out.append((n, by_name[n]))
                    done.add(n)
            continue
        out.append((name, p))
        done.add(name)
    return out


class ParamArena:
    def __init__(self, model: nn.Module, device: Optional[torch.device] = None,
                 no_decay_keys: Sequence[str] = NO_DECAY_KEYS, shadow_dtype: Optional[torch.dtype] = None):
        named = _ordered_named_parameters(model)
        if device is None:
            device = named[0][1].device
        self.device = torch.device(device)
        self.slots: List[Slot] = []
        self.params: List[nn.Parameter] = []
        off = 0
        prev_qkv = False
        for name, p in named:
            is_qkv = ".attention.self." in name
            if not (is_qkv and prev_qkv):           # keep q/k/v blocks gap-free
                off = (off + ALIGN - 1) // ALIGN * ALIGN
            prev_qkv = is_qkv
            decay = not any(k in name for k in no_decay_keys)
            self.slots.append(Slot(name, off, p.numel(), tuple(p.shape), decay))
            self.params.append(p)
            off += p.numel()
        self.numel = (off + ALIGN - 1) // ALIGN * ALIGN
        self.flat_param = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.flat_grad = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.exp_avg: Optional[torch.Tensor] = None
        self.exp_avg_sq: Optional[torch.Tensor] = None
        if shadow_dtype is None and self.device.type == "cuda":
            shadow_dtype = torch.bfloat16
        self.shadow_dtype = shadow_dtype
        self.flat_shadow = (torch.zeros(self.numel, dtype=shadow_dtype, device=self.device)
                            if shadow_dtype is not None else None)
        self.by_name: Dict[str, Slot] = {s.name: s for s in self.slots}
        self.version = 0          # bumped whenever the weights change (consumers cache derived copies, e.g. fp8)
        with torch.no_grad():
            for s, p in zip(self.slots, self.params):
                view = self.flat_param[s.offset:s.offset + s.numel].view(s.shape)
                view.copy_(p.detach().to(device=self.device, dtype=torch.float32))
                p.data = view
                p.grad = self.flat_grad[s.offset:s.offset + s.numel].view(s.shape)
        self._tables = None
        self._opt_tables = None
        import weakref
        ref = weakref.ref(self)
        for mod in model.modules():
            object.__setattr__(mod, "_arena_ref", ref)
        self.refresh_shadow()

    # -- views ----------------------------------------------------------------
    def view(self, name: str, flat: Optional[torch.Tensor] = None) -> torch.Tensor:
        s = self.by_name[name]
        buf = self.flat_param if flat is None else flat
        return buf[s.offset:s.offset + s.numel].view(s.shape)

    def span(self, first: str, last: str, flat: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
        """One view covering the adjacent slots ``first`` .. ``last`` (e.g. the fused QKV weight)."""
        a, b = self.by_name[first], self.by_name[last]
        n = b.offset + b.numel - a.offset
        return flat[a.offset:a.offset + n].view(*shape)

    def shadow(self, name: str) -> torch.Tensor:
        return self.view(name, self.flat_shadow)

    def grad(self, name: str) -> torch.Tensor:
        return self.view(name, self.flat_grad)

    @torch.no_grad()
    def refresh_shadow(self) -> None:
        sync = getattr(self, "_master_sync", None)
        if sync is not None:          # peer-memory backend with a shard-local fp32 master: complete it first
            sync()
        self.version += 1
        if self.flat_shadow is not None:
            self.flat_shadow.copy_(self.flat_param)

    def rebind(self) -> None:
        """Re-point ``param.data`` / ``param.grad`` at the arena (after ``load_state_dict``
        replaced tensors, or after something set ``grad = None``)."""
        with torch.no_grad():
            for s, p in zip(self.slots, self.params):
                view = self.flat_param[s.offset:s.offset + s.numel].view(s.shape)
                if p.data.data_ptr() != view.data_ptr():
                    view.copy_(p.data.to(view.dtype))
                    p.data = view
                if p.grad is None or p.grad.data_ptr() != self.flat_grad[s.offset:].data_ptr():
                    p.grad = self.flat_grad[s.offset:s.offset + s.numel].view(s.shape)
        self.refresh_shadow()

    @torch.no_grad()
    def zero_grad(self) -> None:
        self.flat_grad.zero_()
        for s, p in zip(self.slots, self.params):
            if p.grad is None:
                p.grad = self.flat_grad[s.offset:s.offset + s.numel].view(s.shape)

    # -- optimizer binding ----------------------------------------------------------
    def bind_optimizer(self, optimizer) -> None:
        """Give ``optimizer`` arena-backed state: ``state[p]['exp_avg'/'exp_avg_sq']`` become
        views into two flat moment buffers so ``optimizer.state_dict()`` keeps the per-parameter
        layout of apex FusedLAMB/FusedAdam while the kernels see contiguous memory."""
        if self.exp_avg is None:
            self.exp_avg = torch.zeros_like(self.flat_param)
            self.exp_avg_sq = torch.zeros_like(self.flat_param)
        group_of = {}
        for gi, g in enumerate(optimizer.param_groups):
            for p in g["params"]:
                group_of[id(p)] = gi
        for s, p in zip(self.slots, self.params):
            if id(p) not in group_of:
                raise ValueError(f"parameter {s.name} is not managed by the optimizer")
            s.group = group_of[id(p)]
            s.decay = float(optimizer.param_groups[s.group].get("weight_decay", 0.0)) != 0.0
            st = optimizer.state[p]
            st["exp_avg"] = self.exp_avg[s.offset:s.offset + s.numel].view(s.shape)
            st["exp_avg_sq"] = self.exp_avg_sq[s.offset:s.offset + s.numel].view(s.shape)
        optimizer._arena = self
        self._tables = None
        self._opt_tables = None

    def adopt_optimizer_state(self, optimizer) -> None:
        """After ``optimizer.load_state_dict`` the moments are fresh tensors: copy them into
        the arena and re-install the views."""
        with torch.no_grad():
            for s, p in zip(self.slots, self.params):
                st = optimizer.state.get(p, {})
                for key, flat in (("exp_avg", self.exp_avg), ("exp_avg_sq", self.exp_avg_sq)):
                    view = flat[s.offset:s.offset + s.numel].view(s.shape)
                    if key in st and st[key].data_ptr() != view.data_ptr():
                        view.copy_(st[key].to(device=view.device, dtype=view.dtype))
                    st[key] = view
                optimizer.state[p] = st

    def tables(self):
        """Device tensors describing the slots for the multi-tensor kernels:
        (offsets int64 [T+1 semantics via numel], numels int64, decay flag int32, group int32)."""
        if self._tables is None:
            dev = self.device
            self._tables = dict(
                offsets=torch.tensor([s.offset for s in self.slots], dtype=torch.int64, device=dev),
                numels=torch.tensor([s.numel for s in self.slots], dtype=torch.int64, device=dev),
                decay=torch.tensor([1 if s.decay else 0 for s in self.slots], dtype=torch.int32, device=dev),
                group=torch.tensor([s.group for s in self.slots], dtype=torch.int32, device=dev),
            )
        return self._tables

    # -- fused optimizer entry points (CUDA) ------------------------------------------
    def fused_optimizer_ok(self) -> bool:
        if self.device.type != "cuda":
            return False
        from .. import ops
        return ops.available()

    def unscale_(self, inv_scale: torch.Tensor, found_inf: torch.Tensor) -> None:
        from .. import ops
        ops.flat_unscale_(self.flat_grad, inv_scale, found_inf)

    def fused_lamb_step(self, optimizer, inv_scale=None, found_inf=None) -> None:
        from .. import ops
        self.version += 1
        ops.arena_lamb_step(self, optimizer, inv_scale, found_inf)

    def fused_adam_step(self, optimizer, inv_scale=None, found_inf=None) -> None:
        from .. import ops
        self.version += 1
        ops.arena_adam_step(self, optimizer, inv_scale, found_inf)

    # -- sharding helpers (partitioned optimizer / reduce-scatter) ----------------------
    def shard_bounds(self, world_size: int, rank: int, granule: int = 2048) -> Tuple[int, int]:
        """[lo, hi) of rank's contiguous shard; shard sizes are multiples of ``granule``
        elements (kernel tile) except the last."""
        per = (self.numel + world_size - 1) // world_size
        per = (per + granule - 1) // granule * granule
        lo = min(rank * per, self.numel)
        return lo, min(lo + per, self.numel)
