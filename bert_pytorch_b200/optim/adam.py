"""Adam family.

* :class:`Adam` -- contract of apex ``FusedAdam`` (AdamW-style decoupled decay,
  optional bias correction; both reference call sites pass ``bias_correction=False``:
  run_squad.py:982-988, run_ner.py:243-244).  Fused multi-tensor sm_90a kernel when the
  parameters live in a ParamArena, pure torch otherwise.
* :class:`BertAdam` -- src/optimization.py:64-174: Adam without bias correction,
  decoupled decay, per-parameter gradient clipping and a built-in warm-up schedule
  (the deprecated ``add_(Number, Tensor)`` calls of the reference, Q27, are gone).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch.optim import Optimizer

from .schedulers import SCHEDULES


class Adam(Optimizer):
    def __init__(self, params, lr: float = 1e-3, bias_correction: bool = True, betas=(0.9, 0.999),
                 eps: float = 1e-8, adam_w_mode: bool = True, weight_decay: float = 0.0,
                 amsgrad: bool = False, set_grad_none: bool = True):
        if amsgrad:
            raise RuntimeError("Adam here does not support the AMSGrad variant")
        defaults = dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps,
                        weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.adam_w_mode = bool(adam_w_mode)
        self.set_grad_none = set_grad_none
        self._arena = None

    def zero_grad(self, set_to_none: Optional[bool] = None) -> None:
        if self._arena is not None:
            self._arena.zero_grad()
            return
        super().zero_grad(set_to_none=self.set_grad_none if set_to_none is None else set_to_none)

    @torch.no_grad()
    def step(self, closure=None, *, inv_scale: Optional[torch.Tensor] = None,
             found_inf: Optional[torch.Tensor] = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._arena is not None and self._arena.fused_optimizer_ok():
            self._arena.fused_adam_step(self, inv_scale=inv_scale, found_inf=found_inf)
            return loss
        if found_inf is not None and float(found_inf) != 0.0:
            return loss
        for group in self.param_groups:
            group["step"] = int(group.get("step", 0)) + 1
            step = group["step"]
            b1, b2 = group["betas"]
            bc1 = 1.0 - b1 ** step if group["bias_correction"] else 1.0
            bc2 = 1.0 - b2 ** step if group["bias_correction"] else 1.0
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad.float()
                if inv_scale is not None:
                    g = g * inv_scale.to(g.dtype)
                st = self.state[p]
                if "exp_avg" not in st:
                    st["exp_avg"] = torch.zeros_like(p, dtype=torch.float32)
                    st["exp_avg_sq"] = torch.zeros_like(p, dtype=torch.float32)
                pf = p.float()
                if not self.adam_w_mode and group["weight_decay"] != 0:
                    g = g + group["weight_decay"] * pf
                m, v = st["exp_avg"], st["exp_avg_sq"]
                m.mul_(b1).add_(g, alpha=1.0 - b1)
                v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
                update = (m / bc1) / ((v / bc2).sqrt() + group["eps"])
                if self.adam_w_mode and group["weight_decay"] != 0:
                    update = update + group["weight_decay"] * pf
                p.add_(update.to(p.dtype), alpha=-group["lr"])
        return loss

    def load_state_dict(self, state_dict) -> None:
        super().load_state_dict(state_dict)
        if self._arena is not None:
            self._arena.adopt_optimizer_state(self)


FusedAdam = Adam


class BertAdam(Optimizer):
    def __init__(self, params, lr: float, warmup: float = -1, t_total: int = -1,
                 schedule: str = "warmup_linear", b1: float = 0.9, b2: float = 0.999,
                 e: float = 1e-6, weight_decay: float = 0.01, max_grad_norm: float = 1.0):
        if lr < 0.0:
            raise ValueError(f"invalid learning rate {lr}")
        if schedule not in SCHEDULES:
            raise ValueError(f"invalid schedule {schedule}")
        if not 0.0 <= warmup < 1.0 and warmup != -1:
            raise ValueError(f"invalid warmup {warmup}: should be in [0, 1) or -1")
        for name, b in (("b1", b1), ("b2", b2)):
            if not 0.0 <= b < 1.0:
                raise ValueError(f"invalid {name} {b}: should be in [0, 1)")
        if e < 0.0:
            raise ValueError(f"invalid epsilon {e}")
        super().__init__(params, dict(lr=lr, schedule=schedule, warmup=warmup, t_total=t_total,
                                      b1=b1, b2=b2, e=e, weight_decay=weight_decay,
                                      max_grad_norm=max_grad_norm))

    def _scheduled_lr(self, group, step: int) -> float:
        if group["t_total"] != -1:
            return group["lr"] * SCHEDULES[group["schedule"]](step / group["t_total"], group["warmup"])
        return group["lr"]

    def get_lr(self):
        out = []
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state[p]
                if not st:
                    return [0.0]
                out.append(self._scheduled_lr(group, st["step"]))
        return out

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                if g.is_sparse:
                    raise RuntimeError("BertAdam does not support sparse gradients")
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["next_m"] = torch.zeros_like(p)
                    st["next_v"] = torch.zeros_like(p)
                if group["max_grad_norm"] > 0:
                    torch.nn.utils.clip_grad_norm_(p, group["max_grad_norm"])
                m, v = st["next_m"], st["next_v"]
                m.mul_(group["b1"]).add_(g, alpha=1.0 - group["b1"])
                v.mul_(group["b2"]).addcmul_(g, g, value=1.0 - group["b2"])
                update = m / (v.sqrt() + group["e"])
                if group["weight_decay"] > 0.0:
                    update = update + group["weight_decay"] * p
                p.add_(update, alpha=-self._scheduled_lr(group, st["step"]))
                st["step"] += 1
        arena = getattr(self, "_arena", None)
        if arena is not None:               # parameters are arena views: the bf16 shadow (and cached fp8 copies) follow
            arena.refresh_shadow()
        return loss

    def attach_arena(self, arena) -> None:
        """Parameters / gradients live in a :class:`ParamArena`: ``zero_grad`` must zero the arena in place (the
        default ``set_to_none=True`` would detach ``p.grad`` from the buffer the data-parallel reduction and the fused
        engine use) and every step refreshes the bf16 shadow the tensor-core kernels read (ADVICE r1, high)."""
        self._arena = arena

    def zero_grad(self, set_to_none: Optional[bool] = None) -> None:
        arena = getattr(self, "_arena", None)
        if arena is not None:
            arena.zero_grad()
            return
        super().zero_grad() if set_to_none is None else super().zero_grad(set_to_none=set_to_none)
