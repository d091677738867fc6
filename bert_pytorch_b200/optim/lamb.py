"""LAMB with the behavioural contract of apex ``FusedLAMB`` as the reference uses it
(run_pretraining.py:295-296 passes only ``lr``; SURVEY.md N1/O3):

  betas (0.9, 0.999), eps 1e-6, bias_correction, AdamW-style decoupled decay,
  grad_averaging, ``max_grad_norm=1.0`` global-norm clipping folded into the update,
  trust ratio only where weight_decay != 0 (``use_nvlamb=False``), one ``step``
  counter per param group (read by the LR schedulers), per-parameter state
  ``exp_avg`` / ``exp_avg_sq``.

Two execution paths share this class:
  * the pure-torch path below (CPU, gloo runs, and the numerics oracle for tests);
  * the sm_90a multi-tensor kernels (ops/csrc/optim.cu) when the parameters live in a
    :class:`~bert_pytorch_b200.models.arena.ParamArena` on a CUDA device -- one pass
    for the global grad norm (+ unscale + inf/nan flag), one for moments/update/
    per-tensor norms, one for the trust-ratio apply that also refreshes the bf16
    shadow weights and zeroes the gradient arena.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
from torch.optim import Optimizer


def lamb_reference_step(params: List[torch.Tensor], grads: List[torch.Tensor],
                        exp_avgs: List[torch.Tensor], exp_avg_sqs: List[torch.Tensor], *,
                        lr: float, beta1: float, beta2: float, eps: float, weight_decay: float,
                        step: int, bias_correction: bool, grad_averaging: bool,
                        clip_divisor: float, adam_w_mode: bool = True,
                        use_nvlamb: bool = False) -> None:
    """One LAMB update for one param group, in fp32, in place.  ``clip_divisor`` is
    ``max(global_grad_norm / max_grad_norm, 1)`` computed over *all* groups."""
    bc1 = 1.0 - beta1 ** step if bias_correction else 1.0
    bc2 = 1.0 - beta2 ** step if bias_correction else 1.0
    beta3 = 1.0 - beta1 if grad_averaging else 1.0
    for p, g, m, v in zip(params, grads, exp_avgs, exp_avg_sqs):
        g = g.float() / clip_divisor
        pf = p.float()
        if not adam_w_mode and weight_decay != 0:
            g = g + weight_decay * pf
        m.mul_(beta1).add_(g, alpha=beta3)
        v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
        update = (m / bc1) / ((v / bc2).sqrt() + eps)
        if adam_w_mode and weight_decay != 0:
            update = update + weight_decay * pf
        ratio = lr
        if use_nvlamb or weight_decay != 0:
            pn = float(pf.norm())
            un = float(update.norm())
            if pn > 0 and un > 0:
                ratio = lr * pn / un
        p.add_(update.to(p.dtype), alpha=-ratio)


class Lamb(Optimizer):
    def __init__(self, params, lr: float = 1e-3, bias_correction: bool = True,
                 betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.01,
                 amsgrad: bool = False, adam_w_mode: bool = True, grad_averaging: bool = True,
                 set_grad_none: bool = True, max_grad_norm: float = 1.0, use_nvlamb: bool = False):
        if amsgrad:
            raise RuntimeError("LAMB does not support the AMSGrad variant")
        defaults = dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps,
                        weight_decay=weight_decay, grad_averaging=grad_averaging,
                        max_grad_norm=max_grad_norm)
        super().__init__(params, defaults)
        self.adam_w_mode = bool(adam_w_mode)
        self.set_grad_none = set_grad_none
        self.use_nvlamb = use_nvlamb
        self._arena = None  # set by ParamArena.bind_optimizer
        #: device scalars of the last fused step (global grad norm, found_inf)
        self.last_grad_norm: Optional[torch.Tensor] = None

    # -- plumbing -----------------------------------------------------------
    def zero_grad(self, set_to_none: Optional[bool] = None) -> None:
        if self._arena is not None:
            self._arena.zero_grad()
            return
        super().zero_grad(set_to_none=self.set_grad_none if set_to_none is None else set_to_none)

    def _ensure_state(self, p: torch.Tensor) -> dict:
        st = self.state[p]
        if "exp_avg" not in st:
            st["exp_avg"] = torch.zeros_like(p, dtype=torch.float32)
            st["exp_avg_sq"] = torch.zeros_like(p, dtype=torch.float32)
        return st

    def global_grad_norm(self) -> float:
        sq = 0.0
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None:
                    sq += float(p.grad.float().pow(2).sum())
        return math.sqrt(sq)

    # -- step -----------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None, *, inv_scale: Optional[torch.Tensor] = None,
             found_inf: Optional[torch.Tensor] = None):
        """``inv_scale`` / ``found_inf`` are the GradScaler's device scalars; when given
        to the fused path the unscale and the overflow skip happen inside the kernels
        with no host synchronisation."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._arena is not None and self._arena.fused_optimizer_ok():
            self._arena.fused_lamb_step(self, inv_scale=inv_scale, found_inf=found_inf)
            return loss

        if inv_scale is not None:  # generic path: unscale eagerly
            for group in self.param_groups:
                for p in group["params"]:
                    if p.grad is not None:
                        p.grad.mul_(inv_scale.to(p.grad.dtype))
        if found_inf is not None and float(found_inf) != 0.0:
            return loss
        gnorm = self.global_grad_norm()
        for group in self.param_groups:
            mg = group["max_grad_norm"]
            clip = max(gnorm / mg, 1.0) if (mg is not None and mg > 0) else 1.0
            group["step"] = int(group.get("step", 0)) + 1
            ps, gs, ms, vs = [], [], [], []
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("LAMB does not support sparse gradients")
                st = self._ensure_state(p)
                ps.append(p); gs.append(p.grad); ms.append(st["exp_avg"]); vs.append(st["exp_avg_sq"])
            b1, b2 = group["betas"]
            lamb_reference_step(ps, gs, ms, vs, lr=group["lr"], beta1=b1, beta2=b2, eps=group["eps"],
                                weight_decay=group["weight_decay"], step=group["step"],
                                bias_correction=bool(group["bias_correction"]),
                                grad_averaging=bool(group["grad_averaging"]), clip_divisor=clip,
                                adam_w_mode=self.adam_w_mode, use_nvlamb=self.use_nvlamb)
        self.last_grad_norm = torch.tensor(gnorm)
        return loss

    def load_state_dict(self, state_dict) -> None:
        """Tolerates the extra keys the resume path injects (``step`` inside the
        per-param state, ``t_total`` / ``warmup`` in the groups --
        run_pretraining.py:300-308)."""
        super().load_state_dict(state_dict)
        for st in self.state.values():
            for k in ("exp_avg", "exp_avg_sq"):
                if k in st and st[k].dtype != torch.float32:
                    st[k] = st[k].float()
        if self._arena is not None:
            self._arena.adopt_optimizer_state(self)


#: apex-compatible name
FusedLAMB = Lamb
