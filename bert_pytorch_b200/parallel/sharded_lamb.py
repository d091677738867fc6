"""Partitioned ("ZeRO-1 style") LAMB fused with the gradient reduction -- the *algorithm*,
written against the :class:`Comm` interface so it runs on gloo / the in-process fake and is
the executable specification for the sm_90a peer-memory kernel (ops/csrc/comm.cu;
SURVEY.md 5.8 items 3-4, 7.5 hard part #3).

Per optimizer step, on a flat gradient arena of ``numel`` elements split into one
contiguous shard per rank:

  phase A  reduce-scatter(grad) -> x 1/(world * loss_scale) -> inf/nan flag
           -> partial sum of squares (global grad norm)
  sync 1   all-reduce [found_inf, sum g^2]        (2 floats)
  phase B  skip everything if found_inf; clip divisor from the global norm;
           moments m, v; update u = m^/(sqrt(v^)+eps) + wd p on the shard;
           per-tensor partial ||p||^2, ||u||^2 (tensors may straddle shard boundaries
           -> segmented reduction keyed by the slot table)
  sync 2   all-reduce the [T, 2] norm table
  phase C  p -= lr * trust_ratio(tensor) * u on the shard; all-gather(params)

The reference never shards optimizer state (every rank runs the whole FusedLAMB after
DDP's all-reduce, run_pretraining.py:405-417); results here are numerically the same
update (identical up to fp32 summation order).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .comm import Comm


def slot_segments(offsets: Sequence[int], numels: Sequence[int], lo: int, hi: int) -> List[Tuple[int, int, int]]:
    """(slot index, a, b) for every slot intersecting [lo, hi); [a, b) in arena coordinates."""
    out = []
    for i, (o, n) in enumerate(zip(offsets, numels)):
        a, b = max(o, lo), min(o + n, hi)
        if a < b:
            out.append((i, a, b))
    return out


class ShardedLamb:
    """State: this rank's slices of exp_avg / exp_avg_sq (+ the fp32 master shard)."""

    def __init__(self, arena, comm: Comm, *, lr: float, betas=(0.9, 0.999), eps: float = 1e-6,
                 weight_decay: float = 0.01, max_grad_norm: float = 1.0, bias_correction: bool = True,
                 grad_averaging: bool = True, granule: int = 2048):
        self.arena, self.comm = arena, comm
        self.lr, self.betas, self.eps = lr, betas, eps
        self.weight_decay, self.max_grad_norm = weight_decay, max_grad_norm
        self.bias_correction, self.grad_averaging = bias_correction, grad_averaging
        self.lo, self.hi = arena.shard_bounds(comm.world_size, comm.rank, granule)
        n = self.hi - self.lo
        dev = arena.flat_param.device
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        self.g = torch.zeros(n, dtype=torch.float32, device=dev)
        self.step_count = 0
        self.offsets = [s.offset for s in arena.slots]
        self.numels = [s.numel for s in arena.slots]
        self.decay = [s.decay for s in arena.slots]
        self.segments = slot_segments(self.offsets, self.numels, self.lo, self.hi)
        self.last_grad_norm = 0.0
        self.last_skipped = False

    @torch.no_grad()
    def step(self, loss_scale: float = 1.0, lr: Optional[float] = None) -> bool:
        """Returns True if the update was applied (False = overflow, step skipped everywhere)."""
        A, C = self.arena, self.comm
        lr = self.lr if lr is None else lr
        lo, hi = self.lo, self.hi
        # ---- phase A
        C.reduce_scatter(A.flat_grad, self.g, lo, hi)
        g = self.g[: hi - lo]
        g.mul_(1.0 / (C.world_size * loss_scale))
        finite = bool(torch.isfinite(g).all())
        stats = torch.tensor([0.0 if finite else 1.0, float((g.double() ** 2).sum()) if finite else 0.0],
                             dtype=torch.float64, device=g.device)
        C.all_reduce_(stats)                                           # ---- sync 1
        A.flat_grad.zero_()
        if float(stats[0]) > 0:
            self.last_skipped = True
            return False
        self.last_skipped = False
        gnorm = math.sqrt(float(stats[1]))
        self.last_grad_norm = gnorm
        clip = max(gnorm / self.max_grad_norm, 1.0) if self.max_grad_norm and self.max_grad_norm > 0 else 1.0
        # ---- phase B
        self.step_count += 1
        b1, b2 = self.betas
        bc1 = 1.0 - b1 ** self.step_count if self.bias_correction else 1.0
        bc2 = 1.0 - b2 ** self.step_count if self.bias_correction else 1.0
        b3 = 1.0 - b1 if self.grad_averaging else 1.0
        g.div_(clip)
        p = A.flat_param[lo:hi]
        self.m.mul_(b1).add_(g, alpha=b3)
        self.v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        u = (self.m / bc1) / ((self.v / bc2).sqrt() + self.eps)
        norms = torch.zeros(len(self.offsets), 2, dtype=torch.float64, device=g.device)
        for i, a, b in self.segments:
            sl = slice(a - lo, b - lo)
            if self.decay[i] and self.weight_decay != 0:
                u[sl] += self.weight_decay * p[sl]
                norms[i, 0] = (p[sl].double() ** 2).sum()
                norms[i, 1] = (u[sl].double() ** 2).sum()
        C.all_reduce_(norms)                                           # ---- sync 2
        # ---- phase C
        for i, a, b in self.segments:
            sl = slice(a - lo, b - lo)
            ratio = lr
            if self.decay[i] and self.weight_decay != 0:
                pn, un = math.sqrt(float(norms[i, 0])), math.sqrt(float(norms[i, 1]))
                if pn > 0 and un > 0:
                    ratio = lr * pn / un
            p[sl].add_(u[sl], alpha=-ratio)
        C.all_gather_into(A.flat_param, p.clone(), lo, hi)
        A.refresh_shadow()
        return True

    # -- checkpointing: gather the shards into the per-parameter layout ---------------------
    def full_state(self) -> Dict[str, torch.Tensor]:
        A, C = self.arena, self.comm
        out = {}
        for key, shard in (("exp_avg", self.m), ("exp_avg_sq", self.v)):
            full = torch.zeros_like(A.flat_param)
            C.all_gather_into(full, shard, self.lo, self.hi)
            out[key] = full
        return out
