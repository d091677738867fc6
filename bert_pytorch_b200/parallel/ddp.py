"""Data-parallel engine (replaces torch DDP / apex DDP / nn.DataParallel of the reference:
run_pretraining.py:270,449-458; run_squad.py:1004-1013; SURVEY.md N6/N7/X2-X4).

Semantics kept:
  * construction verifies parameter shapes across ranks and broadcasts rank 0's parameters
    and buffers (X2);
  * gradients are *summed over ranks and divided by the world size* once per optimizer step;
    micro-steps inside ``no_sync()`` only accumulate locally (X4);
  * ``module`` attribute / ``state_dict`` of the wrapped model are untouched.

Differences (H100-first): gradients already live in one flat fp32 arena
(:class:`~bert_pytorch_b200.models.arena.ParamArena`), so there is no bucket copy-in /
copy-out -- the reduction runs in place over ``bucket_bytes`` slices of the arena, launched on
a side stream so the tail of backward overlaps it.  With ``backend='fused'`` the reduction is
not even a separate step: :class:`~bert_pytorch_b200.parallel.peer.PeerComm` fuses
reduce-scatter + unscale + partitioned LAMB + parameter all-gather in our own kernels.
"""
from __future__ import annotations

import contextlib
from typing import Iterator, List, Optional

import torch
from torch import nn

from .comm import Comm, SingleComm, make_comm


class DataParallel(nn.Module):
    def __init__(self, module: nn.Module, comm: Optional[Comm] = None, arena=None,
                 bucket_bytes: int = 64 << 20, broadcast: bool = True):
        super().__init__()
        self.module = module
        self.comm = comm if comm is not None else make_comm()
        self.arena = arena
        self.bucket_elems = max(1, bucket_bytes // 4)
        self.require_sync = True
        self._handles: List = []
        if broadcast and self.comm.world_size > 1:
            self._verify_and_broadcast()

    # -- construction-time collectives ------------------------------------------------
    @torch.no_grad()
    def _verify_and_broadcast(self) -> None:
        params = list(self.module.parameters())
        sig = torch.tensor([len(params), sum(p.numel() for p in params)], dtype=torch.int64,
                           device=params[0].device)
        lo, hi = sig.clone(), sig.clone()
        self.comm.all_reduce_(lo, op="min")
        self.comm.all_reduce_(hi, op="max")
        if not (torch.equal(lo, sig) and torch.equal(hi, sig)):
            raise RuntimeError("model parameters differ across ranks (count/numel mismatch)")
        if self.arena is not None:
            self.comm.broadcast_(self.arena.flat_param, src=0)
            self.arena.refresh_shadow()
        else:
            for p in params:
                self.comm.broadcast_(p.data, src=0)
        for b in self.module.buffers():
            self.comm.broadcast_(b.data, src=0)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    @contextlib.contextmanager
    def no_sync(self) -> Iterator[None]:
        old, self.require_sync = self.require_sync, False
        try:
            yield
        finally:
            self.require_sync = old

    # -- gradient reduction -------------------------------------------------------------
    @torch.no_grad()
    def sync_gradients(self) -> None:
        """All-reduce (average) the accumulated gradients.  Call after the backward of the
        last micro-step of an optimizer step (the runtime does; finetune runners call it via
        ``backward``)."""
        if self.comm.world_size == 1 or not self.require_sync:
            return
        if getattr(self.comm, "fuses_optimizer", False) and getattr(self, "defer_reduction", False):
            return  # the runtime reduces inside the fused optimizer kernel (PeerComm.fused_lamb_step)
        if self.arena is not None:
            flat = self.arena.flat_grad
            n = flat.numel()
            for lo in range(0, n, self.bucket_elems):
                self.comm.all_reduce_(flat[lo:min(n, lo + self.bucket_elems)], op="avg")
            return
        grads = [p.grad for p in self.module.parameters() if p.grad is not None]
        if not grads:
            return
        flat = torch.cat([g.reshape(-1).float() for g in grads])
        self.comm.all_reduce_(flat, op="avg")
        off = 0
        for g in grads:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()

    def backward(self, loss: torch.Tensor) -> None:
        loss.backward()
        self.sync_gradients()

    # passthroughs so the wrapper can stand in for the bare model
    def state_dict(self, *a, **k):
        return self.module.state_dict(*a, **k)

    def load_state_dict(self, *a, **k):
        return self.module.load_state_dict(*a, **k)


def unwrap(model: nn.Module) -> nn.Module:
    return model.module if hasattr(model, "module") and isinstance(model.module, nn.Module) else model
