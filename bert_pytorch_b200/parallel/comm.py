"""Communication backends behind one small interface.

* :class:`TorchComm`  -- torch.distributed process group: ``nccl`` (baseline / cold paths /
  multi-node) or ``gloo`` (the CPU plumbing configuration).  Parity: the reference only ever
  calls NCCL through torch.distributed (run_pretraining.py:185; SURVEY.md 2.3/5.8).
* :class:`FakeComm`   -- N ranks inside one process sharing Python state (threads +
  barriers).  Lets the partitioned all-reduce+LAMB *algorithm* (shard bounds, two-phase
  norms, inf-skip agreement) be verified bit-for-bit on a box with no GPU and no network.
* :class:`bert_pytorch_b200.parallel.peer.PeerComm` -- the product path: CUDA peer memory
  (symmetric buffers mapped into every rank) driven by our own sm_90a kernels; no NCCL on
  the gradient path.

Every backend offers: all_reduce_ (sum / avg / max), reduce_scatter (contiguous shards),
all_gather_into, broadcast_, barrier.
"""
from __future__ import annotations

import threading
from typing import Dict, List, Optional

import torch
import torch.distributed as dist


class Comm:
    rank: int = 0
    world_size: int = 1
    name: str = "single"

    def all_reduce_(self, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        return t

    def all_reduce_many_(self, tensors, op: str = "sum") -> None:
        """In-place all-reduce of a list of tensors (backends may pack them into one transfer)."""
        for t in tensors:
            self.all_reduce_(t, op=op)

    def reduce_scatter(self, full: torch.Tensor, out: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
        """out[:hi-lo] = sum over ranks of full[lo:hi] (each rank passes its own bounds)."""
        out[: hi - lo].copy_(full[lo:hi])
        return out

    def all_gather_into(self, full: torch.Tensor, shard: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
        """full[lo_r:hi_r] = shard_r for every rank r."""
        full[lo:hi].copy_(shard[: hi - lo])
        return full

    def broadcast_(self, t: torch.Tensor, src: int = 0) -> torch.Tensor:
        return t

    def broadcast_group_(self, t: Optional[torch.Tensor], src: int, ranks, shape=None, dtype=None, device=None):
        """Broadcast among the ranks in ``ranks`` only (K-FAC's gradient-worker groups: run_pretraining.py:321-345
        drives kfac_pytorch with HYBRID_OPT).  EVERY rank of the communicator calls this, in the same order; a rank
        outside ``ranks`` passes ``t=None`` and gets ``None`` back.  Default: a world broadcast in which outsiders
        take part with a scratch tensor (what round 1 did everywhere); ``TorchComm`` uses real sub-groups."""
        ranks = list(ranks)
        if self.world_size == 1 or len(ranks) <= 1:
            return t
        member = self.rank in ranks
        buf = t if t is not None else torch.empty(shape, dtype=dtype, device=device)
        self.broadcast_(buf, src=src)
        return buf if member else None

    def barrier(self) -> None:
        return None


class SingleComm(Comm):
    pass


class TorchComm(Comm):
    def __init__(self, group=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world_size = dist.get_world_size(group)
        self.name = dist.get_backend(group)

    _OPS = {"sum": dist.ReduceOp.SUM, "max": dist.ReduceOp.MAX, "min": dist.ReduceOp.MIN}

    def all_reduce_(self, t, op="sum", async_op: bool = False):
        if op == "avg":
            if self.name == "nccl":
                return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op) or t
            w = dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            t.div_(self.world_size)
            return t
        w = dist.all_reduce(t, op=self._OPS[op], group=self.group, async_op=async_op)
        return w if async_op else t

    def _bounds(self, n: int, lo: int, hi: int) -> List[List[int]]:
        mine = torch.tensor([lo, hi], dtype=torch.int64)
        if self.name == "nccl":
            mine = mine.cuda()
        alls = [torch.zeros_like(mine) for _ in range(self.world_size)]
        dist.all_gather(alls, mine, group=self.group)
        return [[int(a[0]), int(a[1])] for a in alls]

    def reduce_scatter(self, full, out, lo, hi):
        # shards may be ragged (last one short) -> all_reduce then slice keeps every backend
        # (gloo has no reduce_scatter) on one code path; the product path never comes here.
        dist.all_reduce(full, op=dist.ReduceOp.SUM, group=self.group)
        out[: hi - lo].copy_(full[lo:hi])
        return out

    def all_gather_into(self, full, shard, lo, hi):
        bounds = self._bounds(full.numel(), lo, hi)
        width = max(b[1] - b[0] for b in bounds)
        pad = torch.zeros(width, dtype=shard.dtype, device=shard.device)
        pad[: hi - lo].copy_(shard[: hi - lo])
        parts = [torch.empty_like(pad) for _ in range(self.world_size)]
        dist.all_gather(parts, pad, group=self.group)
        for (l, h), p in zip(bounds, parts):
            full[l:h].copy_(p[: h - l])
        return full

    def broadcast_(self, t, src=0):
        dist.broadcast(t, src=src, group=self.group)
        return t

    def broadcast_group_(self, t, src, ranks, shape=None, dtype=None, device=None):
        ranks = tuple(sorted(int(r) for r in ranks))
        if self.world_size == 1 or len(ranks) <= 1:
            return t
        if len(ranks) == self.world_size:
            return self.broadcast_(t, src=src)
        if self.group is not None:          # nested communicators: keep the simple (correct) world-broadcast fallback
            return super().broadcast_group_(t, src, ranks, shape, dtype, device)
        groups = self.__dict__.setdefault("_subgroups", {})
        g = groups.get(ranks)
        if g is None:                        # collective: every rank creates every sub-group, in first-use order
            g = dist.new_group(list(ranks))
            groups[ranks] = g
        if self.rank not in ranks:
            return None
        dist.broadcast(t, src=src, group=g)
        return t

    def barrier(self):
        dist.barrier(group=self.group)


class _FakeWorld:
    def __init__(self, world_size: int):
        self.world_size = world_size
        self.barrier = threading.Barrier(world_size)
        self.slots: Dict[str, List[Optional[torch.Tensor]]] = {}
        self.lock = threading.Lock()

    def exchange(self, key: str, rank: int, value):
        with self.lock:
            self.slots.setdefault(key, [None] * self.world_size)[rank] = value
        self.barrier.wait()
        vals = list(self.slots[key])
        self.barrier.wait()
        if rank == 0:
            with self.lock:
                self.slots.pop(key, None)
        self.barrier.wait()
        return vals


class FakeComm(Comm):
    """``FakeComm.spawn(world, fn)`` runs ``fn(comm)`` on ``world`` threads."""

    name = "fake"

    def __init__(self, world: _FakeWorld, rank: int):
        self._w, self.rank, self.world_size = world, rank, world.world_size
        self._seq = 0

    def _key(self, what: str) -> str:
        self._seq += 1
        return f"{what}:{self._seq}"

    def all_reduce_(self, t, op="sum"):
        vals = self._w.exchange(self._key("ar"), self.rank, t.clone())
        acc = vals[0].clone()
        for v in vals[1:]:            # fixed rank order -> bitwise identical on every rank
            acc = torch.maximum(acc, v) if op == "max" else (torch.minimum(acc, v) if op == "min" else acc + v)
        if op == "avg":
            acc = acc / self.world_size
        t.copy_(acc)
        return t

    def reduce_scatter(self, full, out, lo, hi):
        vals = self._w.exchange(self._key("rs"), self.rank, full)
        acc = vals[0][lo:hi].clone()
        for v in vals[1:]:
            acc = acc + v[lo:hi]
        out[: hi - lo].copy_(acc)
        self._w.barrier.wait()
        return out

    def all_gather_into(self, full, shard, lo, hi):
        vals = self._w.exchange(self._key("ag"), self.rank, (lo, hi, shard[: hi - lo].clone()))
        for l, h, s in vals:
            full[l:h].copy_(s)
        return full

    def broadcast_(self, t, src=0):
        vals = self._w.exchange(self._key("bc"), self.rank, t.clone() if self.rank == src else None)
        t.copy_(vals[src])
        return t

    def barrier(self):
        self._w.barrier.wait()

    @staticmethod
    def spawn(world_size: int, fn, *args):
        world = _FakeWorld(world_size)
        results: List = [None] * world_size
        errors: List = []

        def run(r):
            try:
                results[r] = fn(FakeComm(world, r), *args)
            except BaseException as e:  # noqa: BLE001
                errors.append(e)
                world.barrier.abort()
        threads = [threading.Thread(target=run, args=(r,)) for r in range(world_size)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        return results


def make_comm(kind: Optional[str] = None) -> Comm:
    """``kind``: None/auto, 'nccl', 'gloo' (torch.distributed must already be initialised),
    'fused' (peer-memory kernels; falls back to torch when the world is one rank)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size() == 1:
        return SingleComm()
    if kind == "fused":
        if spans_nodes():
            # the peer-memory kernels address the other ranks' arenas through NVLink mappings, which end at the
            # node boundary; a multi-node job keeps the bucket-free NCCL all-reduce of the flat gradient arena
            # unless the two-level variant is requested (B200_HIER_FUSED=1: node-local fused step + rail all-reduce)
            import os
            import warnings
            if os.environ.get("B200_HIER_FUSED") == "1":
                from .peer import HierarchicalPeerComm
                return HierarchicalPeerComm(local_world_size())
            warnings.warn("--backend fused needs all ranks on one NVLink domain; this job spans several nodes "
                          "-> using the NCCL backend (B200_HIER_FUSED=1 selects the two-level fused variant)")
            return TorchComm()
        from .peer import PeerComm
        return PeerComm()
    return TorchComm()


def local_world_size() -> int:
    """Ranks per NVLink domain: torchrun's LOCAL_WORLD_SIZE (B200_FAKE_LOCAL_WORLD overrides it so that one box can
    stand in for several nodes when testing the two-level paths); 0 = unknown."""
    import os
    for key in ("B200_FAKE_LOCAL_WORLD", "LOCAL_WORLD_SIZE"):
        try:
            v = int(os.environ.get(key, "0"))
        except ValueError:
            v = 0
        if v > 0:
            return v
    return 0


def spans_nodes() -> bool:
    """True when there are fewer local ranks than the world size (LOCAL_WORLD_SIZE < WORLD_SIZE)."""
    local = local_world_size()
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    return 0 < local < world
