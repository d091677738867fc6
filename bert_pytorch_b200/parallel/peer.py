"""Peer-memory communication backend: the product path for the gradient reduction.

``PeerComm`` keeps the parameter / gradient / shadow arenas of every rank in CUDA *symmetric memory*
(VMM allocations mapped into every peer over NVLink 5 / NVSwitch, plus the NVLS multicast mapping when the
fabric offers it) and replaces

    DDP bucketed ncclAllReduce  ->  GradScaler.unscale_  ->  FusedLAMB  (reference: run_pretraining.py:405-458)

by ONE persistent sm_90a kernel per optimizer step (ops/csrc/comm.cu): reduce-scatter of the gradient
shards with P2P loads / ``multimem.ld_reduce``, fused 1/(world*scale) + inf/nan detection, partitioned LAMB
with cross-rank norm exchange through peer stores, and the parameter all-gather as P2P / ``multimem.st``
stores of the updated fp32 + bf16 values.  No NCCL call on this path.  The bootstrap (rendezvous, handle
exchange) uses torch.distributed / ``torch.distributed._symmetric_memory``; the kernels are ours.

GEMM -> reduce-scatter fusion: with the gradient arenas registered at the GEMM launcher (``set_grad_peers``) the
weight-gradient GEMMs of the LAST micro-step of an optimizer step (``begin_push`` / ``end_push``) add their
tiles -- plus the locally accumulated value -- straight into the arena of the rank that owns the shard, so most
of the reduce-scatter happens tile by tile under the remaining backward pass and the fused kernel reads those
tensors locally (``set_prereduced``).  ``all_reduce_many_`` is a general packed all-reduce through our own
kernel (K-FAC factor statistics).

The optimizer state (moments) is *partitioned*: each rank only ever touches its own contiguous shard, so
``state_dict`` gathers the shards (cold path, NCCL all-reduce of the zero-padded shards) into the full
per-parameter layout the checkpoint format expects (SURVEY.md 5.4).

The algorithm is specified and unit-tested on CPU in :mod:`bert_pytorch_b200.parallel.sharded_lamb`.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from .comm import TorchComm

GRANULE = 2048        # shard boundaries are multiples of this many elements
CHUNK = 65536


class PeerComm(TorchComm):
    name = "fused"
    fuses_optimizer = True

    def __init__(self, group=None, use_multicast: Optional[bool] = None, push_master: Optional[bool] = None):
        super().__init__(group)
        import os
        # push_master=False keeps the fp32 master weights shard-local (ZeRO-1 style): only the bf16 weights the
        # kernels read (and the fp32 1-D tensors) are all-gathered, 3x less NVLink traffic.
        # ``gather_master()`` completes the fp32 views before
        # anything reads them (checkpoint, ``arena.refresh_shadow``, torch-path evaluation).  The pre-training
        # runtime selects it (pretrain.configure_fused_reduction); B200_PEER_MASTER_LOCAL=0/1 overrides.
        if push_master is None:
            push_master = os.environ.get("B200_PEER_MASTER_LOCAL", "0") != "1"
        self.push_master = bool(push_master)
        self._master_stale = False
        self.name = "fused"
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.arena = None
        self.epoch = 0
        self._want_mc = use_multicast
        self.use_multicast = False
        self.last_stats: Optional[torch.Tensor] = None

    # -- symmetric allocation ---------------------------------------------------------------------
    def _symm(self, numel: int, dtype: torch.dtype):
        import torch.distributed._symmetric_memory as symm
        t = symm.empty(numel, dtype=dtype, device=self.device)
        t.zero_()
        h = symm.rendezvous(t, self.group if self.group is not None else dist.group.WORLD)
        return t, h

    def adopt(self, arena) -> None:
        """Move the arena's buffers into symmetric memory (weights/grad values preserved) and build the
        shard tables.  Call once, before the optimizer is bound."""
        n = arena.numel
        T = len(arena.slots)
        self.grad_t, self.grad_h = self._symm(n, torch.float32)
        self.param_t, self.param_h = self._symm(n, torch.float32)
        self.shadow_t, self.shadow_h = self._symm(n, torch.bfloat16)
        pad_floats = 2 * self.world_size + self.world_size * 2 * T
        self.pad_t, self.pad_h = self._symm(pad_floats + 64, torch.float32)
        self.flag_t, self.flag_h = self._symm(4 * self.world_size + 64, torch.int32)
        with torch.no_grad():
            self.param_t.copy_(arena.flat_param)
            self.grad_t.copy_(arena.flat_grad)
            self.shadow_t.copy_(arena.flat_shadow if arena.flat_shadow is not None else arena.flat_param)
        arena.flat_param, arena.flat_grad, arena.flat_shadow = self.param_t, self.grad_t, self.shadow_t
        arena.shadow_dtype = torch.bfloat16
        for s, p in zip(arena.slots, arena.params):          # re-point the nn.Parameters at the new storage
            p.data = self.param_t[s.offset:s.offset + s.numel].view(s.shape)
            p.grad = self.grad_t[s.offset:s.offset + s.numel].view(s.shape)
        arena._opt_tables = None
        self.arena = arena
        arena._master_sync = self.gather_master
        mc_ok = all(int(getattr(h, "multicast_ptr", 0) or 0) != 0 for h in (self.grad_h, self.param_h))
        # NVLS multimem from 4 ranks up (in-switch reduction / replication); plain P2P at 2 ranks
        self.use_multicast = (mc_ok and self.world_size > 2) if self._want_mc is None else (bool(self._want_mc) and mc_ok)
        self.lo, self.hi = arena.shard_bounds(self.world_size, self.rank, GRANULE)
        # chunk table of the arena restricted to the shard
        ct, cs, cl = [], [], []
        for t, s in enumerate(arena.slots):
            a, b = max(s.offset, self.lo), min(s.offset + s.numel, self.hi)
            x = a
            while x < b:
                ln = min(CHUNK, b - x)
                ct.append(t); cs.append(x); cl.append(ln)
                x += ln
        dev = self.device
        self.chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=dev)
        self.chunk_start = torch.tensor(cs, dtype=torch.int64, device=dev)
        self.chunk_len = torch.tensor(cl, dtype=torch.int32, device=dev)
        # GEMM -> reduce-scatter fusion: register the gradient arenas with the GEMM launcher.  From now on every
        # fp32-accumulate GEMM into the local arena adds atomically, and between begin_push()/end_push() its tiles
        # go straight into the owner rank's arena (ops/csrc/gemm_sm100.cu, peer_push).
        per = (arena.numel + self.world_size - 1) // self.world_size
        per = (per + GRANULE - 1) // GRANULE * GRANULE
        from .. import ops
        ops.extension().set_grad_peers(self.world_size, self.rank, list(self.grad_h.buffer_ptrs), arena.numel, per)
        self._prereduced = None               # int32 [T]: tensors whose reduction happens inside the backward
        self._pushed = False
        self.stats = torch.zeros(16, dtype=torch.float32, device=dev)   # [0..3] sumsq / inf exchange, [8..15] in-kernel timeline (ms)
        self.norms = torch.zeros(2 * T, dtype=torch.float32, device=dev)
        self.grid_bar = torch.zeros(1, dtype=torch.int32, device=dev)
        dist.barrier(group=self.group)
        torch.cuda.synchronize()

    # -- GEMM -> reduce-scatter fusion -------------------------------------------------------------------
    def set_prereduced(self, names) -> None:
        """Names of the tensors whose ENTIRE gradient is produced by fp32-accumulate GEMMs (the engine's
        weight-gradient launches): with push mode on in the last micro-step they arrive fully reduced at
        their owner and the fused step skips their peer reads."""
        names = set(names or ())
        flags = [1 if s.name in names else 0 for s in self.arena.slots]
        self._prereduced = torch.tensor(flags, dtype=torch.int32, device=self.device) if any(flags) else None

    def begin_push(self) -> bool:
        """Call before the forward/backward of the LAST micro-step of an optimizer step."""
        if self._prereduced is None:
            return False
        from .. import ops
        ops.extension().set_grad_push(True)
        self._pushed = True
        return True

    def end_push(self) -> None:
        from .. import ops
        ops.extension().set_grad_push(False)

    # -- the fused step ------------------------------------------------------------------------------
    @torch.no_grad()
    def fused_lamb_step(self, optimizer, loss_scale: float = 1.0) -> None:
        """reduce-scatter + unscale + partitioned LAMB + all-gather, one kernel.  ``optimizer`` supplies the
        hyper-parameters and owns the (arena backed) moment buffers."""
        from .. import ops
        from ..ops.api import _uniform, _uniform_decay
        A = self.arena
        if A is None or A.exp_avg is None:
            raise RuntimeError("PeerComm.adopt(arena) and arena.bind_optimizer(optimizer) must be called first")
        decay = getattr(self, "_decay", None)
        if decay is None:
            decay = torch.tensor([1 if s.decay else 0 for s in A.slots], dtype=torch.int32, device=self.device)
            self._decay = decay
        lr = _uniform(optimizer, "lr")
        b1, b2 = _uniform(optimizer, "betas")
        wd = _uniform_decay(optimizer)
        step = int(optimizer.param_groups[0].get("step", 0)) + 1
        self.epoch += 1
        mc = self.use_multicast
        ops.extension().fused_allreduce_lamb(
            self.rank, self.world_size, mc,
            list(self.grad_h.buffer_ptrs), list(self.param_h.buffer_ptrs), list(self.shadow_h.buffer_ptrs),
            list(self.pad_h.buffer_ptrs), list(self.flag_h.buffer_ptrs),
            int(self.grad_h.multicast_ptr) if mc else 0, int(self.param_h.multicast_ptr) if mc else 0,
            int(getattr(self.shadow_h, "multicast_ptr", 0) or 0) if mc else 0,
            A.exp_avg, A.exp_avg_sq, A.numel, self.lo, self.hi, self.chunk_tensor, self.chunk_start, self.chunk_len,
            decay, self.stats, self.norms, self.grid_bar, self.epoch, 1.0 / (self.world_size * loss_scale),
            float(lr), float(b1), float(b2), float(_uniform(optimizer, "eps")), wd,
            float(_uniform(optimizer, "max_grad_norm") or 0.0), step, bool(_uniform(optimizer, "bias_correction")),
            bool(_uniform(optimizer, "grad_averaging")), bool(optimizer.adam_w_mode), bool(optimizer.use_nvlamb),
            self.push_master, self._prereduced if self._pushed else None)
        self._pushed = False
        self._master_stale = not self.push_master
        A.version += 1
        ops.api._count()
        # apex semantics: the step counter (bias correction, LR schedule) advances only when the update was applied.
        # With a loss scale in play the kernel may have skipped the step (inf agreed across the ranks, stats[3]);
        # reading the flag is the one host sync of an fp16 step -- bf16 (loss_scale == 1) never reads it.
        applied = True
        if loss_scale != 1.0:
            applied = float(self.stats[3]) == 0.0
        if applied:
            for g in optimizer.param_groups:
                g["step"] = step
        self.last_stats = self.stats

    TIMELINE_KEYS = ("barrier_wait_ms", "reduce_scatter_ms", "sync1_ms", "moments_ms", "sync2_ms", "apply_allgather_ms",
                     "zero_final_barrier_ms", "kernel_total_ms")

    def timeline(self) -> dict:
        """In-kernel %globaltimer split of the last fused step on this rank (block 0): where the reduce-scatter + LAMB
        + all-gather kernel spent its time; ``barrier_wait_ms`` is the wait for the slowest rank's backward pass."""
        vals = self.stats[8:16].tolist()
        return {k: round(float(v), 4) for k, v in zip(self.TIMELINE_KEYS, vals)}

    # -- general all-reduce through our own kernel (K-FAC factors etc.) -------------------------------------
    STAGE_FLOATS = 64 << 20          # 256 MB symmetric staging buffer, allocated on first use

    def _stage(self):
        if getattr(self, "_stage_t", None) is None:
            self._stage_t, self._stage_h = self._symm(self.STAGE_FLOATS, torch.float32)
            self._ar_flag_t, self._ar_flag_h = self._symm(2 * self.world_size + 64, torch.int32)
            self._ar_bar = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._ar_epoch = 0
            mc = int(getattr(self._stage_h, "multicast_ptr", 0) or 0)
            self._ar_mc = mc if (self._want_mc is None or self._want_mc) else 0
            dist.barrier(group=self.group)
        return self._stage_t

    def _stage_allreduce(self, n: int, scale: float) -> None:
        from .. import ops
        n4 = (n + 3) // 4 * 4
        self._ar_epoch += 1
        ops.extension().peer_allreduce(self.rank, self.world_size, self._ar_mc != 0, list(self._stage_h.buffer_ptrs),
                                       list(self._ar_flag_h.buffer_ptrs), self._ar_mc, self._ar_bar, self._ar_epoch,
                                       n4, scale)
        ops.api._count()

    @torch.no_grad()
    def all_reduce_many_(self, tensors, op: str = "sum") -> None:
        """fp32 CUDA tensors are packed into the symmetric staging buffer and reduced by ONE peer-memory kernel
        per 256 MB (no NCCL); anything else falls back to the torch.distributed path."""
        mine = [t for t in tensors if t.is_cuda and t.dtype == torch.float32 and op in ("sum", "avg")]
        for t in tensors:
            if not any(t is m for m in mine):
                super().all_reduce_(t, op=op)
        if not mine:
            return
        stage = self._stage()
        scale = 1.0 / self.world_size if op == "avg" else 1.0
        cap = stage.numel()
        pieces = []                                   # (flat view of the source, offset in it, length)
        for t in mine:
            flat = t.reshape(-1) if t.is_contiguous() else None
            src = flat if flat is not None else t.contiguous().reshape(-1)
            off = 0
            while off < src.numel():
                ln = min(src.numel() - off, cap)
                pieces.append((t, src, off, ln, flat is None))
                off += ln
        i = 0
        while i < len(pieces):
            used, batch = 0, []
            while i < len(pieces) and used + (pieces[i][3] + 3) // 4 * 4 <= cap:
                batch.append((pieces[i], used))
                used += (pieces[i][3] + 3) // 4 * 4
                i += 1
            if used < cap:
                stage[used:min(cap, used + 4)].zero_()
            for (t, src, off, ln, _), pos in batch:
                stage[pos:pos + ln].copy_(src[off:off + ln])
                if ln % 4:
                    stage[pos + ln:pos + (ln + 3) // 4 * 4].zero_()
            self._stage_allreduce(used, scale)
            for (t, src, off, ln, copied), pos in batch:
                src[off:off + ln].copy_(stage[pos:pos + ln])
        for t, src, off, ln, copied in pieces:
            if copied and off + ln == src.numel():
                t.copy_(src.view_as(t))

    @torch.no_grad()
    def all_reduce_(self, t, op="sum", async_op: bool = False):
        if async_op or not (t.is_cuda and t.dtype == torch.float32 and op in ("sum", "avg")) or t.numel() < 1024:
            return super().all_reduce_(t, op=op, async_op=async_op)
        self.all_reduce_many_([t], op=op)
        return t

    @torch.no_grad()
    def gather_master(self) -> None:
        """Make every rank's fp32 parameter arena complete again (only needed with ``push_master=False``):
        zero the foreign shards and sum over the ranks -- cold path (checkpoint / evaluation)."""
        if not self._master_stale:
            return
        flat = self.param_t
        flat[: self.lo].zero_()
        flat[self.hi:].zero_()
        dist.all_reduce(flat, group=self.group)
        self._master_stale = False

    # -- checkpoint support ----------------------------------------------------------------------------
    @torch.no_grad()
    def gather_optimizer_state(self) -> None:
        """Make every rank's moment arenas complete (each rank only maintains its shard): zero everything
        outside the shard and sum over ranks.  Cold path (checkpoint time) -> NCCL."""
        A = self.arena
        for buf in (A.exp_avg, A.exp_avg_sq):
            buf[: self.lo].zero_()
            buf[self.hi:].zero_()
            dist.all_reduce(buf, group=self.group)


class HierarchicalPeerComm(TorchComm):
    """The fused backend on a job that spans several NVLink domains (nodes): opt-in (``B200_HIER_FUSED=1``), not yet
    exercised on hardware (one box can emulate it with ``B200_FAKE_LOCAL_WORLD=k``: ranks [0,k), [k,2k), ... act as nodes).

    Ranks are ``node * local_world + local_rank``.  Inside a node the gradient arena lives in symmetric memory and
    the unmodified single-node machinery runs (:class:`PeerComm` over the node's process group: GEMM -> reduce-scatter
    push, reduce-scatter + LAMB + all-gather kernel).  Across nodes every rank first all-reduces its gradient arena
    with the ranks of the same local index ("rail" groups: NCCL over the NICs, one rail per GPU), so each node then
    holds the job-wide sums partitioned over its local ranks and the node-local kernel finishes the step; the
    averaging factor 1 / (nodes * local_world) is folded into the kernel's unscale constant.  Every node ends up with
    the same parameters and (partitioned) LAMB state, so checkpoints gather inside node 0 only.
    Generic collectives (broadcast at start-up, K-FAC factors, barriers) use the world NCCL group.
    The rail all-reduce moves the whole arena; shard-only traffic needs the reduction kernel split at the phase
    boundary."""
    fuses_optimizer = True

    def __init__(self, local_world: int, **peer_kw):
        super().__init__(None)                                   # world group: rank / world_size stay global
        world, rank = self.world_size, self.rank
        if local_world <= 0 or world % local_world != 0:
            raise ValueError(f"world size {world} is not a multiple of the node size {local_world}")
        self.nodes, self.local_world = world // local_world, local_world
        node, lrank = divmod(rank, local_world)
        # every rank creates every group, in the same order (torch.distributed requirement)
        local_groups = [dist.new_group(list(range(n * local_world, (n + 1) * local_world))) for n in range(self.nodes)]
        rail_groups = [dist.new_group(list(range(l, world, local_world))) for l in range(local_world)]
        self.rail = rail_groups[lrank]
        self.inner = PeerComm(group=local_groups[node], **peer_kw)
        self.name = "fused-hier"
        self.device = self.inner.device

    # -- what the runtime touches on a fused backend -------------------------------------------------------------
    @property
    def push_master(self) -> bool:
        return self.inner.push_master

    @push_master.setter
    def push_master(self, v: bool) -> None:
        self.inner.push_master = bool(v)

    @property
    def stats(self):
        return self.inner.stats

    @property
    def arena(self):
        return self.inner.arena

    def adopt(self, arena) -> None:
        self.inner.adopt(arena)

    def set_prereduced(self, names) -> None:
        # GEMM -> reduce-scatter push is OFF in hierarchical mode (ADVICE r1, medium): same-node peers would still be
        # adding tiles into this rank's arena while the rail all-reduce below reads it -- the only cross-rank barrier
        # of the push protocol sits inside the fused kernel, which runs after the rail reduction.
        self.inner.set_prereduced(None)

    def begin_push(self) -> bool:
        return False

    def end_push(self) -> None:
        pass

    def timeline(self) -> dict:
        return self.inner.timeline()

    @torch.no_grad()
    def fused_lamb_step(self, optimizer, loss_scale: float = 1.0) -> None:
        dist.all_reduce(self.inner.grad_t, group=self.rail)      # sums over nodes, rail by rail
        self.inner.fused_lamb_step(optimizer, loss_scale=loss_scale * self.nodes)

    def gather_master(self) -> None:
        self.inner.gather_master()

    def gather_optimizer_state(self) -> None:
        self.inner.gather_optimizer_state()
