"""T2 (SURVEY 4.2): multi-rank plumbing without GPUs -- the in-process fake backend verifies the partitioned
all-reduce+LAMB algorithm against the unfused reference; gloo multi-process verifies the real torch path."""
import copy
import os

import pytest
import torch
import torch.multiprocessing as mp

from bert_pytorch_b200 import BertConfig
from bert_pytorch_b200 import models as M
from bert_pytorch_b200.models.arena import ParamArena
from bert_pytorch_b200.optim import Lamb
from bert_pytorch_b200.parallel import DataParallel, FakeComm, ShardedLamb
from bert_pytorch_b200.parallel.sharded_lamb import slot_segments


def _model():
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=256, hidden_size=32, num_hidden_layers=1, num_attention_heads=2,
                     intermediate_size=64, max_position_embeddings=32, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    return M.BertForPreTraining(cfg)


def test_fake_comm_collectives():
    def fn(comm):
        t = torch.full((4,), float(comm.rank + 1))
        comm.all_reduce_(t)
        mx = torch.tensor([float(comm.rank)])
        comm.all_reduce_(mx, op="max")
        b = torch.tensor([float(comm.rank)])
        comm.broadcast_(b, src=2)
        full = torch.arange(8.0) * (comm.rank + 1)
        out = torch.zeros(2)
        comm.reduce_scatter(full.clone(), out, comm.rank * 2, comm.rank * 2 + 2)
        gathered = torch.zeros(8)
        comm.all_gather_into(gathered, out, comm.rank * 2, comm.rank * 2 + 2)
        return t, mx, b, gathered
    res = FakeComm.spawn(4, fn)
    for t, mx, b, g in res:
        assert t.tolist() == [10.0] * 4 and mx.item() == 3.0 and b.item() == 2.0
        assert torch.equal(g, torch.arange(8.0) * 10)


def test_slot_segments_straddle():
    segs = slot_segments([0, 10, 64], [10, 50, 30], 5, 70)
    assert segs == [(0, 5, 10), (1, 10, 60), (2, 64, 70)]


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_lamb_equals_unfused_reference(world):
    """reduce-scatter + partitioned LAMB (two-phase norms) + all-gather == all-reduce(avg) + full LAMB."""
    base = _model()
    grads = []
    for r in range(world):
        torch.manual_seed(100 + r)
        grads.append([torch.randn_like(p) * (5.0 if r == 0 else 0.2) for p in base.parameters()])
    # unfused reference on one rank: averaged grads, plain LAMB
    ref = copy.deepcopy(base)
    named = list(ref.named_parameters())
    nd = ("bias", "LayerNorm")
    opt = Lamb([{"params": [p for n, p in named if not any(k in n for k in nd)], "weight_decay": 0.01},
                {"params": [p for n, p in named if any(k in n for k in nd)], "weight_decay": 0.0}], lr=5e-3)
    for step in range(2):
        for i, p in enumerate(ref.parameters()):
            p.grad = sum(g[i] for g in grads) / world * (1.0 + step)
        opt.step()

    def fn(comm):
        m = copy.deepcopy(base)
        arena = ParamArena(m)
        sl = ShardedLamb(arena, comm, lr=5e-3, weight_decay=0.01, granule=64)
        for step in range(2):
            for i, p in enumerate(m.parameters()):
                p.grad.copy_(grads[comm.rank][i] * (1.0 + step))
            assert sl.step(loss_scale=1.0)
        return [p.detach().clone() for p in m.parameters()], sl.last_grad_norm
    outs = FakeComm.spawn(world, fn)
    for params, gnorm in outs:
        for (n, pr), pf in zip(ref.named_parameters(), params):
            assert torch.allclose(pr, pf, rtol=2e-5, atol=2e-6), (world, n, (pr - pf).abs().max().item())
    assert all(torch.equal(a, b) for a, b in zip(outs[0][0], outs[-1][0]))       # ranks agree bit for bit


def test_sharded_lamb_overflow_skips_everywhere():
    base = _model()

    def fn(comm):
        m = copy.deepcopy(base)
        arena = ParamArena(m)
        before = arena.flat_param.clone()
        sl = ShardedLamb(arena, comm, lr=1e-2, granule=64)
        for p in m.parameters():
            p.grad.fill_(1.0)
        if comm.rank == 1:
            arena.flat_grad[3] = float("inf")      # only one rank overflows
        applied = sl.step(loss_scale=128.0)
        return applied, torch.equal(arena.flat_param, before), float(arena.flat_grad.abs().sum())
    for applied, unchanged, gsum in FakeComm.spawn(3, fn):
        assert applied is False and unchanged and gsum == 0.0


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="env://")
    from bert_pytorch_b200.parallel import TorchComm
    m = _model()
    if rank != 0:
        for p in m.parameters():
            p.data.add_(1.0)                      # diverge; ctor must broadcast rank 0's weights
    arena = ParamArena(m)
    ddp = DataParallel(m, comm=TorchComm(), arena=arena)
    w0 = arena.flat_param.clone()
    torch.manual_seed(5)
    ids = torch.randint(0, 256, (2 * world, 16))
    mine = ids[rank * 2:(rank + 1) * 2]
    with ddp.no_sync():
        s, n = ddp(mine)
        (s.float().mean() + n.float().mean()).backward()
        ddp.sync_gradients()                      # suppressed inside no_sync
    g_local = arena.flat_grad.clone()
    ddp.sync_gradients()
    # by value: a tensor in a queue is a file descriptor served by this process, which may exit before the parent reads it
    q.put((rank, w0.numpy().copy(), g_local.numpy().copy(), arena.flat_grad.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


def test_gloo_data_parallel_broadcast_nosync_and_average():
    world, port = 2, 29655
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    (_, w0a, ga, sa), (_, w0b, gb, sb) = [(r, *(torch.from_numpy(a) for a in arrs)) for r, *arrs in res]
    assert torch.equal(w0a, w0b)                                   # broadcast at construction
    assert not torch.equal(ga, gb)                                 # no_sync kept gradients local
    assert torch.allclose(sa, (ga + gb) / 2, atol=1e-7) and torch.equal(sa, sb)


def test_all_reduce_many_default_and_fused_reduction_config():
    """Comm.all_reduce_many_ (packed by the peer backend, a loop elsewhere) and the runtime's choice of where the
    gradient reduction happens (deferred into the fused optimizer kernel unless a preconditioner needs averaged grads)."""
    import torch
    from bert_pytorch_b200 import pretrain
    from bert_pytorch_b200.parallel.comm import FakeComm

    def run(c):
        ts = [torch.full((3, 2), float(c.rank + 1)), torch.arange(5, dtype=torch.float32) * (c.rank + 1)]
        c.all_reduce_many_(ts, op="avg")
        return ts
    outs = FakeComm.spawn(3, run)
    for ts in outs:
        assert torch.allclose(ts[0], torch.full((3, 2), 2.0)) and torch.allclose(ts[1], torch.arange(5.0) * 2.0)

    class _Peer:                                   # the interface pretrain.configure_fused_reduction relies on
        fuses_optimizer = True
        push_master = True
        def __init__(self): self.names = None
        def set_prereduced(self, names): self.names = list(names)

    class _Wrapped(torch.nn.Module):
        def __init__(self, comm):
            super().__init__()
            self.module = torch.nn.Linear(2, 2)
            self.comm = comm
    w = _Wrapped(_Peer())
    pretrain.configure_fused_reduction(w, preconditioner=None)
    assert w.defer_reduction is True and w.comm.push_master is False and w.comm.names is None   # no fused engine on CPU
    w2 = _Wrapped(_Peer())
    pretrain.configure_fused_reduction(w2, preconditioner=object())
    assert w2.defer_reduction is False and w2.comm.push_master is True          # K-FAC: classic all-reduce first


def test_fused_backend_falls_back_across_nodes(monkeypatch):
    """`--backend fused` on a job that spans several nodes (LOCAL_WORLD_SIZE < WORLD_SIZE) keeps the torch backend:
    NVLink peer mappings end at the node boundary."""
    import warnings
    from bert_pytorch_b200.parallel import comm as C

    class _Dist:
        @staticmethod
        def is_available(): return True
        @staticmethod
        def is_initialized(): return True
        @staticmethod
        def get_world_size(*a): return 16
        @staticmethod
        def get_rank(*a): return 0
    monkeypatch.setattr(C, "dist", _Dist)
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "8")
    assert C.spans_nodes()
    made = []
    monkeypatch.setattr(C, "TorchComm", lambda *a, **k: made.append("torch") or "torch-comm")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert C.make_comm("fused") == "torch-comm"
    assert any("spans several nodes" in str(x.message) for x in w)
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "16")
    assert not C.spans_nodes()


class _StubPeer:
    """Stands in for PeerComm on CPU: 'symmetric' gradient arena = a plain tensor, the fused step = node-local sum
    times the kernel's unscale constant 1 / (local_world * loss_scale)."""
    def __init__(self, group=None, **kw):
        import torch.distributed as dist
        self.group, self.rank, self.world_size = group, dist.get_rank(group), dist.get_world_size(group)
        self.device, self.push_master, self.stats, self.arena = torch.device("cpu"), True, torch.zeros(4), None
        self.grad_t = torch.full((8,), float(dist.get_rank() + 1))
        self.result = None

    def fused_lamb_step(self, optimizer, loss_scale=1.0):
        import torch.distributed as dist
        t = self.grad_t.clone()
        dist.all_reduce(t, group=self.group)
        self.result = t / (self.world_size * loss_scale)


def _hier_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      B200_FAKE_LOCAL_WORLD="2", B200_HIER_FUSED="1")
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="env://")
    from bert_pytorch_b200.parallel import comm as C, peer as P
    P.PeerComm = _StubPeer
    c = C.make_comm("fused")
    assert isinstance(c, P.HierarchicalPeerComm) and (c.rank, c.world_size, c.nodes, c.local_world) == (rank, world, 2, 2)
    assert c.inner.rank == rank % 2 and c.inner.world_size == 2
    c.push_master = False
    c.fused_lamb_step(optimizer=None, loss_scale=4.0)
    q.put((rank, c.inner.result.numpy().copy(), c.inner.push_master))       # by value, as in _gloo_worker
    dist.barrier()
    dist.destroy_process_group()


def test_two_level_fused_backend_composition_gloo():
    """4 gloo ranks as 2 'nodes' x 2: rail all-reduce + node-local step = job-wide mean / loss_scale on every rank."""
    world, port = 4, 29657
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_hier_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for _, out, pm in res:
        assert pm is False
        assert torch.allclose(torch.from_numpy(out), torch.full((8,), (1 + 2 + 3 + 4) / 4 / 4.0))


def _ddp_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="env://")
    from torch.nn.parallel import DistributedDataParallel as TorchDDP
    from bert_pytorch_b200.parallel import TorchComm
    m_ref = _model()
    m_mine = copy.deepcopy(m_ref)
    ddp_ref = TorchDDP(m_ref)                       # what the reference wraps its model in (run_pretraining.py:270)
    arena = ParamArena(m_mine)
    ddp_mine = DataParallel(m_mine, comm=TorchComm(), arena=arena)
    torch.manual_seed(7)
    ids = torch.randint(0, 256, (2 * world, 16))
    mine = ids[rank * 2:(rank + 1) * 2]
    worst = 0.0
    for step in range(2):                           # second step: accumulate one local micro-step first (no_sync)
        for w in (ddp_ref, ddp_mine):
            if step == 1:
                with w.no_sync():
                    s, n = w(torch.roll(mine, 3, 1))
                    (s.float().mean() + n.float().mean()).backward()
            s, n = w(mine)
            (s.float().mean() + n.float().mean()).backward()
        ddp_mine.sync_gradients()
        for (k, p), p2 in zip(m_ref.named_parameters(), m_mine.parameters()):
            worst = max(worst, float((p.grad - p2.grad).abs().max()))
        m_ref.zero_grad(); arena.zero_grad()
    q.put((rank, worst))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_matches_torch_ddp_gloo():
    """Same model and batches under torch DistributedDataParallel and under this repo's DataParallel (one flat
    all-reduce of the gradient arena): identical averaged gradients, also after a ``no_sync`` accumulation step."""
    world, port = 2, 29661
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(w < 1e-6 for _, w in res), res
