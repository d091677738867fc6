"""Multi-GPU check of the fused peer-memory all-reduce + LAMB kernel (run under torchrun, >= 2 GPUs):

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29577 tools/peer_check.py [--big]

1. correctness: fused kernel == NCCL all-reduce(avg) + single-GPU arena LAMB, incl. a clipped step, a
   tensor straddling shard boundaries and an overflow step that every rank must skip;
2. (--big) device-timed step on a BERT-large sized arena (336 M parameters): fused kernel vs
   NCCL all-reduce + unfused LAMB, max over ranks, with the roofline fraction of SURVEY.md 5.8.
Rank 0 prints one JSON line per section."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bert_pytorch_b200 import BertConfig  # noqa: E402
from bert_pytorch_b200.models import BertForPreTraining  # noqa: E402
from bert_pytorch_b200.models.arena import NO_DECAY_KEYS, ParamArena  # noqa: E402
from bert_pytorch_b200.optim import Lamb  # noqa: E402
from bert_pytorch_b200.parallel.peer import PeerComm  # noqa: E402


def groups(model):
    named = list(model.named_parameters())
    return [{"params": [p for n, p in named if not any(k in n for k in NO_DECAY_KEYS)], "weight_decay": 0.01},
            {"params": [p for n, p in named if any(k in n for k in NO_DECAY_KEYS)], "weight_decay": 0.0}]


def build(cfg, dev, fused, use_mc=None):
    torch.manual_seed(0)
    model = BertForPreTraining(cfg).to(dev)
    arena = ParamArena(model, device=dev)
    comm = None
    if fused:
        comm = PeerComm(use_multicast=use_mc)
        comm.adopt(arena)
    opt = Lamb(groups(model), lr=5e-3)
    arena.bind_optimizer(opt)
    return model, arena, opt, comm


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", init_method="env://", device_id=dev)
    out = {"world": world}
    cfg = BertConfig(vocab_size_or_config_json_file=2048, hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                     intermediate_size=1024, max_position_embeddings=128)
    for mc in ([False, True] if "--no-mc" not in sys.argv else [False]):
        m_f, a_f, o_f, comm = build(cfg, dev, True, use_mc=mc)
        if mc and not comm.use_multicast:
            out["multicast"] = "unavailable"
            continue
        m_r, a_r, o_r, _ = build(cfg, dev, False)
        worst = 0.0
        for step in range(4):
            torch.manual_seed(1000 * step + rank)
            g = torch.randn(a_f.numel, device=dev) * (8.0 if step == 1 else 0.05)
            if step == 3 and rank == world - 1:
                g[12345] = float("inf")                       # overflow on one rank only
            a_f.flat_grad.copy_(g)
            a_r.flat_grad.copy_(g)
            torch.cuda.synchronize(); dist.barrier()
            before = a_f.flat_param.clone()
            comm.fused_lamb_step(o_f, loss_scale=4.0)
            torch.cuda.synchronize()
            if step == 3:
                skipped = bool(torch.equal(a_f.flat_param, before)) and float(a_f.flat_grad.abs().max()) == 0.0
                out[f"overflow_skipped_mc{int(mc)}"] = skipped and float(comm.stats[3]) > 0
                continue
            dist.all_reduce(a_r.flat_grad)
            a_r.flat_grad.mul_(1.0 / (world * 4.0))
            o_r.step()
            torch.cuda.synchronize()
            diff = (a_f.flat_param - a_r.flat_param).abs()
            d = diff.max().item()
            sh = (a_f.flat_shadow.float() - a_f.flat_param).abs().max().item()
            if rank == 0:
                i = int(diff.argmax())
                slot = next((sl for sl in a_f.slots if sl.offset <= i < sl.offset + sl.numel), None)
                lo, hi = comm.lo, comm.hi
                dm = (a_f.exp_avg[lo:hi] - a_r.exp_avg[lo:hi]).abs().max().item()
                dv = (a_f.exp_avg_sq[lo:hi] - a_r.exp_avg_sq[lo:hi]).abs().max().item()
                out.setdefault(f"detail_mc{int(mc)}", []).append(
                    dict(step=step, max_diff=d, at=i, slot=(slot.name if slot else "gap"), decay=(slot.decay if slot else None),
                         p_fused=float(a_f.flat_param[i]), p_ref=float(a_r.flat_param[i]), dm=dm, dv=dv,
                         gnorm_fused=float(comm.stats[2].sqrt()), gnorm_ref=float(o_r.last_grad_norm)))
            worst = max(worst, d)
            assert sh < 2e-2, sh
            # every rank must hold identical parameters
            ref = a_f.flat_param.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(ref, a_f.flat_param), "ranks disagree after the fused step"
        out[f"max_abs_diff_mc{int(mc)}"] = worst
        out[f"grad_norm_mc{int(mc)}"] = float(comm.stats[2].sqrt())
        # GEMM -> reduce-scatter fusion: two micro-steps of the real engine per optimizer step, the second one with
        # its weight-gradient tiles pushed into the owners' arenas, against local accumulation + NCCL + LAMB
        from bert_pytorch_b200.ops import api as K
        ext = K.extension()
        pcfg = BertConfig(vocab_size_or_config_json_file=2048, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                          intermediate_size=1024, max_position_embeddings=128, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0)
        pcfg.max_predictions_per_seq = 16
        m_p, a_p, o_p, comm_p = build(pcfg, dev, True, use_mc=mc)
        m_q, a_q, o_q, _ = build(pcfg, dev, False)
        m_p.train(); m_q.train()
        e_p, e_q = m_p.pretrain_engine(), m_q.pretrain_engine()
        e_p.use_graphs = e_q.use_graphs = False
        comm_p.set_prereduced(e_p.engine.gemm_reduced_parameters())
        gen = torch.Generator(device=dev).manual_seed(4321 + rank)
        push_worst, push_steps = 0.0, []
        for step in range(3):
            for micro in range(2):
                ids = torch.randint(5, 2048, (4, 64), device=dev, generator=gen)
                seg = torch.zeros_like(ids); seg[:, 32:] = 1
                mask = torch.ones_like(ids)
                labels = torch.full_like(ids, -1)
                pos = torch.randint(0, 64, (4, 10), device=dev, generator=gen)
                labels.scatter_(1, pos, ids.gather(1, pos))
                nsl = torch.randint(0, 2, (4,), device=dev, generator=gen)
                e_q.forward_backward(ids, seg, mask, labels, nsl, grad_scale=0.5)
                if micro == 1:
                    assert comm_p.begin_push()
                e_p.forward_backward(ids, seg, mask, labels, nsl, grad_scale=0.5)
                if micro == 1:
                    comm_p.end_push()
            torch.cuda.synchronize(); dist.barrier()
            comm_p.fused_lamb_step(o_p, loss_scale=1.0)
            dist.all_reduce(a_q.flat_grad)
            a_q.flat_grad.mul_(1.0 / world)
            o_q.step()
            a_q.zero_grad()
            torch.cuda.synchronize()
            push_steps.append((a_p.flat_param - a_q.flat_param).abs().max().item())
            push_worst = max(push_worst, push_steps[-1])
            ref = a_p.flat_param.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(ref, a_p.flat_param), "ranks disagree after the pushed step"
        out[f"push_max_abs_diff_mc{int(mc)}"] = push_worst
        out[f"push_diff_per_step_mc{int(mc)}"] = push_steps     # the two arms train independently: only step 0 is a bitwise-level comparison
        del comm_p, m_p, a_p, o_p, m_q, a_q, o_q, e_p, e_q
        ext.set_grad_peers(0, 0, [], 0, 1)
        # general all-reduce through our own kernel (K-FAC factor path): odd sizes, packing, avg
        torch.manual_seed(77 + rank)
        ts = [torch.randn(1025, 1025, device=dev), torch.randn(7, device=dev), torch.randn(300, 64, device=dev).t()]
        refs = [t.detach().clone(memory_format=torch.contiguous_format) for t in ts]
        comm.all_reduce_many_(ts, op="avg")
        for r in refs:
            dist.all_reduce(r, op=dist.ReduceOp.AVG)
        torch.cuda.synchronize()
        out[f"allreduce_many_err_mc{int(mc)}"] = max(float((t - r).abs().max()) for t, r in zip(ts, refs))
        big_t = torch.randn(64 << 20, device=dev)
        def run_ar():
            comm.all_reduce_many_([big_t], op="sum")
        def run_nccl():
            dist.all_reduce(big_t)
        for name, fn in (("peer", run_ar), ("nccl", run_nccl)):
            for _ in range(2):
                fn()
            torch.cuda.synchronize(); dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                fn()
            e1.record(); torch.cuda.synchronize()
            tt = torch.tensor([e0.elapsed_time(e1) / 5], device=dev)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            out[f"allreduce_256MB_{name}_ms_mc{int(mc)}"] = round(float(tt), 3)
            big_t.normal_()
        del comm, m_f, a_f, o_f, big_t
    if "--big" in sys.argv:
        big = BertConfig(vocab_size_or_config_json_file=30528, hidden_size=1024, num_hidden_layers=24,
                         num_attention_heads=16, intermediate_size=4096, max_position_embeddings=512)
        for mc in (False, True):
            m_f, a_f, o_f, comm = build(big, dev, True, use_mc=mc)
            if mc and not comm.use_multicast:
                continue
            def run_fused():
                comm.fused_lamb_step(o_f, loss_scale=1.0)
            def timeit(fn, n=6):
                for _ in range(2):
                    fn()
                torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(n):
                    fn()
                e1.record(); torch.cuda.synchronize()
                t = torch.tensor([e0.elapsed_time(e1) / n], device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                return float(t)
            a_f.flat_grad.normal_()
            t_f = timeit(run_fused)
            out[f"fused_ms_mc{int(mc)}"] = round(t_f, 3)
            comm.push_master = False                         # ZeRO-1 style: only bf16 weights + fp32 1-D tensors travel
            out[f"fused_ms_mc{int(mc)}_master_local"] = round(timeit(run_fused), 3)
            comm.push_master = True
            # with the weight-gradient tiles already reduced by the GEMM epilogues (push mode), phase A is local for 90 %
            eng_names = [s_.name for s_ in a_f.slots if s_.name.endswith(".weight") and ".encoder.layer." in s_.name
                         and "LayerNorm" not in s_.name]
            comm.set_prereduced(eng_names)
            def run_fused_pre():
                comm._pushed = True
                comm.fused_lamb_step(o_f, loss_scale=1.0)
            out[f"fused_ms_mc{int(mc)}_prereduced"] = round(timeit(run_fused_pre), 3)
            comm.push_master = False
            out[f"fused_ms_mc{int(mc)}_prereduced_master_local"] = round(timeit(run_fused_pre), 3)
            del comm, m_f, a_f, o_f
            torch.cuda.empty_cache()
        m_r, a_r, o_r, _ = build(big, dev, False)
        def run_ref():
            dist.all_reduce(a_r.flat_grad)
            a_r.flat_grad.mul_(1.0 / world)
            o_r.step()
        a_r.flat_grad.normal_()
        out["nccl_allreduce_plus_lamb_ms"] = round(timeit(run_ref), 3)
        n = a_r.numel
        link = 450e9   # NVLink 4 data-sheet bandwidth per direction (H100 SXM), not a measured rate
        rs_bytes = 4.0 * n * (world - 1) / world          # gradient shards pulled from the peers
        ag_bytes = 6.0 * n * (world - 1) / world          # fp32 + bf16 pushed to the peers
        out["roofline_ms_nvlink"] = round(max(rs_bytes, ag_bytes) / link * 1e3, 3)
        hbm = 3.35e12                                     # HBM3 data-sheet bandwidth (H100 SXM), not a measured rate
        lamb_bytes = (28.0 + 18.0) * n / world            # phase B (g,p,m,v in; m,v,u out) + phase C local traffic + zeroing share
        # the three phases depend on each other (global norm, trust ratios): their times add up
        out["roofline_ms_serial"] = round((rs_bytes / link + lamb_bytes / hbm + 4.0 * n / hbm + ag_bytes / link) * 1e3, 3)
        out["roofline_ms_serial_bf16_allgather"] = round((rs_bytes / link + lamb_bytes / hbm + 4.0 * n / hbm
                                                          + 2.0 * n * (world - 1) / world / link) * 1e3, 3)
        out["arena_numel"] = n
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
