"""Loss curves on a LEARNABLE synthetic corpus (data/synthetic.py:learnable_tokens) for the same model / data / LAMB
schedule through three execution paths -- VERDICT r1 #7 / #8:

    oracle-fp32   plain PyTorch autograd, fp32 everywhere (bert.use_fused = False)
    fused-bf16    the sm_90a kernel program (bf16 operands, fp32 accumulate / master weights)
    fused-fp8     same engine with per-tensor delayed-scaling fp8 GEMM operands (e4m3 fwd / e5m2 grads)

    python tools/convergence.py [--steps 300] [--hidden 1024 --layers 4] > convergence.jsonl

One JSON line per arm with the per-step MLM+NSP loss (dropout off so the three arms see the same function), then a
summary line with the final-loss ratios (mean of the last 10 % of the steps)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bert_pytorch_b200 import BertConfig  # noqa: E402
from bert_pytorch_b200.data import synthetic  # noqa: E402
from bert_pytorch_b200.data.dataset import mask_batch, segment_ids_and_input_mask  # noqa: E402
from bert_pytorch_b200.models import BertForPreTraining, BertPretrainingCriterion  # noqa: E402
from bert_pytorch_b200.models.arena import NO_DECAY_KEYS, ParamArena  # noqa: E402
from bert_pytorch_b200.optim import Lamb, PolyWarmUpScheduler  # noqa: E402


def batches(n, B, S, V, max_pred, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        ids, sp, nsl = synthetic.make_samples(B, S, V, True, rng, learnable=True)
        seg, im = segment_ids_and_input_mask(ids, sp)
        masked, labels = mask_batch(ids, sp, mask_token_index=4, max_pred_per_seq=max_pred, masked_lm_prob=0.15,
                                    vocab_size=V, rng=rng)
        out.append([torch.from_numpy(np.ascontiguousarray(a)).to(torch.int32).cuda()
                    for a in (masked, seg, im, labels, nsl.astype(np.int32))])
    return out


def run(arm, args, data):
    torch.manual_seed(1234)
    cfg = BertConfig(vocab_size_or_config_json_file=args.vocab, hidden_size=args.hidden, num_hidden_layers=args.layers,
                     num_attention_heads=args.hidden // 64, intermediate_size=4 * args.hidden,
                     max_position_embeddings=args.seq, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg.max_predictions_per_seq = args.max_pred
    model = BertForPreTraining(cfg).cuda()
    model.train()
    named = list(model.named_parameters())
    groups = [{"params": [p for n, p in named if not any(k in n for k in NO_DECAY_KEYS)], "weight_decay": 0.01},
              {"params": [p for n, p in named if any(k in n for k in NO_DECAY_KEYS)], "weight_decay": 0.0}]
    opt = Lamb(groups, lr=args.lr)
    crit = BertPretrainingCriterion(cfg.vocab_size)
    eng = None
    if arm == "oracle-fp32":
        model.bert.use_fused = False
    else:
        arena = ParamArena(model)
        arena.bind_optimizer(opt)
        eng = model.pretrain_engine()
        if arm == "fused-fp8":
            model.bert.fused_engine().enable_fp8()
    sched = PolyWarmUpScheduler(opt, warmup=0.1, total_steps=args.steps)
    losses = []
    for step in range(args.steps):
        ids, seg, mask, labels, nsl = data[step % len(data)]
        if eng is not None:
            loss = eng.forward_backward(ids, seg, mask, labels, nsl, grad_scale=1.0)
        else:
            scores, nsp = model(ids.long(), seg.long(), mask.long())
            loss = crit(scores, labels.long(), nsp, nsl.long())
            loss.backward()
        sched.step()
        opt.step()
        opt.zero_grad()
        losses.append(round(float(loss), 5))
    return losses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--vocab", type=int, default=1024)
    ap.add_argument("--max-pred", type=int, default=20)
    ap.add_argument("--lr", type=float, default=2e-3)
    ap.add_argument("--arms", default="oracle-fp32,fused-bf16,fused-fp8")
    args = ap.parse_args()
    data = batches(64, args.batch, args.seq, args.vocab, args.max_pred, seed=7)
    tail = max(1, args.steps // 10)
    finals = {}
    for arm in args.arms.split(","):
        losses = run(arm, args, data)
        finals[arm] = sum(losses[-tail:]) / tail
        print(json.dumps({"arm": arm, "config": vars(args), "first_loss": losses[0], "final_loss_mean_last_10pct": round(finals[arm], 5),
                          "loss": losses}), flush=True)
    ref = finals.get("oracle-fp32")
    if ref:
        print(json.dumps({"summary": {a: {"final": round(v, 5), "rel_to_oracle": round(v / ref - 1.0, 5)} for a, v in finals.items()},
                          "criteria": "fused-bf16 within 1 %, fused-fp8 within 3 % of the oracle's final loss"}), flush=True)


if __name__ == "__main__":
    main()
