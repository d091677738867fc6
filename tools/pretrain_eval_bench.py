"""Cost of the held-out evaluation of BERT-large pre-training, device-timed.

    python tools/pretrain_eval_bench.py [--reps 5] [--batches 4] [--out DIR]

BERT-large (H = 1024, 24 layers, 16 heads, I = 4096, vocabulary 30528, NSP on), bf16, at the phase-1 shape (S = 128,
batch 96, 20 predictions per sequence) and the phase-2 shape (S = 512, batch 16, 80 predictions), the shipped per-GPU
micro-batches.  Timed per case, in sequences per second:

* ``fused``: ``FusedPretrainer.evaluate`` with CUDA graphs, padded and unpadded (``BertModel.unpad``);
* ``torch``: the plain PyTorch forward under bf16 autocast plus the same metric sums (padded only).

Sequence lengths are synthetic and seeded: uniform on [S / 2, S] (mean fill about 0.75).  Each window evaluates
``--batches`` distinct batches and ends in a device synchronise; the arms alternate ``--reps`` times and the median
window is reported.  One training micro-step of the fused program (graphs, dropout 0.1) is timed the same way, and the
cost of a 10000-sample evaluation is given in optimizer steps at the shipped accumulation (the micro-steps of one step,
LAMB left out: phase 1 86 x 96 sequences, phase 2 256 x 16 per GPU, the 65536 / 32768 global batches on 8 GPUs).  The card's name and power limit are
read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"phase1": (128, 96, 20, 86), "phase2": (512, 16, 80, 256)}   # S, B, max_pred, accumulation steps
V = 30528


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


def batches(S, B, mp, n, seed):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        lens = g.integers(S // 2, S + 1, B)
        mask = (np.arange(S)[None, :] < lens[:, None]).astype(np.int32)
        ids = g.integers(5, V, (B, S)).astype(np.int32) * mask
        seg = ((np.arange(S)[None, :] > lens[:, None] // 2) & (mask > 0)).astype(np.int32)
        labels = np.full((B, S), -1, np.int32)
        for b in range(B):
            p = g.choice(np.arange(1, lens[b]), size=min(mp, int(lens[b]) - 1), replace=False)
            labels[b, p] = ids[b, p]
        nsl = g.integers(0, 2, B).astype(np.int32)
        out.append([torch.from_numpy(a).cuda() for a in (ids, seg, mask, labels, nsl)])
    return out


def model(S, mp):
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    from bert_pytorch_b200.models.arena import ParamArena
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=V, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                     intermediate_size=4096, max_position_embeddings=512)
    cfg.max_predictions_per_seq = mp
    m = BertForPreTraining(cfg).cuda()
    arena = ParamArena(m)                   # the engine holds the arena weakly: the caller keeps it
    m.train()
    return m, arena


def window(fn, data) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in data:
        fn(b)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--shapes", default="phase1,phase2")
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from bert_pytorch_b200.models.fused import packed_tokens
    from bert_pytorch_b200.models.modeling import _metric_sums
    res = {"card": card(), "cases": {}}
    for shape in a.shapes.split(","):
        S, B, mp, acc_steps = SHAPES[shape]
        m, arena = model(S, mp)
        pt = m.pretrain_engine()
        data = batches(S, B, mp, a.batches, seed=S)
        toks = {id(b): packed_tokens(b[2].cpu()) for b in data}
        acc = torch.zeros(6, dtype=torch.float64, device="cuda")

        def fused_padded(b):
            m.bert.unpad = False
            pt.evaluate(*b, acc)

        def fused_unpadded(b):
            m.bert.unpad = True
            pt.evaluate(*b, acc, tokens=toks[id(b)])

        def plain(b):
            m.bert.use_fused = False
            was = m.training
            m.eval()
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                scores, nsp = m(b[0].long(), b[1].long(), b[2].long())
                acc[0:3] += _metric_sums(scores.view(-1, V), b[3].view(-1))
                acc[3:6] += _metric_sums(nsp, b[4])
            m.train(was)
            m.bert.use_fused = True

        def train(b):
            m.bert.unpad = False
            pt.forward_backward(*b, grad_scale=1.0 / acc_steps)

        arms = {"fused_padded": fused_padded, "fused_unpadded": fused_unpadded, "torch_bf16_padded": plain,
                "train_micro_step": train}
        times = {k: [] for k in arms}
        for k, fn in arms.items():                       # warm-up: every signature captured and replayed
            for _ in range(pt.graph_warmup + 2):
                window(fn, data)
        for _ in range(a.reps):
            for k, fn in arms.items():
                times[k].append(window(fn, data))
        case = {"S": S, "B": B, "max_pred": mp, "fill": float(np.mean([b[2].float().mean().item() for b in data]))}
        for k, ts in times.items():
            med = statistics.median(ts)
            case[k] = {"ms_per_batch": round(1e3 * med / a.batches, 3), "seq_per_s": round(a.batches * B / med, 1),
                       "spread": round((max(ts) - min(ts)) / med, 4)}
        step_s = acc_steps * case["train_micro_step"]["ms_per_batch"] / 1e3
        for k in ("fused_padded", "fused_unpadded", "torch_bf16_padded"):
            secs = 10000 / case[k]["seq_per_s"]
            case[k]["s_per_10000"] = round(secs, 2)
            case[k]["optimizer_steps_per_10000"] = round(secs / step_s, 3)
        case["optimizer_step_s"] = round(step_s, 3)
        res["cases"][shape] = case
        print(json.dumps({shape: case}), flush=True)
        del pt, m, arena
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pretrain_eval_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
