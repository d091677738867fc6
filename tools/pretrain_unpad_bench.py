"""Padded against unpadded (``--unpad``) BERT-large pre-training micro-steps, device-timed, alternating the two modes.

    python tools/pretrain_unpad_bench.py [--reps 5] [--steps 4] [--input_dir DIR] [--out DIR]

The workload is ``FusedPretrainer.forward_backward`` of BERT-large (H = 1024, 24 layers, 16 heads, I = 4096, vocabulary
30528, NSP on) with CUDA graphs, dropout 0.1 and bf16, at the phase-1 shape (S = 128, B = 96, 20 predictions per
sequence) and the phase-2 shape (S = 512, B = 16, 80 predictions), the shipped per-GPU micro-batches.  Each timed
window runs ``--steps`` micro-steps over as many distinct batches; the modes alternate ``--reps`` times and the median
window is reported.

Sequence lengths are SYNTHETIC and seeded: per sequence uniform on [(2f - 1) S, S] for a mean fill f of about 0.95
(today's synthetic shards), 0.75 and 0.50, plus f = 1 (every token real: the cost of the unpadded path itself -- the
pack kernel, the dummy-sequence CTAs and varlen instead of padded attention).  ``--input_dir`` takes the masks from
real HDF5 shards instead and prints their fill.  Reported per case: the card, T / T_cap waste, the graphs captured,
both step times and the ratio; plus the pack kernel alone.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"phase1": (128, 96, 20), "phase2": (512, 16, 80)}


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


def synthetic_masks(rng, S, B, fill, n):
    lo = max(1, int(round((2 * fill - 1) * S)))
    out = []
    for _ in range(n):
        lens = rng.integers(lo, S + 1, B) if fill < 1 else np.full(B, S)
        out.append((np.arange(S)[None, :] < lens[:, None]).astype(np.int32))
    return out


def shard_masks(input_dir, S, B, n):
    from bert_pytorch_b200.data import BatchedPretrainingLoader, DistributedSampler, ShardedPretrainingDataset
    from bert_pytorch_b200.pretrain import find_input_files
    ds = ShardedPretrainingDataset(find_input_files(input_dir), 4, 20, 0.15, vocab_size=30528, seed=0)
    loader = BatchedPretrainingLoader(ds, DistributedSampler(ds, 1, rank=0, seed=0), B, pin_memory=False)
    out = []
    for batch in loader:
        m = batch[2].numpy().astype(np.int32)
        if m.shape[1] != S:
            raise SystemExit(f"shards have S = {m.shape[1]}, this case needs {S}")
        out.append(m)
        if len(out) == n:
            break
    loader.close()
    return out


def make_batch(mask, V, mp, rng):
    B, S = mask.shape
    ids = rng.integers(5, V, (B, S)).astype(np.int32) * mask
    seg = ((np.arange(S)[None, :] > mask.sum(1, keepdims=True) // 2) & (mask > 0)).astype(np.int32)
    labels = np.full((B, S), -1, np.int32)
    for b in range(B):
        n = max(int(mask[b].sum()), 1)
        p = rng.choice(n, min(mp, max(1, int(0.15 * n))), replace=False)
        labels[b, p] = ids[b, p]
    nsl = rng.integers(0, 2, B).astype(np.int32)
    return [torch.from_numpy(a).cuda() for a in (ids, seg, mask, labels, nsl)]


def window(pt, batches, tokens):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for b, t in zip(batches, tokens):
        pt.forward_backward(*b, tokens=t)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / len(batches)


def pack_kernel_ms(mask, T_cap, D, iters=200):
    from bert_pytorch_b200.ops import api as K
    m = torch.from_numpy(mask).cuda()
    for _ in range(10):
        K.pack_tokens(m, m, m, T_cap, D)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        K.pack_tokens(m, m, m, T_cap, D)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--shapes", default="phase1,phase2")
    ap.add_argument("--fills", default="1.0,0.95,0.75,0.5")
    ap.add_argument("--input_dir", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    from bert_pytorch_b200 import BertConfig, ops
    from bert_pytorch_b200.models import BertForPreTraining
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.models.fused import packed_tokens, token_bucket
    assert ops.available(), "sm_90a extension not built"
    info = {"card": card(), "rows": []}
    print(json.dumps(info["card"]), flush=True)
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=30528, hidden_size=1024, num_hidden_layers=24,
                     num_attention_heads=16, intermediate_size=4096, max_position_embeddings=512)
    for shape in a.shapes.split(","):
        S, B, mp = SHAPES[shape]
        cfg.max_predictions_per_seq = mp
        model = BertForPreTraining(cfg).cuda()
        arena = ParamArena(model)
        model.train()
        pt = model.pretrain_engine()
        rng = np.random.default_rng(1)
        sets = [("shards", shard_masks(a.input_dir, S, B, a.steps))] if a.input_dir else \
            [(f"fill {f}", synthetic_masks(rng, S, B, float(f), a.steps)) for f in a.fills.split(",")]
        for name, ms in sets:
            batches = [make_batch(m, cfg.vocab_size, mp, rng) for m in ms]
            tokens = [packed_tokens(torch.from_numpy(m)) for m in ms]
            caps = [token_bucket(t, B, S)[0] for t in tokens]
            res = {}
            n_graphs0 = sum("graph" in e for e in pt._graphs.values())
            for unpad in (False, True):                   # warm-up: eager calls, then the capture of every bucket
                model.bert.unpad = unpad
                for _ in range(pt.graph_warmup + 1):
                    window(pt, batches, tokens)
            graphs = sum("graph" in e for e in pt._graphs.values()) - n_graphs0
            for _ in range(a.reps):
                for unpad in (False, True):
                    model.bert.unpad = unpad
                    res.setdefault(unpad, []).append(window(pt, batches, tokens))
                arena.zero_grad()
            pad_ms, unpad_ms = float(np.median(res[False])), float(np.median(res[True]))
            T_cap, D = token_bucket(tokens[0], B, S)
            row = {"shape": shape, "S": S, "B": B, "set": name, "fill": round(sum(tokens) / (len(tokens) * B * S), 4),
                   "T_over_T_cap": round(sum(tokens) / sum(caps), 4), "graphs_captured": graphs,
                   "padded_ms": round(pad_ms, 3), "unpadded_ms": round(unpad_ms, 3),
                   "unpadded_over_padded": round(unpad_ms / pad_ms, 4),
                   "spread_ms": [round(float(np.ptp(res[False])), 3), round(float(np.ptp(res[True])), 3)],
                   "pack_kernel_ms": round(pack_kernel_ms(ms[0], T_cap, D), 4)}
            info["rows"].append(row)
            print(json.dumps(row), flush=True)
        model.bert.unpad = False
        del pt, model, arena
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pretrain_unpad_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
