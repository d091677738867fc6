"""Cost of deterministic mode: BERT-large pre-training micro-steps and one arena-LAMB step, device-timed, with the mode
off and on, alternating.

    python tools/deterministic_bench.py [--reps 5] [--steps 4] [--out DIR]

The workload is ``FusedPretrainer.forward_backward`` of BERT-large (H = 1024, 24 layers, 16 heads, I = 4096, vocabulary
30528, NSP on) with CUDA graphs, dropout 0.1 and bf16, padded, at the phase-1 shape (S = 128, B = 96, 20 predictions)
and the phase-2 shape (S = 512, B = 16, 80 predictions), and the arena-LAMB step over its 336 M parameters.  The modes
alternate ``--reps`` times (each mode replays its own graph) and the median window is reported.  The eager program
(no graphs) then runs in deterministic mode with and without torch's flag and its fill of uninitialised memory, which
the runners' ``--deterministic`` turns off (the graphs of both would be the same key).  Then each deterministic site is timed alone at the BERT-large shapes
against its default form (CUDA events over 20 calls, once per layer where the step runs it once per layer).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from pretrain_unpad_bench import SHAPES, card, make_batch, synthetic_masks, window  # noqa: E402


def set_mode(mode):
    os.environ["B200_DETERMINISTIC"] = "1" if mode == "on" else "0"
    torch.use_deterministic_algorithms(mode == "torch+fill")
    torch.utils.deterministic.fill_uninitialized_memory = True      # only acts under torch's flag


def event_ms(fn, iters=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def sites(S, B):
    """(name, per-step count, fn) of every site whose form differs, at the BERT-large shapes of one micro-step"""
    from bert_pytorch_b200.ops import api as K
    H, I, V, M = 1024, 4096, 30528, B * S
    r = lambda *s: torch.randn(*s, device="cuda").bfloat16()      # noqa: E731
    dy, x, dq3, y1 = r(M, H), r(M, H), r(M, 3 * H), r(M, I)
    w2 = r(H, I)
    g = torch.zeros(H, H, device="cuda")
    cs = torch.zeros(I, device="cuda")
    gamma, beta = torch.ones(H, device="cuda"), torch.zeros(H, device="cuda")
    _, mean, rstd = K.layer_norm_fwd(x, gamma, beta)
    ids = torch.randint(0, V, (M,), device="cuda", dtype=torch.int32)
    seg = torch.randint(0, 2, (M,), device="cuda", dtype=torch.int32)
    gw, gp, gt = torch.zeros(V, H, device="cuda"), torch.zeros(512, H, device="cuda"), torch.zeros(2, H, device="cuda")
    qkv, dctx = r(B, S, 3 * H), r(B, S, H)
    seqlens = torch.full((B,), S, dtype=torch.int32, device="cuda")
    ctx, lse = K.attention_fwd(qkv, seqlens, 16, p_drop=0.1, seed=1, stream=1)
    return [
        ("wgrad [H, H] (split-K in order)", 2, lambda: K.wgrad_accumulate(dy, x, g)),
        ("FFN-1 dgrad + bias column sum", 1, lambda: K.gemm(dy, w2, layout=K.NN, epi=K.EPI_MUL, res=y1, colsum=cs)),
        ("QKV bias column sum", 1, lambda: K.colsum_accumulate(dq3, cs[:3 * H])),
        ("LayerNorm backward", 2, lambda: K.layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma=cs[:H], dbeta=cs[H:2 * H],
                                                           dbias=cs[2 * H:3 * H], want_dropped=True)),
        ("attention backward", 1, lambda: K.attention_bwd(qkv, seqlens, ctx, dctx, lse, 16, p_drop=0.1, seed=1, stream=1)),
        ("embedding backward", 1 / 24, lambda: K.embedding_bwd_scatter(dy, ids, seg, gw, gp, gt, S)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--shapes", default="phase1,phase2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    from bert_pytorch_b200 import BertConfig, ops
    from bert_pytorch_b200.models import BertForPreTraining
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Lamb
    assert ops.available(), "sm_90a extension not built"
    info = {"card": card(), "rows": [], "sites": []}
    print(json.dumps(info["card"]), flush=True)
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=30528, hidden_size=1024, num_hidden_layers=24,
                     num_attention_heads=16, intermediate_size=4096, max_position_embeddings=512)
    modes = ("off", "on")
    step_ms = {}
    for shape in a.shapes.split(","):
        S, B, mp = SHAPES[shape]
        cfg.max_predictions_per_seq = mp
        model = BertForPreTraining(cfg).cuda()
        arena = ParamArena(model)
        opt = Lamb([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-4)
        arena.bind_optimizer(opt)
        model.train()
        pt = model.pretrain_engine()
        rng = np.random.default_rng(1)
        batches = [make_batch(m, cfg.vocab_size, mp, rng) for m in synthetic_masks(rng, S, B, 0.95, a.steps)]
        tokens = [None] * len(batches)
        res, lamb = {}, {}
        for mode in modes:                               # warm-up: eager calls, then the capture of each mode's graph
            set_mode(mode)
            for _ in range(pt.graph_warmup + 1):
                window(pt, batches, tokens)
        for _ in range(a.reps):
            for mode in modes:
                set_mode(mode)
                res.setdefault(mode, []).append(window(pt, batches, tokens))
                lamb.setdefault(mode, []).append(event_ms(opt.step, iters=5))
            arena.zero_grad()
        pt.use_graphs = False
        for _ in range(a.reps):
            for mode in ("on", "torch+fill"):
                set_mode(mode)
                res.setdefault("eager " + mode, []).append(window(pt, batches, tokens))
            arena.zero_grad()
        set_mode("off")
        med = {m: float(np.median(v)) for m, v in res.items()}
        step_ms[shape] = med["off"]
        row = {"shape": shape, "S": S, "B": B, "micro_step_ms": {m: round(v, 3) for m, v in med.items()},
               "on_over_off": round(med["on"] / med["off"], 4),
               "eager_torch_fill_over_eager_on": round(med["eager torch+fill"] / med["eager on"], 4),
               "spread_ms": {m: round(float(np.ptp(v)), 3) for m, v in res.items()},
               "lamb_step_ms": {m: round(float(np.median(v)), 3) for m, v in lamb.items()}}
        info["rows"].append(row)
        print(json.dumps(row), flush=True)
        del pt, model, arena, opt
        torch.cuda.empty_cache()
        for name, per_layer, fn in sites(S, B):
            t = {}
            for mode in ("off", "on"):
                set_mode(mode)
                t[mode] = event_ms(fn)
            set_mode("off")
            extra = (t["on"] - t["off"]) * per_layer * 24
            site = {"shape": shape, "site": name, "off_ms": round(t["off"], 4), "on_ms": round(t["on"], 4),
                    "extra_ms_per_micro_step": round(extra, 3),
                    "share_of_micro_step": round(extra / step_ms[shape], 4)}
            info["sites"].append(site)
            print(json.dumps(site), flush=True)
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "deterministic_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
