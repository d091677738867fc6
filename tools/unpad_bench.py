"""Padded against unpadded (``BertModel.unpad``) fused encoder, device-timed, alternating the two modes.

    python tools/unpad_bench.py [--reps 5] [--out DIR]

Measures, at BERT-large shapes (H = 1024, 16 heads, I = 4096, 24 layers):
  * the attention forward and backward alone (B = 32, S = 512, NER lengths);
  * a ``BertForTokenClassification`` training step (forward, backward, Adam) and its evaluation forward at B = 32,
    S = 512 (``run_ner.py``'s defaults);
  * ``BertForQuestionAnswering`` prediction at S = 384 and ``run_squad.py``'s batch size 8, and at B = 64.
No CoNLL or SQuAD files are read: the sequence lengths are SYNTHETIC, drawn from seeded distributions that the script
prints (NER: sentences of a few dozen WordPiece tokens; SQuAD: about half the features are full 384-token windows of
long contexts, the rest shorter).  The same run reports the largest output difference between the two modes.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


def ner_lengths(rng, n):
    """Sentence lengths in WordPiece tokens plus [CLS] / [SEP]: log-normal, median about 24."""
    return np.clip(np.round(rng.lognormal(np.log(22), 0.55, n)), 3, 510).astype(int) + 2


def squad_lengths(rng, n, S=384):
    """Feature lengths at max_seq_length S: 45 % full windows, the rest question + a shorter context."""
    full = rng.random(n) < 0.45
    short = np.clip(np.round(rng.normal(210, 70, n)), 40, S).astype(int)
    return np.where(full, S, short)


def describe(name, lens):
    q = np.percentile(lens, [5, 25, 50, 75, 95]).round(1).tolist()
    return {"set": name, "n": int(len(lens)), "mean": round(float(np.mean(lens)), 1), "p5_25_50_75_95": q}


def mask_of(lens, S):
    lens = torch.as_tensor(np.asarray(lens), device="cuda")
    return (torch.arange(S, device="cuda")[None, :] < lens[:, None]).long()


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def alternate(fns, reps, iters, warm=2):
    """{mode: median ms} of the callables in ``fns``, run in turn ``reps`` times after ``warm`` warm-up calls each."""
    for f in fns.values():
        for _ in range(warm):
            f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ts[k].append(timed(f, iters))
    return {k: round(float(np.median(v)), 3) for k, v in ts.items()}, {k: [round(x, 3) for x in v] for k, v in ts.items()}


def large_config(S):
    from bert_pytorch_b200 import BertConfig
    cfg = BertConfig(vocab_size_or_config_json_file=30528, hidden_size=1024, num_hidden_layers=24,
                     num_attention_heads=16, intermediate_size=4096, max_position_embeddings=512)
    return cfg


def bench_attention(rng, reps, rows):
    from bert_pytorch_b200.models.fused import pack_rows
    from bert_pytorch_b200.ops import api as K
    B, S, h, H = 32, 512, 16, 1024
    lens = ner_lengths(rng, B)
    mask = mask_of(lens, S)
    pk = pack_rows(mask)
    qkv = (torch.randn(B, S, 3 * H, device="cuda") * 0.5).bfloat16()
    seqlens = torch.as_tensor(lens, device="cuda", dtype=torch.int32)
    qkv_p = qkv.view(B * S, 3 * H)[pk.rows.long()].contiguous()
    ctx, lse = K.attention_fwd(qkv, seqlens, h, p_drop=0.1, seed=1, stream=1)
    ctx_p, lse_p = K.attention_fwd(qkv_p, None, h, p_drop=0.1, seed=1, stream=1, cu_seqlens=pk.cu_seqlens, S=S)
    diff = (ctx.view(B * S, H)[pk.rows.long()].float() - ctx_p.float()).abs().max().item()
    d = (torch.randn(B, S, H, device="cuda") * 0.5).bfloat16() * mask[:, :, None].bfloat16()
    d_p = d.view(B * S, H)[pk.rows.long()].contiguous()
    med, raw = alternate({
        "padded_fwd": lambda: K.attention_fwd(qkv, seqlens, h, p_drop=0.1, seed=1, stream=1),
        "unpadded_fwd": lambda: K.attention_fwd(qkv_p, None, h, p_drop=0.1, seed=1, stream=1,
                                                cu_seqlens=pk.cu_seqlens, S=S),
        "padded_bwd": lambda: K.attention_bwd(qkv, seqlens, ctx, d, lse, h, p_drop=0.1, seed=1, stream=1),
        "unpadded_bwd": lambda: K.attention_bwd(qkv_p, None, ctx_p, d_p, lse_p, h, p_drop=0.1, seed=1, stream=1,
                                                cu_seqlens=pk.cu_seqlens, S=S),
    }, reps, iters=20)
    rows.append({"what": "attention fwd (B=32, S=512)", "padded_ms": med["padded_fwd"], "unpadded_ms": med["unpadded_fwd"],
                 "max_abs_diff": diff, "tokens": f"{pk.T}/{B * S}", "raw": {k: raw[k] for k in raw if "fwd" in k}})
    rows.append({"what": "attention bwd (B=32, S=512)", "padded_ms": med["padded_bwd"], "unpadded_ms": med["unpadded_bwd"],
                 "max_abs_diff": None, "tokens": f"{pk.T}/{B * S}", "raw": {k: raw[k] for k in raw if "bwd" in k}})


def bench_ner(rng, reps, rows):
    from bert_pytorch_b200.models import BertForTokenClassification
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Adam
    B, S, labels_n = 32, 512, 10
    torch.manual_seed(0)
    model = BertForTokenClassification(large_config(S), num_labels=labels_n).cuda()
    arena = ParamArena(model)
    opt = Adam(model.parameters(), lr=1e-5, bias_correction=False)
    arena.bind_optimizer(opt)
    lens = ner_lengths(rng, B)
    mask = mask_of(lens, S)
    ids = torch.randint(1000, 30000, (B, S), device="cuda") * mask
    tt = torch.zeros_like(mask)
    labels = torch.randint(0, labels_n, (B, S), device="cuda")

    def step(unpad):
        def f():
            model.bert.unpad = unpad
            opt.zero_grad()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = model(ids, tt, mask, labels=labels)
            loss.backward()
            opt.step()
        return f

    def evaluate(unpad):
        def f():
            model.bert.unpad = unpad
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return model(ids, tt, mask)
        return f

    model.eval()
    v = mask.bool()
    diff = (evaluate(False)()[v].float() - evaluate(True)()[v].float()).abs().max().item()
    med, raw = alternate({"padded": evaluate(False), "unpadded": evaluate(True)}, reps, iters=5)
    rows.append({"what": "NER eval forward (B=32, S=512)", "padded_ms": med["padded"], "unpadded_ms": med["unpadded"],
                 "max_abs_diff": diff, "tokens": f"{int(mask.sum())}/{B * S}", "raw": raw})
    model.train()
    med, raw = alternate({"padded": step(False), "unpadded": step(True)}, reps, iters=3)
    rows.append({"what": "NER train step fwd+bwd+Adam (B=32, S=512)", "padded_ms": med["padded"],
                 "unpadded_ms": med["unpadded"], "max_abs_diff": None, "tokens": f"{int(mask.sum())}/{B * S}", "raw": raw})
    del model, arena, opt
    torch.cuda.empty_cache()


def bench_squad(rng, reps, rows):
    from bert_pytorch_b200.models import BertForQuestionAnswering
    S = 384
    torch.manual_seed(0)
    model = BertForQuestionAnswering(large_config(S)).cuda().eval()
    for B in (8, 64):
        lens = squad_lengths(rng, B)
        mask = mask_of(lens, S)
        ids = torch.randint(1000, 30000, (B, S), device="cuda") * mask
        seg = (torch.arange(S, device="cuda")[None, :] > 20).long() * mask

        def pred(unpad):
            def f():
                model.bert.unpad = unpad
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                    return model(ids, seg, mask)
            return f
        v = mask.bool()
        a, b = pred(False)(), pred(True)()
        diff = max((x[v].float() - y[v].float()).abs().max().item() for x, y in zip(a, b))
        med, raw = alternate({"padded": pred(False), "unpadded": pred(True)}, reps, iters=10 if B == 8 else 3)
        rows.append({"what": f"SQuAD prediction (B={B}, S=384)", "padded_ms": med["padded"], "unpadded_ms": med["unpadded"],
                     "max_abs_diff": diff, "tokens": f"{int(mask.sum())}/{B * S}", "raw": raw})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for unpad_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unpad_bench needs a GPU")
    from bert_pytorch_b200 import ops
    assert ops.available(), "sm_90a extension not built"
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rng = np.random.default_rng(2024)
    print(json.dumps({"synthetic_lengths": [describe("NER (B=32 x 200 draws)", ner_lengths(np.random.default_rng(1), 6400)),
                                            describe("SQuAD features", squad_lengths(np.random.default_rng(1), 6400))]}),
          flush=True)
    rows = []
    bench_attention(rng, args.reps, rows)
    bench_ner(rng, args.reps, rows)
    bench_squad(rng, args.reps, rows)
    for r in rows:
        r["speedup"] = round(r["padded_ms"] / r["unpadded_ms"], 2)
        print(json.dumps(r), flush=True)
    print(f"\nSynthetic sequence lengths; {info['name']}, power limit {info.get('power_limit')}; median of {args.reps} "
          "alternated runs, device events")
    print("| Workload | Tokens computed (unpadded / padded) | Padded (ms) | Unpadded (ms) | Speed-up | Max |diff| |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        d = "n/a" if r["max_abs_diff"] is None else f"{r['max_abs_diff']:.3g}"
        print(f"| {r['what']} | {r['tokens']} | {r['padded_ms']} | {r['unpadded_ms']} | {r['speedup']}x | {d} |")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "unpad_bench.json"), "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
