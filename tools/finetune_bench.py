"""Cost of SQuAD and NER fine-tuning steps and prediction batches on BERT-large, device-timed, fused against module.

    python tools/finetune_bench.py [--reps 5] [--steps 4] [--out DIR]

BERT-large (H = 1024, 24 layers, 16 heads, I = 4096, vocabulary 30528).  Sequence lengths are the seeded synthetic
ones of ``tools/unpad_bench.py`` (``squad_lengths``: 45 % full 384-token windows; ``ner_lengths``: sentences of a few
dozen WordPiece tokens).  Workloads:

* SQuAD training step, B = 32, S = 384: forward, loss, backward, gradient clipping at 1.0 and arena Adam (padded: the
  span softmax normalises over every position);
* SQuAD prediction, S = 384, B = 8 (``run_squad.py``'s default) and 64, padded and unpadded;
* NER training step (the same optimizer work) and evaluation batch, B = 32, S = 512 (``run_ner.py``'s defaults), 10
  labels, padded and unpadded.

Arms: ``module`` is today's ``forward`` under bf16 autocast (+ ``loss.backward()``) through the autograd bridge of the
fused encoder (unpadded: ``pack_rows``, one host sync per batch); ``fused`` is ``train_step`` / ``predict`` of the
fused program, eager (``use_graphs = False``) and replayed as CUDA graphs.  Every window runs ``--steps`` distinct
batches and ends in a device synchronise, timed with CUDA events; the arms alternate ``--reps`` times, in an order
rotated every round, and the median and the spread (min - max) of the windows are reported in ms per batch.  The head
alone (``token_logits`` + loss + ``token_head_bwd`` against ``head_linear`` forward and backward) is timed too.  The card's name, power limit and max SM clock
are read in the same run, and the same run checks that the fused and the module losses and logits agree at these sizes
(dropout off).
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.unpad_bench import card, ner_lengths, squad_lengths   # noqa: E402

V, NER_LABELS = 30528, 10


def _config():
    from bert_pytorch_b200 import BertConfig
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = BertConfig.from_json_file(os.path.join(root, "config", "bert_large_uncased_config.json"))
    cfg.vocab_size = V
    return cfg


def _mask(lens, S):
    return (np.arange(S)[None, :] < np.asarray(lens)[:, None]).astype(np.int64)


def squad_batches(n, B, seed, S=384):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        mask = _mask(squad_lengths(g, B, S), S)
        ids = g.integers(1000, V, (B, S)) * mask
        seg = (np.arange(S)[None, :] > 20).astype(np.int64) * mask
        sp = g.integers(21, 200, B)
        ep = sp + g.integers(0, 20, B)
        out.append(([torch.from_numpy(t).cuda() for t in (ids, seg, mask, sp, ep)], int(mask.sum())))
    return out


def ner_batches(n, B, seed, S=512):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        lens = ner_lengths(g, B)
        mask = _mask(lens, S)
        ids = g.integers(1000, V, (B, S)) * mask
        labels = g.integers(1, NER_LABELS, (B, S))
        labels[:, 0] = -100
        labels[np.arange(B), lens - 1] = -100
        out.append(([torch.from_numpy(t).cuda() for t in (ids, np.zeros_like(ids), mask, labels)], int(mask.sum())))
    return out


def time_arms(arms, data, fn, reps, rows, **tags):
    """Alternate ``arms`` over ``reps`` windows of ``data``, the order rotated by one arm per round (under the power
    cap a window's clock depends on the load of the window before it); append one row per arm."""
    for arm in arms:                                      # warm-up: every shape, bucket and graph of the windows
        for b in data:
            for _ in range(3 if arm[1] else 1):
                fn(arm, b)
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for i in range(reps):
        for arm in arms[i % len(arms):] + arms[:i % len(arms)]:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for b in data:
                fn(arm, b)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1) / len(data))
    for (path, graphs), ts in times.items():
        row = dict(tags, path=path, graphs=graphs, ms_median=round(statistics.median(ts), 3),
                   ms_min=round(min(ts), 3), ms_max=round(max(ts), 3))
        rows.append(row)
        print(json.dumps(row), flush=True)


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def bench_squad(args, rows, checks):
    from bert_pytorch_b200.finetune_squad import squad_loss
    from bert_pytorch_b200.models import BertForQuestionAnswering
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Adam, GradientClipper
    torch.manual_seed(0)
    model = BertForQuestionAnswering(_config()).cuda()
    arena = ParamArena(model)
    opt = Adam([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-7, bias_correction=False)
    arena.bind_optimizer(opt)
    clip = GradientClipper(max_grad_norm=1.0)
    eng = model.qa_engine()
    train = squad_batches(args.steps, 32, seed=1)

    # agreement, dropout off: the training loss and the start / end logits of both paths
    model.eval()
    (ids, seg, mask, sp, ep), tok = train[0]
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        s_m, e_m = model(ids, seg, mask)
        loss_m = squad_loss(s_m, e_m, sp, ep)
    loss_f = model.train_step(ids, seg, mask, sp, ep)
    s_f, e_f = model.predict(ids, seg, mask)
    opt.zero_grad()
    scale = max(s_m.float().abs().max().item(), e_m.float().abs().max().item())
    checks.append(dict(what="SQuAD train loss (B=32)", module=float(loss_m), fused=float(loss_f),
                       rel_diff=_rel(loss_f, loss_m), ok=_rel(loss_f, loss_m) <= 2e-2))
    diff = max((s_f - s_m.float()).abs().max().item(), (e_f - e_m.float()).abs().max().item()) / scale
    checks.append(dict(what="SQuAD logits (B=32)", max_abs_diff_over_max=diff, ok=diff <= 3e-2))
    model.train()

    def step(arm, batch):
        (ids, seg, mask, sp, ep), _ = batch
        eng.use_graphs = arm[1]
        if arm[0] == "module":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = squad_loss(*model(ids, seg, mask), sp, ep)
            loss.backward()
        else:
            model.train_step(ids, seg, mask, sp, ep)
        clip.step(model.parameters())
        opt.step()
        opt.zero_grad()

    model.bert.unpad = False
    time_arms([("module", False), ("fused", False), ("fused", True)], train, step, args.reps, rows,
              task="SQuAD", what="train", B=32, S=384, fill=round(sum(t for _, t in train) / (len(train) * 32 * 384), 3))

    def pred(arm, batch):
        (ids, seg, mask, *_), tok = batch
        model.bert.unpad = arm[0].endswith("unpad")
        eng.use_graphs = arm[1]
        if arm[0].startswith("module"):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                model(ids, seg, mask)
        else:
            model.predict(ids, seg, mask, tokens=tok)

    model.eval()
    for B in (8, 64):
        data = squad_batches(args.steps, B, seed=10 + B)
        (ids, seg, mask, *_), tok = data[0]
        v = mask.bool()
        for unpad in (False, True):
            model.bert.unpad = unpad
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                s_m, e_m = model(ids, seg, mask)
            s_f, e_f = model.predict(ids, seg, mask, tokens=tok)
            scale = max(s_m[v].float().abs().max().item(), e_m[v].float().abs().max().item())
            diff = max((s_f[v] - s_m[v].float()).abs().max().item(), (e_f[v] - e_m[v].float()).abs().max().item())
            checks.append(dict(what=f"SQuAD prediction logits (B={B}, unpad={unpad})", max_abs_diff_over_max=diff / scale,
                               ok=diff / scale <= 3e-2))
        arms = [("module", False), ("module-unpad", False), ("fused", False), ("fused", True), ("fused-unpad", False),
                ("fused-unpad", True)]
        time_arms(arms, data, pred, args.reps, rows, task="SQuAD", what="predict", B=B, S=384,
                  fill=round(sum(t for _, t in data) / (len(data) * B * 384), 3))
    del model, arena, opt, eng
    torch.cuda.empty_cache()


def bench_ner(args, rows, checks):
    from bert_pytorch_b200.models import BertForTokenClassification
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.models.modeling import token_loss
    from bert_pytorch_b200.optim import Adam, GradientClipper
    torch.manual_seed(0)
    model = BertForTokenClassification(_config(), NER_LABELS).cuda()
    arena = ParamArena(model)
    opt = Adam(model.parameters(), lr=1e-7, bias_correction=False)
    arena.bind_optimizer(opt)
    clip = GradientClipper(5.0)
    eng = model.token_engine()
    data = ner_batches(args.steps, 32, seed=3)

    model.eval()
    (ids, seg, mask, labels), tok = data[0]
    v = mask.bool()
    for unpad in (False, True):
        model.bert.unpad = unpad
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            lg_m = model(ids, seg, mask).float()
        loss_m = token_loss(lg_m, labels, mask)
        loss_f = model.train_step(ids, seg, mask, labels, tokens=tok)
        lg_f = model.predict(ids, seg, mask, tokens=tok)
        opt.zero_grad()
        checks.append(dict(what=f"NER train loss (unpad={unpad})", module=float(loss_m), fused=float(loss_f),
                           rel_diff=_rel(loss_f, loss_m), ok=_rel(loss_f, loss_m) <= 2e-2))
        diff = (lg_f[v] - lg_m[v]).abs().max().item() / lg_m[v].abs().max().item()
        checks.append(dict(what=f"NER logits (unpad={unpad})", max_abs_diff_over_max=diff, ok=diff <= 3e-2))

    def step(arm, batch):
        (ids, seg, mask, labels), tok = batch
        model.bert.unpad = arm[0].endswith("unpad")
        eng.use_graphs = arm[1]
        opt.zero_grad()
        if arm[0].startswith("module"):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = model(ids, seg, mask, labels=labels)
            loss.backward()
        else:
            model.train_step(ids, seg, mask, labels, tokens=tok)
        clip.step(model.parameters())
        opt.step()

    def evaluate(arm, batch):
        (ids, seg, mask, _), tok = batch
        model.bert.unpad = arm[0].endswith("unpad")
        eng.use_graphs = arm[1]
        if arm[0].startswith("module"):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                model(ids, seg, mask)
        else:
            model.predict(ids, seg, mask, tokens=tok)

    arms = [("module", False), ("module-unpad", False), ("fused", False), ("fused", True), ("fused-unpad", False),
            ("fused-unpad", True)]
    fill = round(sum(t for _, t in data) / (len(data) * 32 * 512), 3)
    model.train()
    time_arms(arms, data, step, args.reps, rows, task="NER", what="train", B=32, S=512, fill=fill)
    model.eval()
    time_arms(arms, data, evaluate, args.reps, rows, task="NER", what="eval", B=32, S=512, fill=fill)


def bench_heads(args, rows):
    """The head alone at the NER (M = 16384, N = 10, dropout 0.1) and SQuAD (M = 12288, N = 2) training shapes:
    ``token_logits`` + loss + ``token_head_bwd`` against ``head_linear`` (the module path's three-GEMM head) forward and
    backward, each timed over 50 calls."""
    from bert_pytorch_b200.models.fused import TOKEN_STREAM, head_linear
    from bert_pytorch_b200.ops import api as K
    H = 1024
    for task, M, N, p in (("NER", 16384, NER_LABELS, 0.1), ("SQuAD", 12288, 2, 0.0)):
        g = torch.Generator(device="cuda").manual_seed(0)
        seq = torch.randn(M, H, device="cuda", generator=g).bfloat16()
        lin = torch.nn.Linear(H, N).cuda()
        w = lin.weight.detach().bfloat16().contiguous()
        dw, db = torch.zeros(N, H, device="cuda"), torch.zeros(N, device="cuda")
        labels = torch.randint(0, N, (M,), device="cuda", generator=g)
        pos = torch.randint(0, 384, (M // 384,), device="cuda", generator=g)
        loss = torch.zeros(1, device="cuda")
        x = seq.clone().requires_grad_(True)

        def fused():
            lg = K.token_logits(seq, w, lin.bias, p, 1, TOKEN_STREAM)
            if task == "NER":
                K.token_ce_(lg, labels, 1.0, loss)
            else:
                K.span_ce_(lg, pos, pos, 1.0, loss)
            K.token_head_bwd(lg, seq, w, dw, db, p, 1, TOKEN_STREAM)

        def module():
            head_linear(lin, x).float().sum().backward()

        fns = {"fused head": fused, "module head": module}
        for f in fns.values():
            f()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(args.reps):
            for k, f in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(50):
                    f()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / 50)
        for k, ts in times.items():
            row = dict(task=task, what=f"head fwd + bwd (M={M}, N={N})", path=k, ms_median=round(statistics.median(ts), 4),
                       ms_min=round(min(ts), 4), ms_max=round(max(ts), 4))
            rows.append(row)
            print(json.dumps(row), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("finetune_bench needs a GPU")
    from bert_pytorch_b200 import ops
    assert ops.available(), "sm_90a extension not built"
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows, checks, heads = [], [], []
    bench_heads(args, heads)
    bench_squad(args, rows, checks)
    bench_ner(args, rows, checks)
    for c in checks:
        print(json.dumps(c), flush=True)
    lines = [f"card: {info['name']}, power limit {info.get('power_limit')}, max SM clock {info.get('max_sm_clock')}",
             f"BERT-large, ms per batch: median of {args.reps} alternated windows of {args.steps} distinct batches "
             "(min - max)", "",
             "| task | batch | B x S | fill | path | graphs | ms | spread |", "|---|---|---|---|---|---|---|---|"]
    for r in rows:
        lines.append(f"| {r['task']} | {r['what']} | {r['B']} x {r['S']} | {r['fill']:.3f} | {r['path']} | "
                     f"{'yes' if r['graphs'] else 'no'} | {r['ms_median']:.2f} | {r['ms_min']:.2f} - {r['ms_max']:.2f} |")
    lines += ["", "| head alone | path | ms | spread |", "|---|---|---|---|"]
    lines += [f"| {r['task']} {r['what']} | {r['path']} | {r['ms_median']:.3f} | {r['ms_min']:.3f} - {r['ms_max']:.3f} |"
              for r in heads]
    lines += ["", "agreement (dropout off): " + ("all pass" if all(c["ok"] for c in checks) else "FAILED")]
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "finetune_bench.md"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "finetune_bench.json"), "w") as f:
            json.dump({"card": info, "rows": rows, "heads": heads, "checks": checks}, f, indent=1)
    if not all(c["ok"] for c in checks):
        raise SystemExit("fused and module results disagree")


if __name__ == "__main__":
    main()
