"""Cost of a GLUE fine-tuning step and of an evaluation batch on BERT-large, device-timed.

    python tools/glue_bench.py [--reps 5] [--steps 8] [--out DIR]

BERT-large (H = 1024, 24 layers, 16 heads, I = 4096, vocabulary 30528), ``BertForSequenceClassification`` with 2
labels, S = 128, batch 32: GLUE's usual fine-tuning shape.  Sequence lengths are synthetic and seeded, in tokens
including [CLS] / [SEP]:

* ``sst2`` (short single sentences, SST-2-like): 2 + a, a log-normal with median 20 tokens (sigma 0.5), clipped to
  [3, 126];
* ``pair`` (sentence pairs, MRPC / MNLI-like): 3 + a + b, a and b log-normal with median 24 tokens (sigma 0.4),
  truncated longest-first to 128.

Paths, each timed for a training step (forward, loss, backward, gradient clipping at 1.0, arena Adam) and for an
evaluation batch (logits, no dropout):

* ``module``: today's ``BertForSequenceClassification.forward`` under bf16 autocast + ``loss.backward()`` through the
  autograd bridge of the fused encoder (padded, and ``unpad`` with its host sync per batch);
* ``fused`` / ``fused-unpad``: ``train_step`` / ``predict`` of the fused program, padded and unpadded, eager
  (``use_graphs = False``) and replayed as CUDA graphs.

Every window runs ``--steps`` distinct batches and ends in a device synchronise, timed with CUDA events; the arms
alternate ``--reps`` times, and the median and the spread (min - max) of the windows are reported in ms per batch.  The
card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

S, B, V = 128, 32, 30528


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


def lengths(kind: str, g) -> np.ndarray:
    if kind == "sst2":
        return 2 + np.clip(np.round(g.lognormal(np.log(20), 0.5, B)), 1, S - 2).astype(int)
    a = np.maximum(1, np.round(g.lognormal(np.log(24), 0.4, B))).astype(int)
    b = np.maximum(1, np.round(g.lognormal(np.log(24), 0.4, B))).astype(int)
    while (over := a + b > S - 3).any():                         # longest-first truncation
        take_a = over & (a > b)
        a[take_a] -= 1
        b[over & ~take_a] -= 1
    return 3 + a + b


def batches(kind: str, n: int, seed: int):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        lens = lengths(kind, g)
        pos = np.arange(S)[None, :]
        mask = (pos < lens[:, None]).astype(np.int64)
        ids = g.integers(5, V, (B, S)) * mask
        seg = ((pos >= lens[:, None] // 2) & (mask > 0)).astype(np.int64) if kind == "pair" else np.zeros_like(ids)
        y = g.integers(0, 2, B)
        out.append(([torch.from_numpy(t).cuda() for t in (ids, seg, mask, y)], int(mask.sum())))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("glue_bench needs a GPU")
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForSequenceClassification
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Adam, GradientClipper
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = BertConfig.from_json_file(os.path.join(root, "config", "bert_large_uncased_config.json"))
    cfg.vocab_size = V
    torch.manual_seed(0)
    model = BertForSequenceClassification(cfg, 2).cuda()
    arena = ParamArena(model)
    opt = Adam([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-7, bias_correction=False)
    arena.bind_optimizer(opt)
    clip = GradientClipper(max_grad_norm=1.0)
    eng = model.classifier_engine()
    info = card()

    def step(path, graphs, batch):
        (ids, seg, mask, y), tok = batch
        model.bert.unpad = path.endswith("unpad")
        eng.use_graphs = graphs
        if path.startswith("module"):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(ids, seg, mask).float(), y)
            loss.backward()
        else:
            model.train_step(ids, seg, mask, y, tokens=tok)
        clip.step(model.parameters())
        opt.step()
        opt.zero_grad()

    def evaluate(path, graphs, batch):
        (ids, seg, mask, _), tok = batch
        model.bert.unpad = path.endswith("unpad")
        eng.use_graphs = graphs
        if path.startswith("module"):
            model.eval()
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                model(ids, seg, mask)
            model.train()
        else:
            model.predict(ids, seg, mask, tokens=tok)

    arms = [("module", False), ("module-unpad", False), ("fused", False), ("fused", True), ("fused-unpad", False),
            ("fused-unpad", True)]
    rows = []
    for kind in ("sst2", "pair"):
        data = batches(kind, args.steps, seed={"sst2": 1, "pair": 2}[kind])
        fill = sum(t for _, t in data) / (len(data) * B * S)
        for what, fn in (("train", step), ("eval", evaluate)):
            for path, graphs in arms:                           # warm-up: every shape, bucket and graph of the windows
                for b in data:
                    for _ in range(3 if graphs else 1):
                        fn(path, graphs, b)
            torch.cuda.synchronize()
            times = {a: [] for a in arms}
            for _ in range(args.reps):
                for arm in arms:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for b in data:
                        fn(arm[0], arm[1], b)
                    e1.record()
                    torch.cuda.synchronize()
                    times[arm].append(e0.elapsed_time(e1) / len(data))
            for (path, graphs), ts in times.items():
                row = dict(lengths=kind, fill=round(fill, 3), what=what, path=path, graphs=graphs,
                           ms_median=round(statistics.median(ts), 3), ms_min=round(min(ts), 3), ms_max=round(max(ts), 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
    lines = [f"card: {info['name']}, power limit {info.get('power_limit')}, max SM clock {info.get('max_sm_clock')}",
             f"BERT-large, S = {S}, B = {B}, ms per batch: median of {args.reps} alternated windows of {args.steps} "
             "batches (min - max)", "",
             "| lengths | fill | batch | path | graphs | ms | spread |", "|---|---|---|---|---|---|---|"]
    for r in rows:
        lines.append(f"| {r['lengths']} | {r['fill']:.3f} | {r['what']} | {r['path']} | {'yes' if r['graphs'] else 'no'} | "
                     f"{r['ms_median']:.2f} | {r['ms_min']:.2f} - {r['ms_max']:.2f} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "glue_bench.md"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "glue_bench.json"), "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
