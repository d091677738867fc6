"""Token-classification (NER) fine-tuning runtime (CLI shim: ``run_ner.py``).

Flags and behaviour follow the reference's run_ner.py (:19-261; SURVEY.md 2.5.7): builds
``BertForTokenClassification(config, len(labels) + 1)``, loads ``ckpt['model']`` non-strictly, Adam without
bias correction (apex FusedAdam contract -> the fused arena kernel on CUDA), ``LambdaLR 1/(1+0.05*epoch)``,
gradient-norm clipping, macro-F1 over labels > 0, prints validation / test loss + F1.
With ``--bf16`` on a GPU (and a ``--max_seq_len`` the engine serves) every training step and evaluation batch runs as
the fused sm_90a program of ``BertForTokenClassification`` (``train_step`` / ``predict``: encoder, token head, its
dropout and the masked loss in our kernels, replayed as one CUDA graph per batch shape and token bucket); ``--unpad``
then packs each batch on the device, with no host sync.  A short last batch is filled with inert rows (label -100).
Fixed quirk Q23: evaluation runs the model once per batch (the reference runs it twice) and accumulates
python floats, not tensors.
"""
from __future__ import annotations

import argparse
import json
import random
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
from torch.utils.data import DataLoader

from . import models as modeling
from . import ops
from .config import BertConfig
from .data.ner import NERDataset
from .data.tokenization import get_bpe_tokenizer, get_wordpiece_tokenizer
from .models.arena import ParamArena
from .optim import Adam, GradientClipper


def parse_arguments(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--train_file", required=True)
    p.add_argument("--val_file", default=None)
    p.add_argument("--test_file", default=None)
    p.add_argument("--labels", nargs="+", required=True)
    p.add_argument("--model_config_file", required=True)
    p.add_argument("--model_checkpoint", required=True)
    p.add_argument("--vocab_file", default=None)
    p.add_argument("--uppercase", action="store_true", default=False)
    p.add_argument("--tokenizer", default=None, choices=[None, "wordpiece", "bpe"])
    p.add_argument("--epochs", type=int, default=10)
    p.add_argument("--lr", type=float, default=0.2)
    p.add_argument("--clip_grad", type=float, default=5.0)
    p.add_argument("--batch_size", type=int, default=32)
    p.add_argument("--max_seq_len", type=int, default=512)
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--no_cuda", action="store_true")
    p.add_argument("--bf16", action="store_true", help="bf16 compute through the fused engine (new)")
    p.add_argument("--unpad", action="store_true", default=False,
                   help="with --bf16: the fused engine computes only the unmasked tokens, in training and evaluation "
                        "(exact: the loss and F1 read unmasked positions only) (new)")
    p.add_argument("--deterministic", action="store_true", default=False,
                   help="bitwise-reproducible training: the fused engine's fixed-order reductions (no floating-point "
                        "atomics) and torch.use_deterministic_algorithms(True); the same program on the same inputs, GPU "
                        "and build gives the same loss, gradients and weights (new)")
    args = p.parse_args(argv)
    args.cuda = torch.cuda.is_available() and not args.no_cuda
    return args


def get_data(args) -> Tuple[DataLoader, Optional[DataLoader], Optional[DataLoader]]:
    with open(args.model_config_file) as f:
        cfg = json.load(f)
    vocab_file = args.vocab_file or cfg.get("vocab_file")
    kind = args.tokenizer or cfg.get("tokenizer", "wordpiece")
    if vocab_file is None:
        raise ValueError("vocab_file must be provided on the command line or in the model config")
    args.vocab_file, args.tokenizer = vocab_file, kind       # resolved values are visible to the caller (run_ner.py:67-81)
    tok = (get_wordpiece_tokenizer if kind == "wordpiece" else get_bpe_tokenizer)(vocab_file, uppercase=args.uppercase)
    def make(path, shuffle):
        if path is None:
            return None
        return DataLoader(NERDataset(path, tok, args.labels, args.max_seq_len), batch_size=args.batch_size,
                          shuffle=shuffle, pin_memory=args.cuda)
    return make(args.train_file, True), make(args.val_file, False), make(args.test_file, False)


class Metric:
    def __init__(self):
        self.total, self.n = 0.0, 0

    def update(self, value: float) -> None:
        self.total += float(value)
        self.n += 1

    @property
    def avg(self) -> float:
        return self.total / max(self.n, 1)


def macro_f1(true: List[int], pred: List[int]) -> float:
    try:
        from sklearn.metrics import f1_score
        return float(f1_score(true, pred, average="macro"))
    except ImportError:  # pragma: no cover
        labels = sorted(set(true) | set(pred))
        f1s = []
        for l in labels:
            tp = sum(1 for t, p in zip(true, pred) if t == l and p == l)
            fp = sum(1 for t, p in zip(true, pred) if t != l and p == l)
            fn = sum(1 for t, p in zip(true, pred) if t == l and p != l)
            f1s.append(2 * tp / max(2 * tp + fp + fn, 1))
        return sum(f1s) / max(len(f1s), 1)


def compute_metrics(predictions: np.ndarray, labels: np.ndarray, idx_to_label: Dict[int, str]) -> float:
    """Macro-F1 over the positions whose label id is > 0 (drops special tokens and padding)."""
    pred_ids = predictions.argmax(axis=2)
    keep = labels > 0
    return macro_f1([idx_to_label[int(l)] for l in labels[keep]],
                    [idx_to_label.get(int(p), "O") for p in pred_ids[keep]])


def _autocast(args):
    dev = "cuda" if args.cuda else "cpu"
    return torch.autocast(device_type=dev, dtype=torch.bfloat16, enabled=bool(args.bf16 and args.cuda))


def fill_batch(seqs, labels, masks, batch_size: int):
    """A short batch (host tensors [n, S]) filled up to ``batch_size`` rows with inert ones -- one unmasked [PAD]
    token, every label -100 -- so that one batch shape (one CUDA graph) serves the whole epoch."""
    k = batch_size - seqs.size(0)
    if k <= 0:
        return seqs, labels, masks
    fill_mask = torch.zeros((k, masks.size(1)), dtype=masks.dtype)
    fill_mask[:, 0] = 1
    return (torch.cat([seqs, torch.zeros((k, seqs.size(1)), dtype=seqs.dtype)]),
            torch.cat([labels, torch.full((k, labels.size(1)), -100, dtype=labels.dtype)]),
            torch.cat([masks, fill_mask]))


def fused_program(model, args) -> bool:
    """Whether training and evaluation run through the model's fused sm_90a program: ``--bf16`` on a GPU, and an
    encoder, sequence length and label count the engine serves."""
    if not (args.cuda and args.bf16):
        return False
    probe = torch.zeros(1, args.max_seq_len, dtype=torch.long, device="cuda")
    return model.bert._can_fuse(probe) and model.num_labels <= ops.api.TOKEN_HEAD_MAX_N


def train(model, optimizer, loader, epoch: int, args, clipper: GradientClipper) -> float:
    model.train()
    metric = Metric()
    dev = torch.device("cuda" if args.cuda else "cpu")
    for seqs, labels, masks in loader:
        if getattr(args, "fused", False):
            seqs, labels, masks = fill_batch(seqs, labels, masks, args.batch_size)
            tokens = int(masks.sum())                   # on the host batch: no device sync for the unpadded bucket
        seqs, labels, masks = seqs.to(dev), labels.to(dev), masks.to(dev)
        optimizer.zero_grad()
        if getattr(args, "fused", False):
            loss = model.train_step(seqs, torch.zeros_like(masks), masks, labels, tokens=tokens)
        else:
            with _autocast(args):
                loss = model(seqs, token_type_ids=torch.zeros_like(masks), attention_mask=masks, labels=labels)
            loss.backward()
        clipper.step(model.parameters())
        optimizer.step()
        metric.update(loss.item())
    print(f"Epoch {epoch}/{args.epochs} train_loss: {metric.avg:.5f}, lr: {optimizer.param_groups[0]['lr']:.2e}")
    return metric.avg


@torch.no_grad()
def evaluate(model, loader, args) -> Tuple[float, float]:
    model.eval()
    dev = torch.device("cuda" if args.cuda else "cpu")
    metric = Metric()
    preds, trues = [], []
    for seqs, labels, masks in loader:
        n = seqs.size(0)
        if getattr(args, "fused", False):
            seqs, labels, masks = fill_batch(seqs, labels, masks, args.batch_size)
            tokens = int(masks.sum())
        seqs, labels, masks = seqs.to(dev), labels.to(dev), masks.to(dev)
        if getattr(args, "fused", False):
            logits = model.predict(seqs, torch.zeros_like(masks), masks, tokens=tokens)
            seqs, labels, masks, logits = seqs[:n], labels[:n], masks[:n], logits[:n]
        else:
            with _autocast(args):
                logits = model(seqs, token_type_ids=torch.zeros_like(masks), attention_mask=masks)
        keep = masks.view(-1) == 1
        loss = torch.nn.functional.cross_entropy(logits.view(-1, logits.size(-1)).float()[keep], labels.view(-1)[keep])
        metric.update(loss.item())
        preds.append(logits.float().cpu().numpy())
        trues.append(labels.cpu().numpy())
    idx_map = {i: tag for i, tag in enumerate(args.labels, start=1)}
    return metric.avg, compute_metrics(np.concatenate(preds), np.concatenate(trues), idx_map)


def main(argv=None) -> Dict[str, float]:
    args = parse_arguments(argv)
    if args.deterministic:
        ops.use_deterministic()
    random.seed(args.seed); np.random.seed(args.seed); torch.manual_seed(args.seed)
    config = BertConfig.from_json_file(args.model_config_file)
    config.pad_vocab(8)
    modeling.ACT2FN["bias_gelu"] = modeling.bias_gelu_training
    model = modeling.BertForTokenClassification(config, num_labels=len(args.labels) + 1)
    ckpt = torch.load(args.model_checkpoint, map_location="cpu", weights_only=False)
    model.load_compatible_state_dict(ckpt["model"] if "model" in ckpt else ckpt, strict=False)
    dev = torch.device("cuda" if args.cuda else "cpu")
    model.to(dev)
    if not (args.cuda and args.bf16):
        model.bert.use_fused = False          # fp32 requested: plain PyTorch path
    model.bert.unpad = bool(args.unpad)
    arena = ParamArena(model, device=dev)
    args.fused = fused_program(model, args)
    optimizer = Adam(model.parameters(), lr=args.lr, bias_correction=False)
    arena.bind_optimizer(optimizer)
    scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, lambda e: 1.0 / (1.0 + 0.05 * e))
    clipper = GradientClipper(args.clip_grad)
    train_loader, val_loader, test_loader = get_data(args)
    out: Dict[str, float] = {}
    for epoch in range(1, args.epochs + 1):
        out["train_loss"] = train(model, optimizer, train_loader, epoch, args, clipper)
        if val_loader is not None:
            vl, vf = evaluate(model, val_loader, args)
            out.update(val_loss=vl, val_f1=vf)
            print(f"Epoch {epoch}/{args.epochs} val_loss: {vl:.5f}, val_f1: {vf:.5f}")
        scheduler.step()
    if test_loader is not None:
        tl, tf = evaluate(model, test_loader, args)
        out.update(test_loss=tl, test_f1=tf)
        print(f"test_loss: {tl:.5f}, test_f1: {tf:.5f}")
    return out


if __name__ == "__main__":
    main()
