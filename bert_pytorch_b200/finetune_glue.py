"""GLUE fine-tuning, evaluation and test prediction for the classification tasks (CLI shim: ``run_glue.py``).

Flags share ``run_squad.py``'s names wherever the concept is shared.  With ``--bf16`` on a GPU every batch runs through
the fused sm_90a program of ``BertForSequenceClassification`` (:class:`~.models.fused.FusedClassifier`: the encoder,
the pooler and a one-launch classifier + loss + backward, replayed as one CUDA graph per batch shape and token bucket),
with the arena Adam kernel (no bias correction), weight decay 0.01 except on biases and LayerNorm, a linear warm-up
schedule and device-side gradient clipping at 1.0.  Otherwise the same loop runs the plain fp32 PyTorch model with
``BertAdam``.  ``--unpad`` computes only the real tokens of each batch (packed on the device, no host sync).  The last,
short batch of an epoch or a dev / test set is filled up to the batch size with inert rows (label -1), so that one batch
shape serves every step.

Outputs in ``--output_dir``: ``eval_results.json`` (the metrics of every dev set, by name), ``<TASK>.tsv`` per test set
in GLUE's submission format, ``pytorch_model.bin`` + ``bert_config.json`` after training, and the JSON log.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import time

import numpy as np
import torch

from . import models as modeling
from . import ops
from .config import BertConfig
from .data import glue as G
from .models.arena import ParamArena
from .optim import Adam, BertAdam, GradientClipper, LinearWarmUpScheduler
from .utils import logging as L
from .utils.dist import format_step


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser()
    p.add_argument("--task_name", required=True, type=str, help=f"one of {', '.join(sorted(G.TASKS))}")
    p.add_argument("--data_dir", required=True, type=str, help="the task's directory of .tsv files")
    p.add_argument("--bert_model", default=None, type=str)
    p.add_argument("--init_checkpoint", default=None, type=str)
    p.add_argument("--config_file", required=True, type=str)
    p.add_argument("--vocab_file", default=None, type=str)
    p.add_argument("--do_lower_case", action="store_true")
    p.add_argument("--output_dir", required=True, type=str)
    p.add_argument("--max_seq_length", default=128, type=int)
    p.add_argument("--do_train", action="store_true")
    p.add_argument("--do_eval", action="store_true")
    p.add_argument("--do_predict", action="store_true")
    p.add_argument("--train_batch_size", default=32, type=int)
    p.add_argument("--eval_batch_size", default=None, type=int, help="default: --train_batch_size")
    p.add_argument("--learning_rate", default=2e-5, type=float)
    p.add_argument("--num_train_epochs", default=3, type=int)
    p.add_argument("--warmup_proportion", default=0.1, type=float)
    p.add_argument("--seed", default=42, type=int)
    p.add_argument("--log_freq", default=50, type=int)
    p.add_argument("--bf16", action="store_true", help="the fused bf16 program on the GPU (fp32 PyTorch otherwise)")
    p.add_argument("--unpad", action="store_true", help="the fused program computes only the unmasked tokens")
    p.add_argument("--deterministic", action="store_true",
                   help="bitwise-reproducible runs: the fused engine's fixed-order reductions and "
                        "torch.use_deterministic_algorithms(True)")
    p.add_argument("--json-summary", default="glue_log.json", type=str, dest="json_summary")
    return p


def _batches(arrays, batch_size: int, order=None):
    """(tensors of batch, real row count): the rows of ``arrays`` in ``order``, the last batch filled with inert
    rows up to ``batch_size``."""
    n = len(arrays[0])
    order = np.arange(n) if order is None else order
    for lo in range(0, n, batch_size):
        sel = order[lo:lo + batch_size]
        yield G.fill_batch(*(torch.from_numpy(a[sel]) for a in arrays), batch_size), len(sel)


def _to(device, batch):
    ids, seg, mask, labels = batch
    tokens = int(mask.sum())                  # on the host batch: no device sync for the unpadded bucket
    return tuple(t.to(device, non_blocking=True) for t in (ids, seg, mask, labels)) + (tokens,)


def _predict(model, arrays, batch_size: int, device) -> np.ndarray:
    preds = []
    for batch, n in _batches(arrays, batch_size):
        ids, seg, mask, _, tokens = _to(device, batch)
        logits = model.predict(ids, seg, mask, tokens=tokens)
        preds.append(logits[:n].argmax(dim=-1).cpu().numpy())
    return np.concatenate(preds) if preds else np.zeros(0, dtype=np.int64)


def main(argv=None) -> dict:
    args = build_parser().parse_args(argv)
    if args.deterministic:
        ops.use_deterministic()
    task = G.get_task(args.task_name)
    if not (args.do_train or args.do_eval or args.do_predict):
        raise ValueError("at least one of --do_train, --do_eval and --do_predict is needed")
    with open(args.config_file) as f:
        model_json = json.load(f)
    if args.vocab_file is None:
        args.vocab_file = model_json.get("vocab_file")
    if args.vocab_file is None:
        raise ValueError("vocab_file must be given on the command line or in the model config")
    eval_bs = args.eval_batch_size or args.train_batch_size

    use_cuda = torch.cuda.is_available()
    device = torch.device("cuda", 0) if use_cuda else torch.device("cpu")
    fused = use_cuda and args.bf16
    os.makedirs(args.output_dir, exist_ok=True)
    L.dllogger.init([L.JSONStreamBackend(L.Verbosity.VERBOSE, os.path.join(args.output_dir, args.json_summary)),
                     L.StdOutBackend(L.Verbosity.VERBOSE, step_format=format_step)])
    dll = L.dllogger
    dll.log(step="PARAMETER", data={"Config": [str(args)]})
    random.seed(args.seed); np.random.seed(args.seed); torch.manual_seed(args.seed)
    if use_cuda:
        torch.cuda.manual_seed_all(args.seed)

    featurize = G.Featurizer(args.vocab_file, args.do_lower_case, args.max_seq_length)
    config = BertConfig.from_json_file(args.config_file)
    config.pad_vocab(8)
    model = modeling.BertForSequenceClassification(config, task.num_labels)
    if args.init_checkpoint:
        ckpt = torch.load(args.init_checkpoint, map_location="cpu", weights_only=False)
        model.load_compatible_state_dict(ckpt["model"] if "model" in ckpt else ckpt, strict=False)
        dll.log(step="PARAMETER", data={"loaded_checkpoint": args.init_checkpoint})
    model.to(device)
    model.bert.use_fused = fused
    model.bert.unpad = bool(args.unpad)
    arena = ParamArena(model, device=device)
    summary: dict = {}

    if args.do_train:
        train = featurize(task, G.train_examples(task, args.data_dir))
        n = len(train[0])
        steps_per_epoch = -(-n // args.train_batch_size)
        total_steps = steps_per_epoch * args.num_train_epochs
        for k, v in (("training_samples", n), ("train_batch_size", args.train_batch_size), ("steps", total_steps)):
            dll.log(step="PARAMETER", data={k: v})
        named = list(model.named_parameters())
        no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
        groups = [{"params": [p for nm, p in named if not any(nd in nm for nd in no_decay)], "weight_decay": 0.01},
                  {"params": [p for nm, p in named if any(nd in nm for nd in no_decay)], "weight_decay": 0.0}]
        scheduler = None
        if fused:
            optimizer = Adam(groups, lr=args.learning_rate, bias_correction=False)
            arena.bind_optimizer(optimizer)
            scheduler = LinearWarmUpScheduler(optimizer, warmup=args.warmup_proportion, total_steps=total_steps)
        else:
            optimizer = BertAdam(groups, lr=args.learning_rate, warmup=args.warmup_proportion, t_total=total_steps)
            optimizer.attach_arena(arena)
        clipper = GradientClipper(max_grad_norm=1.0)
        gen = np.random.default_rng(args.seed)
        model.train()
        step, final_loss, t0 = 0, None, time.time()
        for epoch in range(args.num_train_epochs):
            for batch, _ in _batches(train, args.train_batch_size, gen.permutation(n)):
                ids, seg, mask, labels, tokens = _to(device, batch)
                loss = model.train_step(ids, seg, mask, labels, tokens=tokens)
                clipper.step(model.parameters())
                if scheduler is not None:
                    scheduler.step()
                optimizer.step()
                optimizer.zero_grad()
                if step % args.log_freq == 0:
                    final_loss = float(loss)
                    dll.log(step=(epoch, step), data={"step_loss": final_loss,
                                                      "learning_rate": optimizer.param_groups[0]["lr"]})
                step += 1
        final_loss = float(loss)
        t = time.time() - t0
        summary.update(e2e_train_time=t, final_loss=final_loss,
                       training_sequences_per_second=n * args.num_train_epochs / max(t, 1e-9))
        torch.save({"model": model.state_dict()}, os.path.join(args.output_dir, modeling.WEIGHTS_NAME))
        with open(os.path.join(args.output_dir, modeling.CONFIG_NAME), "w") as f:
            f.write(config.to_json_string())

    if args.do_eval:
        results = {}
        t0 = time.time()
        for name, examples in G.dev_sets(task, args.data_dir):
            ids, seg, mask, labels = featurize(task, examples)
            pred = _predict(model, (ids, seg, mask, labels), eval_bs, device)
            results[name] = dict(G.compute_metrics(task, pred, labels), eval_samples=len(examples))
            dll.log(step="PARAMETER", data=dict(dev_set=name, **results[name]))
        summary.update(e2e_inference_time=time.time() - t0, eval=results)
        with open(os.path.join(args.output_dir, "eval_results.json"), "w") as f:
            json.dump(results, f, indent=2, sort_keys=True)

    if args.do_predict:
        for name, examples in G.test_sets(task, args.data_dir):
            arrays = featurize(task, examples)
            pred = _predict(model, arrays, eval_bs, device)
            G.write_submission(task, os.path.join(args.output_dir, f"{name}.tsv"), examples, pred)
            dll.log(step="PARAMETER", data={"predictions": f"{name}.tsv", "test_samples": len(examples)})

    dll.log(step=tuple(), data={k: v for k, v in summary.items() if k != "eval"})
    dll.flush()
    return summary


if __name__ == "__main__":
    main()
