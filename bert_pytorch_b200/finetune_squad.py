"""SQuAD fine-tuning + prediction runtime (CLI shim: ``run_squad.py``).

Flags, outputs and metrics follow the reference's run_squad.py (:732-857, :1115-1224; SURVEY.md 2.5.6):
``pytorch_model.bin`` (``{"model": state_dict}``) + ``bert_config.json``, ``predictions.json``,
``nbest_predictions.json``, the dllogger-style JSON log ``squad_log.json`` with ``e2e_train_time``,
``training_sequences_per_second``, ``final_loss``, ``e2e_inference_time``,
``inference_sequences_per_second``, ``exact_match``, ``F1``; the feature cache pickle is named
``<train>_<bert_model>_<max_seq>_<stride>_<max_query>``.

Execution differs (H100-first): with bf16 compute (``--bf16``, or ``--fp16``/``--amp`` without ``--loss_scale``) on
one GPU, every training step and prediction batch runs as the fused sm_90a program of ``BertForQuestionAnswering``
(``train_step`` / ``predict``: encoder, span head and loss in our kernels, replayed as one CUDA graph; a short last
batch is filled with inert rows); otherwise the encoder runs through the fused engine behind an autograd bridge.
``--fp16``/``--amp`` select 16-bit compute (bf16 by default on CUDA -- no loss scaling needed;
``--loss_scale`` is honoured for fp16) with the fused multi-tensor Adam kernel (apex FusedAdam contract,
``bias_correction=False``) on the flat arena and device-side gradient clipping (no ``.item()`` per
micro-step, SURVEY O7); without them the fp32 ``BertAdam`` path of the reference is kept.  Data
parallelism is this repo's engine (NCCL / gloo / fused), replacing apex DDP; the reference's single-process
nn.DataParallel fallback (local_rank == -1 and several GPUs) is kept as a legacy mode on the plain PyTorch forward.
Fixed reference quirks: Q19 (BPE casing flag inverted), Q20 (v2 null scores keyed by the wrong id),
Q21 (amp.master_params on the non-amp path), Q22 (max_steps off by one).
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import random
import subprocess
import sys
import time
from typing import List

import numpy as np
import torch
from torch.utils.data import DataLoader, RandomSampler, SequentialSampler, TensorDataset
from torch.utils.data.distributed import DistributedSampler as TorchDistributedSampler

from . import models as modeling
from . import ops
from .config import BertConfig
from .data import squad as SQ
from .data.squad import (  # noqa: F401  (public helpers of run_squad.py, implemented in data/squad.py)
    InputFeatures, SquadExample, convert_examples_to_features, get_answer_text, get_answers, get_final_text,
    get_valid_prelim_predictions, match_results, read_squad_examples)
from .data.tokenization import get_bpe_tokenizer, get_wordpiece_tokenizer
from .models.arena import ParamArena
from .optim import Adam, BertAdam, GradScaler, GradientClipper, LinearWarmUpScheduler
from .parallel import DataParallel, make_comm, unwrap
from .utils import logging as L
from .utils.dist import format_step, get_world_size, init_distributed, is_main_process


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser()
    p.add_argument("--bert_model", default=None, type=str, required=True)
    p.add_argument("--output_dir", default=None, type=str, required=True)
    p.add_argument("--init_checkpoint", default=None, type=str, required=True)
    p.add_argument("--config_file", default=None, type=str, required=True)
    p.add_argument("--train_file", default=None, type=str)
    p.add_argument("--predict_file", default=None, type=str)
    p.add_argument("--max_seq_length", default=384, type=int)
    p.add_argument("--doc_stride", default=128, type=int)
    p.add_argument("--max_query_length", default=64, type=int)
    p.add_argument("--do_train", action="store_true")
    p.add_argument("--do_predict", action="store_true")
    p.add_argument("--train_batch_size", default=32, type=int)
    p.add_argument("--predict_batch_size", default=8, type=int)
    p.add_argument("--learning_rate", default=5e-5, type=float)
    p.add_argument("--num_train_epochs", default=3.0, type=float)
    p.add_argument("--max_steps", default=-1.0, type=float)
    p.add_argument("--warmup_proportion", default=0.1, type=float)
    p.add_argument("--n_best_size", default=20, type=int)
    p.add_argument("--max_answer_length", default=30, type=int)
    p.add_argument("--verbose_logging", action="store_true")
    p.add_argument("--no_cuda", action="store_true")
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--gradient_accumulation_steps", type=int, default=1)
    p.add_argument("--do_lower_case", action="store_true")
    p.add_argument("--local_rank", type=int, default=int(os.environ.get("LOCAL_RANK", -1)))
    p.add_argument("--fp16", default=False, action="store_true",
                   help="reference flag (apex amp O2): 16-bit compute. The fused engine runs bf16 operands; with "
                        "--loss_scale != 0 the fp16-style GradScaler semantics are kept (DESIGN.md section 2)")
    p.add_argument("--amp", default=False, action="store_true")
    p.add_argument("--loss_scale", type=float, default=0)
    p.add_argument("--version_2_with_negative", action="store_true")
    p.add_argument("--null_score_diff_threshold", type=float, default=0.0)
    p.add_argument("--vocab_file", type=str, default=None)
    p.add_argument("--log_freq", type=int, default=50)
    p.add_argument("--json-summary", type=str, default="squad_log.json", dest="json_summary")
    p.add_argument("--eval_script", default="evaluate.py", type=str)
    p.add_argument("--do_eval", action="store_true")
    p.add_argument("--use_env", action="store_true")
    p.add_argument("--skip_checkpoint", default=False, action="store_true")
    p.add_argument("--disable-progress-bar", default=False, action="store_true", dest="disable_progress_bar")
    p.add_argument("--skip_cache", default=False, action="store_true")
    p.add_argument("--cache_dir", default=None, type=str)
    p.add_argument("--tokenizer", type=str, default=None, choices=[None, "wordpiece", "bpe"])
    # new
    p.add_argument("--bf16", default=False, action="store_true")
    p.add_argument("--backend", default=None, choices=[None, "nccl", "gloo", "fused"])
    p.add_argument("--unpad", default=False, action="store_true",
                   help="prediction through the fused engine computes only the unmasked tokens. Training stays padded: "
                        "the start / end cross-entropy normalises over every position, padded ones included, so an "
                        "unpadded training step would not be exact")
    p.add_argument("--deterministic", default=False, action="store_true",
                   help="bitwise-reproducible training: the fused engine's fixed-order reductions (no floating-point "
                        "atomics) and torch.use_deterministic_algorithms(True); the same program on the same inputs, GPU "
                        "and build gives the same loss, gradients and weights")
    return p


def _features_to_tensors(features: List[SQ.InputFeatures], training: bool):
    ids = torch.tensor([f.input_ids for f in features], dtype=torch.long)
    mask = torch.tensor([f.input_mask for f in features], dtype=torch.long)
    seg = torch.tensor([f.segment_ids for f in features], dtype=torch.long)
    if training:
        sp = torch.tensor([f.start_position for f in features], dtype=torch.long)
        ep = torch.tensor([f.end_position for f in features], dtype=torch.long)
        return TensorDataset(ids, mask, seg, sp, ep)
    return TensorDataset(ids, mask, seg, torch.arange(ids.size(0), dtype=torch.long))


def fill_batch(batch, batch_size: int, S: int):
    """A short batch (the loader's host tensors: ids, mask, segments, then the start and end positions of a training
    batch) filled up to ``batch_size`` rows with inert ones, so that one batch shape (one CUDA graph) serves the whole
    epoch: one unmasked [PAD] token (id 0, segment 0) and positions S -- the ignored index after the clamp (-1 would
    clamp to the valid target 0).  Prediction discards the filled rows."""
    n = batch[0].size(0)
    k = batch_size - n
    if k <= 0:
        return batch
    ids, mask, seg = batch[:3]

    def pad(t, fill):
        return torch.cat([t, torch.full((k,) + tuple(t.shape[1:]), fill, dtype=t.dtype)])
    mask_fill = torch.zeros((k,) + tuple(mask.shape[1:]), dtype=mask.dtype)
    mask_fill[:, 0] = 1
    return (pad(ids, 0), torch.cat([mask, mask_fill]), pad(seg, 0), *(pad(t, S) for t in batch[3:]))


def fused_program(model, S: int, device, compute_dtype) -> bool:
    """Whether training and prediction run through the model's fused sm_90a program: bf16 compute on a GPU, and an
    encoder and sequence length the engine serves."""
    if compute_dtype != torch.bfloat16 or device.type != "cuda":
        return False
    return model.bert._can_fuse(torch.zeros(1, S, dtype=torch.long, device=device))


def squad_loss(start_logits, end_logits, start_positions, end_positions):
    """Mean of the start and end cross-entropies; positions outside the window are clamped to an ignored
    index (run_squad.py:1085-1092)."""
    ignored = start_logits.size(1)
    sp = start_positions.clamp(0, ignored)
    ep = end_positions.clamp(0, ignored)
    ce = torch.nn.functional.cross_entropy
    return (ce(start_logits.float(), sp, ignore_index=ignored) + ce(end_logits.float(), ep, ignore_index=ignored)) / 2


def main(argv=None) -> dict:
    args = build_parser().parse_args(argv)
    if args.deterministic:
        ops.use_deterministic()
    args.fp16 = args.fp16 or args.amp
    with open(args.config_file) as f:
        model_json = json.load(f)
    if args.vocab_file is None:
        args.vocab_file = model_json.get("vocab_file")
    if args.tokenizer is None:
        args.tokenizer = model_json.get("tokenizer", "wordpiece")
    if args.vocab_file is None:
        raise ValueError("vocab_file must be given on the command line or in the model config")

    use_cuda = torch.cuda.is_available() and not args.no_cuda
    distributed = args.local_rank != -1 and "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1
    if use_cuda:
        torch.cuda.set_device(max(args.local_rank, 0))
        device = torch.device("cuda", max(args.local_rank, 0))
    else:
        device = torch.device("cpu")
    if distributed:
        init_distributed({"fused": "nccl"}.get(args.backend, args.backend), device)
    if args.gradient_accumulation_steps < 1:
        raise ValueError("gradient_accumulation_steps must be >= 1")
    if args.train_batch_size % args.gradient_accumulation_steps != 0:
        raise ValueError("train_batch_size must be divisible by gradient_accumulation_steps")
    args.train_batch_size //= args.gradient_accumulation_steps
    if not args.do_train and not args.do_predict:
        raise ValueError("At least one of `do_train` or `do_predict` must be True.")
    if args.do_train and not args.train_file:
        raise ValueError("If `do_train` is True, then `train_file` must be specified.")
    if args.do_predict and not args.predict_file:
        raise ValueError("If `do_predict` is True, then `predict_file` must be specified.")

    os.makedirs(args.output_dir, exist_ok=True)
    if is_main_process():
        L.dllogger.init([L.JSONStreamBackend(L.Verbosity.VERBOSE, os.path.join(args.output_dir, args.json_summary)),
                         L.StdOutBackend(L.Verbosity.VERBOSE, step_format=format_step)])
    else:
        L.dllogger.init([])
    dll = L.dllogger
    dll.log(step="PARAMETER", data={"Config": [str(args)]})

    random.seed(args.seed); np.random.seed(args.seed); torch.manual_seed(args.seed)
    if use_cuda:
        torch.cuda.manual_seed_all(args.seed)

    if args.tokenizer == "wordpiece":
        tokenizer = get_wordpiece_tokenizer(args.vocab_file, uppercase=not args.do_lower_case)
    else:
        tokenizer = get_bpe_tokenizer(args.vocab_file, uppercase=not args.do_lower_case)   # Q19 fixed

    train_examples, total_steps = None, None
    world = get_world_size()
    if args.do_train:
        train_examples = SQ.read_squad_examples(args.train_file, True, args.version_2_with_negative)
        total_steps = int(len(train_examples) / args.train_batch_size / args.gradient_accumulation_steps
                          * args.num_train_epochs)
        if distributed:
            total_steps //= world

    config = BertConfig.from_json_file(args.config_file)
    config.pad_vocab(8)
    modeling.ACT2FN["bias_gelu"] = modeling.bias_gelu_training
    model = modeling.BertForQuestionAnswering(config)
    dll.log(step="PARAMETER", data={"loading_checkpoint": True})
    ckpt = torch.load(args.init_checkpoint, map_location="cpu", weights_only=False)
    model.load_compatible_state_dict(ckpt["model"] if "model" in ckpt else ckpt, strict=False)
    dll.log(step="PARAMETER", data={"loaded_checkpoint": True})
    model.to(device)
    dll.log(step="PARAMETER", data={"model_weights_num": sum(p.numel() for p in model.parameters() if p.requires_grad)})

    compute_dtype = torch.float32
    if use_cuda:
        compute_dtype = torch.float16 if (args.fp16 and not args.bf16 and args.loss_scale != 0) else \
            (torch.bfloat16 if (args.fp16 or args.bf16) else torch.float32)
    arena = ParamArena(model, device=device)
    comm = make_comm(args.backend)
    ddp = DataParallel(model, comm=comm, arena=arena)
    # Single-process multi-GPU fallback (reference: run_squad.py:1012-1013, nn.DataParallel when local_rank == -1 and
    # n_gpu > 1).  The fused engine is a one-device kernel program, so this legacy mode runs the plain PyTorch
    # forward replicated by torch.nn.DataParallel; gradients land in the arena views on device 0.  One process per
    # GPU (torchrun) is the supported way to scale; B200_DATAPARALLEL=0 turns the fallback off.
    forward_model = ddp
    if (use_cuda and not distributed and args.local_rank == -1 and torch.cuda.device_count() > 1
            and os.environ.get("B200_DATAPARALLEL", "1") != "0"):
        model.bert.use_fused = False
        forward_model = torch.nn.DataParallel(model)
        dll.log(step="PARAMETER", data={"single_process_data_parallel_gpus": torch.cuda.device_count()})
    # bf16 compute: training steps and prediction batches run as the model's fused program (graph-replayed); the fp16
    # loss-scaled path, fp32 and the legacy nn.DataParallel mode keep the module path
    fused = forward_model is ddp and fused_program(model, args.max_seq_length, device, compute_dtype)

    optimizer = scheduler = scaler = None
    if args.do_train:
        named = list(model.named_parameters())
        no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
        groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": 0.01},
                  {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
        if args.fp16 or args.bf16:
            optimizer = Adam(groups, lr=args.learning_rate, bias_correction=False)
            arena.bind_optimizer(optimizer)
            scheduler = LinearWarmUpScheduler(optimizer, warmup=args.warmup_proportion, total_steps=total_steps)
            scaler = GradScaler(init_scale=args.loss_scale if args.loss_scale else 2.0 ** 16,
                                enabled=(compute_dtype == torch.float16), device=device)
        else:
            # fp32 requested: plain PyTorch forward/backward on the fp32 master views (like finetune_ner); BertAdam
            # is attached to the arena so zero_grad keeps p.grad inside flat_grad (what sync_gradients reduces) and
            # every step refreshes the bf16 shadow that evaluation through the fused engine reads
            model.bert.use_fused = False
            optimizer = BertAdam(groups, lr=args.learning_rate, warmup=args.warmup_proportion, t_total=total_steps)
            optimizer.attach_arena(arena)

    summary: dict = {}
    global_step = 0
    if args.do_train:
        tag = [s for s in args.bert_model.split("/") if s][-1]
        name = f"_{tag}_{args.max_seq_length}_{args.doc_stride}_{args.max_query_length}"
        cache = (args.train_file + name if args.cache_dir is None
                 else os.path.join(args.cache_dir, os.path.basename(args.train_file) + name))
        try:
            with open(cache, "rb") as r:
                train_features = pickle.load(r)
        except Exception:  # noqa: BLE001 - any problem with the cache means: rebuild it
            train_features = SQ.convert_examples_to_features(train_examples, tokenizer, args.max_seq_length,
                                                             args.doc_stride, args.max_query_length, True)
            if not args.skip_cache and is_main_process():
                dll.log(step="PARAMETER", data={"Cached_train features_file": cache})
                with open(cache, "wb") as w:
                    pickle.dump(train_features, w)
        for k, v in (("train_start", True), ("training_samples", len(train_examples)),
                     ("training_features", len(train_features)), ("train_batch_size", args.train_batch_size),
                     ("steps", total_steps)):
            dll.log(step="PARAMETER", data={k: v})
        data = _features_to_tensors(train_features, True)
        sampler = TorchDistributedSampler(data) if distributed else RandomSampler(data)
        loader = DataLoader(data, sampler=sampler, batch_size=args.train_batch_size, pin_memory=use_cuda)
        model.train()
        clipper = GradientClipper(max_grad_norm=1.0)
        final_loss = None
        t0 = time.time()
        acc = args.gradient_accumulation_steps
        done = False
        for epoch in range(int(args.num_train_epochs)):
            if distributed:
                sampler.set_epoch(epoch)
            for step, batch in enumerate(loader):
                if args.max_steps > 0 and global_step >= args.max_steps:      # Q22 fixed
                    done = True
                    break
                if fused:
                    batch = fill_batch(batch, args.train_batch_size, args.max_seq_length)
                ids, mask, seg, sp, ep = (t.to(device, non_blocking=True) for t in batch)
                if fused:
                    loss = model.train_step(ids, seg, mask, sp, ep, grad_scale=1.0 / acc)
                else:
                    with torch.autocast(device_type=device.type, dtype=compute_dtype,
                                        enabled=compute_dtype != torch.float32):
                        start_logits, end_logits = forward_model(ids, seg, mask)
                        loss = squad_loss(start_logits, end_logits, sp, ep)
                if acc > 1:
                    loss = loss / acc
                boundary = (step + 1) % acc == 0
                if not fused:
                    (scaler.scale(loss) if scaler is not None else loss).backward()
                if boundary:
                    ddp.sync_gradients()
                    if scaler is not None:
                        scaler.unscale_(optimizer)
                    clipper.step(model.parameters())                           # device-side coefficient
                    if scheduler is not None:
                        scheduler.step()
                    if scaler is not None:
                        scaler.step(optimizer); scaler.update()
                    else:
                        optimizer.step()
                    optimizer.zero_grad()
                    global_step += 1
                if step % args.log_freq == 0:
                    final_loss = float(loss.detach())
                    dll.log(step=(epoch, global_step), data={"step_loss": final_loss,
                                                             "learning_rate": optimizer.param_groups[0]["lr"]})
            if done:
                break
        if final_loss is None:
            final_loss = float(loss)
        time_to_train = time.time() - t0
        summary.update(e2e_train_time=time_to_train, final_loss=final_loss,
                       training_sequences_per_second=len(train_features) * (epoch + 1 if done else args.num_train_epochs)
                       * 1.0 / max(time_to_train, 1e-9))
        if is_main_process() and not args.skip_checkpoint:
            torch.save({"model": unwrap(ddp).state_dict()}, os.path.join(args.output_dir, modeling.WEIGHTS_NAME))
            with open(os.path.join(args.output_dir, modeling.CONFIG_NAME), "w") as f:
                f.write(config.to_json_string())

    if args.do_predict and is_main_process():
        eval_examples = SQ.read_squad_examples(args.predict_file, False, args.version_2_with_negative)
        eval_features = SQ.convert_examples_to_features(eval_examples, tokenizer, args.max_seq_length, args.doc_stride,
                                                        args.max_query_length, False)
        dll.log(step="PARAMETER", data={"infer_start": True})
        dll.log(step="PARAMETER", data={"eval_samples": len(eval_examples)})
        dll.log(step="PARAMETER", data={"eval_features": len(eval_features)})
        dll.log(step="PARAMETER", data={"predict_batch_size": args.predict_batch_size})
        data = _features_to_tensors(eval_features, False)
        loader = DataLoader(data, sampler=SequentialSampler(data), batch_size=args.predict_batch_size)
        model.eval()
        model.bert.unpad = bool(args.unpad)
        results: List[SQ.RawResult] = []
        t0 = time.time()
        with torch.no_grad():
            for ids, mask, seg, idx in loader:
                if fused:
                    ids, mask, seg = fill_batch((ids, mask, seg), args.predict_batch_size, args.max_seq_length)
                    s, e = model.predict(ids.to(device), seg.to(device), mask.to(device), tokens=int(mask.sum()))
                else:
                    with torch.autocast(device_type=device.type, dtype=compute_dtype,
                                        enabled=compute_dtype != torch.float32):
                        s, e = model(ids.to(device), seg.to(device), mask.to(device))
                n = idx.numel()
                s, e = s[:n].float().cpu().tolist(), e[:n].float().cpu().tolist()   # one D2H per batch, not per example
                for j, i in enumerate(idx.tolist()):
                    results.append(SQ.RawResult(eval_features[i].unique_id, s[j], e[j]))
        time_to_infer = time.time() - t0
        answers, nbest = SQ.get_answers(eval_examples, eval_features, results, n_best_size=args.n_best_size,
                                        max_answer_length=args.max_answer_length, do_lower_case=args.do_lower_case,
                                        version_2_with_negative=args.version_2_with_negative,
                                        null_score_diff_threshold=args.null_score_diff_threshold,
                                        verbose_logging=args.verbose_logging)
        pred_file = os.path.join(args.output_dir, "predictions.json")
        with open(pred_file, "w") as f:
            f.write(json.dumps(answers, indent=4) + "\n")
        with open(os.path.join(args.output_dir, "nbest_predictions.json"), "w") as f:
            f.write(json.dumps(nbest, indent=4) + "\n")
        summary.update(e2e_inference_time=time_to_infer,
                       inference_sequences_per_second=len(eval_features) / max(time_to_infer, 1e-9))
        if args.do_eval:
            if args.eval_script and os.path.isfile(args.eval_script):
                out = subprocess.check_output([sys.executable, args.eval_script, args.predict_file, pred_file]).decode()
                scores = json.loads(out.strip().splitlines()[-1].replace("'", '"'))
                summary.update(exact_match=float(scores["exact_match"]), F1=float(scores["f1"]))
            else:   # offline: built-in implementation of the official metric
                scores = SQ.evaluate_predictions(args.predict_file, answers)
                summary.update(exact_match=scores["exact_match"], F1=scores["f1"])
    if is_main_process():
        dll.log(step=tuple(), data=summary)
        dll.flush()
    return summary


if __name__ == "__main__":
    main()
