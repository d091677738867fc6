"""Pre-training runtime (the L4 layer of SURVEY.md 1): argument/JSON handling, process-group
setup, model / optimizer / dataset preparation, the accumulation loop, checkpoint + resume
and metric logging.  ``run_pretraining.py`` at the repo root is the CLI shim.

Function names, flags, output files and checkpoint layout follow the reference
(run_pretraining.py:75-600; SURVEY.md 2.5.1/2.5.2/5.4); the execution underneath does not:
  * parameters/gradients/moments live in a flat arena; on CUDA the forward/backward of the
    whole model is the fused sm_90a engine (models/fused.py) and the optimizer step is the
    multi-tensor LAMB kernels; on CPU everything runs the plain-PyTorch oracle path;
  * ``--backend fused`` replaces DDP's NCCL all-reduce + unscale + LAMB by one peer-memory
    kernel sequence (parallel/peer.py); ``nccl`` / ``gloo`` remain (baseline / CPU plumbing);
  * the loss stays on the device between micro-steps (the reference syncs the host every
    micro-step, run_pretraining.py:542); data arrives through the batched pinned loader;
  * new flags: ``--bf16`` (default compute type on CUDA), ``--fp8``, ``--backend``,
    ``--device``, ``--no_fused``, ``--loader_depth``.
Documented deviations from reference quirks: Q7 (first update used acc+1 micro-batches) and
Q9/Q10 (throughput accounting) are fixed; Q6 (sampler index ran ahead of consumption) is
fixed by the loader; the rest of the arithmetic (ceil-based accumulation, step numbering of
checkpoints, phase-2 optimizer surgery) is kept bit-for-bit.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import warnings
from pathlib import Path
from time import perf_counter
from typing import Any, Dict, List, Tuple

import numpy as np
import torch

from . import models as modeling
from .config import BertConfig, batch_arithmetic, overlay_json_config
from .data import BatchedPretrainingLoader, DistributedSampler, ShardedPretrainingDataset
from .data.tokenization import get_bpe_tokenizer, get_wordpiece_tokenizer
from .models import BertPretrainingCriterion  # noqa: F401  (public name of run_pretraining.py:96)
from .models.arena import NO_DECAY_KEYS, ParamArena
from .optim import GradScaler, Lamb, LinearWarmUpScheduler, PolyWarmUpScheduler
from .parallel import DataParallel, make_comm, unwrap
from .utils import checkpoint as ckpt_utils
from .utils import logging as logger
from .utils.dist import get_rank, get_world_size, init_distributed, is_main_process
from .utils.timing import DeviceTimer, StepClock, max_over_ranks, nvtx_range


# ---------------------------------------------------------------------------
# arguments
# ---------------------------------------------------------------------------

def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="BERT pre-training (H100-native)")
    p.add_argument("--config_file", default=None, type=str, help="JSON config overriding the defaults below")
    # required (may come from the JSON)
    p.add_argument("--input_dir", default=None, type=str, help="file or directory (recursive *.hdf5)")
    p.add_argument("--output_dir", default=None, type=str, help="checkpoints and logs")
    p.add_argument("--model_config_file", default=None, type=str, help="BERT model JSON")
    # dynamic masking
    p.add_argument("--masked_token_fraction", type=float, default=0.2)
    p.add_argument("--max_predictions_per_seq", type=int, default=80)
    # training configuration
    p.add_argument("--disable_progress_bar", default=False, action="store_true")
    p.add_argument("--num_steps_per_checkpoint", type=int, default=200)
    p.add_argument("--skip_checkpoint", default=False, action="store_true")
    p.add_argument("--checkpoint_activations", default=False, action="store_true")
    p.add_argument("--log_prefix", type=str, default="logfile")
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--fp16", default=False, action="store_true",
                   help="reference flag: dynamic loss scaling (GradScaler) on. On an H100 the fused engine multiplies bf16 "
                        "operands either way -- fp16 selects the scaler semantics, not fp16 tensor-core operands "
                        "(DESIGN.md section 2); the plain-PyTorch fallback path autocasts to fp16")
    # hyper-parameters
    p.add_argument("--learning_rate", default=5e-5, type=float)
    p.add_argument("--lr_decay", default="poly", type=str, choices=["poly", "linear"])
    p.add_argument("--warmup_proportion", default=0.01, type=float)
    p.add_argument("--global_batch_size", default=2 ** 16, type=int)
    p.add_argument("--local_batch_size", default=8, type=int)
    p.add_argument("--max_steps", default=1000, type=float)
    p.add_argument("--steps", default=1000, type=float, help="steps to perform this session")
    p.add_argument("--previous_phase_end_step", default=0, type=int)
    # K-FAC
    p.add_argument("--kfac", default=False, action="store_true")
    p.add_argument("--kfac_inv_interval", type=int, default=10)
    p.add_argument("--kfac_factor_interval", type=int, default=1)
    p.add_argument("--kfac_stat_decay", type=float, default=0.95)
    p.add_argument("--kfac_damping", type=float, default=0.003)
    p.add_argument("--kfac_kl_clip", type=float, default=0.001)
    p.add_argument("--kfac_skip_layers", nargs="+", type=str, default=["BertLMPredictionHead", "embedding"])
    p.add_argument("--local_rank", type=int, default=0)
    # new in this code base
    p.add_argument("--bf16", default=False, action="store_true", help="bf16 compute (default on CUDA unless --fp16)")
    p.add_argument("--backend", default=None, choices=[None, "nccl", "gloo", "fused"],
                   help="gradient-reduction backend (default: nccl on CUDA, gloo on CPU)")
    p.add_argument("--device", default=None, choices=[None, "cuda", "cpu"])
    p.add_argument("--no_fused", default=False, action="store_true", help="run the plain-PyTorch oracle path")
    p.add_argument("--fp8", default=False, action="store_true",
                   help="fp8 GEMM operands in the fused engine (e4m3 activations/weights, e5m2 gradients, "
                        "per-tensor delayed scaling); LayerNorm, attention, master weights unchanged")
    p.add_argument("--loader_depth", type=int, default=4)
    return p


def parse_arguments(argv=None) -> argparse.Namespace:
    args = overlay_json_config(build_parser(), argv)
    if "LOCAL_RANK" in os.environ:
        args.local_rank = int(os.environ["LOCAL_RANK"])
    return args


def check_required(args) -> None:
    for k in ("input_dir", "output_dir", "model_config_file"):
        if getattr(args, k) is None:
            raise ValueError(f"--{k} must be provided via arguments or the config file")


# ---------------------------------------------------------------------------
# setup
# ---------------------------------------------------------------------------

def setup_training(args):
    use_cuda = torch.cuda.is_available() if args.device is None else args.device == "cuda"
    if use_cuda:
        torch.cuda.set_device(args.local_rank)
        args.device_obj = torch.device("cuda", args.local_rank)
    else:
        args.device_obj = torch.device("cpu")
    backend = args.backend
    torch_backend = {"fused": "nccl", None: None}.get(backend, backend)
    args.dist_backend = init_distributed(torch_backend, args.device_obj)

    args.model_output_dir = os.path.join(args.output_dir, "pretrain_ckpts")
    if is_main_process():
        os.makedirs(args.model_output_dir, exist_ok=True)
    from .utils.dist import barrier
    barrier()

    main = is_main_process()
    logger.init(handlers=[
        logger.StreamHandler(verbose=main),
        logger.FileHandler(os.path.join(args.output_dir, args.log_prefix + ".txt"), overwrite=False, verbose=main),
        logger.TorchTensorboardHandler(os.path.join(args.output_dir, "tensorboard"), verbose=main),
        logger.CSVHandler(os.path.join(args.output_dir, args.log_prefix + "_metrics.csv"), overwrite=False,
                          verbose=main),
    ])
    logger.info(f"Torch distributed initialized (world_size={get_world_size()}, backend={args.dist_backend}, "
                f"grad-reduction={backend or args.dist_backend})")

    ws = get_world_size()
    if args.global_batch_size % ws != 0 and main:
        warnings.warn(f"global_batch_size={args.global_batch_size} is not divisible by world_size={ws}. "
                      "The last batch will be padded with additional samples.")
    args.local_accumulated_batch_size, args.accumulation_steps = batch_arithmetic(
        args.global_batch_size, args.local_batch_size, ws)
    if args.local_accumulated_batch_size % args.local_batch_size != 0 and main:
        warnings.warn(f"local_accumulated_batch_size={args.local_accumulated_batch_size} is not divisible by "
                      f"local_batch_size={args.local_batch_size}; the last micro-batch pads the global batch "
                      f"to {args.accumulation_steps * args.local_batch_size * ws}.")
    # precision policy
    if use_cuda and not args.fp16:
        args.bf16 = True
    args.compute_dtype = (torch.float16 if args.fp16 else torch.bfloat16 if args.bf16 else torch.float32)
    return args


def prepare_model(args):
    config = BertConfig.from_json_file(args.model_config_file)
    config.pad_vocab(8)
    modeling.ACT2FN["bias_gelu"] = modeling.bias_gelu_training
    model = modeling.BertForPreTraining(config)

    checkpoint, global_steps = None, 0
    ckpt, args.resume_step = ckpt_utils.load_latest(args.model_output_dir)
    if ckpt is not None:
        checkpoint = ckpt
        logger.info(f"Loading checkpoint {ckpt_utils.checkpoint_path(args.model_output_dir, args.resume_step)}")
        model.load_compatible_state_dict(checkpoint["model"], strict=False)
        if args.previous_phase_end_step > args.resume_step:
            raise ValueError(f"previous_phase_end_step={args.previous_phase_end_step} cannot be larger than "
                             f"resume_step={args.resume_step}")
        global_steps = args.resume_step - args.previous_phase_end_step
        logger.info(f"Resume from step {args.resume_step} checkpoint")

    model.to(args.device_obj)
    model.checkpoint_activations(args.checkpoint_activations)
    if args.no_fused:
        model.enable_apex(False)
    config.max_predictions_per_seq = args.max_predictions_per_seq    # static MLM row capacity of the fused head
    arena = ParamArena(model, device=args.device_obj)
    if getattr(args, "fp8", False) and not args.no_fused and args.device_obj.type == "cuda":
        model.bert.fused_engine().enable_fp8()      # this model's engine only (no process-wide switch)
    comm = make_comm(args.backend)
    if getattr(comm, "fuses_optimizer", False):
        comm.adopt(arena)        # arenas move into NVLink symmetric memory; optimizer + reduction fuse
    model = DataParallel(model, comm=comm, arena=arena)
    criterion = modeling.BertPretrainingCriterion(config.vocab_size)
    args.config_obj = config
    return model, checkpoint, global_steps, criterion, args


def prepare_optimizers(args, model, checkpoint, global_steps):
    base = unwrap(model)
    named = list(base.named_parameters())
    groups = [
        {"params": [p for n, p in named if not any(nd in n for nd in NO_DECAY_KEYS)], "weight_decay": 0.01},
        {"params": [p for n, p in named if any(nd in n for nd in NO_DECAY_KEYS)], "weight_decay": 0.0},
    ]
    Scheduler = {"poly": PolyWarmUpScheduler, "linear": LinearWarmUpScheduler}.get(args.lr_decay)
    if Scheduler is None:
        raise ValueError(f'Unknown lr decay "{args.lr_decay}"')
    optimizer = Lamb(groups, lr=args.learning_rate)
    model.arena.bind_optimizer(optimizer)

    if checkpoint is not None:
        if args.resume_step >= args.previous_phase_end_step:
            ckpt_utils.override_optimizer_hparams(checkpoint, global_steps=global_steps, max_steps=args.max_steps,
                                                  warmup=args.warmup_proportion, lr=args.learning_rate)
        optimizer.load_state_dict(checkpoint["optimizer"])

    lr_schedulers = [Scheduler(optimizer, warmup=args.warmup_proportion, total_steps=args.max_steps)]

    scaler = None
    if args.fp16:
        scaler = GradScaler(device=args.device_obj)
    else:
        scaler = GradScaler(enabled=False)   # bf16/fp32: identity, state_dict keys kept for layout compat
    if checkpoint is not None and "scaler" in checkpoint:
        scaler.load_state_dict(checkpoint["scaler"])

    preconditioner = None
    if args.kfac:
        from . import kfac
        preconditioner = kfac.KFAC(
            base, lr=args.learning_rate, factor_decay=args.kfac_stat_decay, damping=args.kfac_damping,
            kl_clip=args.kfac_kl_clip, factor_update_freq=args.kfac_factor_interval,
            inv_update_freq=args.kfac_inv_interval, skip_layers=args.kfac_skip_layers,
            comm_method=kfac.CommMethod.HYBRID_OPT, grad_worker_fraction=0.5, inv_dtype=torch.float16,
            accumulate_data=False, compute_factor_in_hook=True, distribute_layer_factors=False,
            grad_scaler=scaler, comm=model.comm)
        lr_schedulers.append(Scheduler(preconditioner, warmup=args.warmup_proportion, total_steps=args.max_steps))
        if checkpoint is not None and "preconditioner" in checkpoint:
            preconditioner.load_state_dict(checkpoint["preconditioner"])
        if is_main_process():
            logger.info(preconditioner)
    configure_fused_reduction(model, preconditioner)
    return optimizer, preconditioner, lr_schedulers, scaler


def configure_fused_reduction(model, preconditioner=None) -> None:
    """Peer-memory backend: the gradient reduction is deferred into the fused LAMB kernel, and the engine's
    weight-gradient GEMMs of the last micro-step reduce-scatter straight into the owner ranks' arenas
    (``B200_PEER_PUSH=0`` keeps the reduction entirely inside the optimizer kernel).  With a preconditioner
    (K-FAC needs the averaged gradients before the optimizer) the reduction stays a separate all-reduce."""
    comm = getattr(model, "comm", None)
    if comm is None or not getattr(comm, "fuses_optimizer", False):
        return
    model.defer_reduction = preconditioner is None
    if model.defer_reduction and "B200_PEER_MASTER_LOCAL" not in os.environ and hasattr(comm, "push_master"):
        comm.push_master = False      # fp32 master stays with its owner; checkpoints gather it (save())
    base = unwrap(model)
    eng = base.pretrain_engine() if hasattr(base, "pretrain_engine") else None
    if model.defer_reduction and eng is not None and os.environ.get("B200_PEER_PUSH", "1") != "0":
        comm.set_prereduced(eng.engine.gemm_reduced_parameters())


def find_input_files(input_dir: str) -> List[str]:
    if os.path.isfile(input_dir):
        return [input_dir]
    if os.path.isdir(input_dir):
        return sorted(str(p) for p in Path(input_dir).rglob("*.hdf5") if p.is_file())
    return []


def prepare_dataset(args, checkpoint):
    input_files = find_input_files(args.input_dir)
    with open(args.model_config_file) as f:
        cfg = json.load(f)
    vocab_size, vocab_file = cfg["vocab_size"], cfg["vocab_file"]
    lowercase, tok_kind = cfg.get("lowercase", True), cfg.get("tokenizer", "wordpiece")
    if tok_kind == "wordpiece":
        tokenizer = get_wordpiece_tokenizer(vocab_file, uppercase=not lowercase)
    elif tok_kind == "bpe":
        tokenizer = get_bpe_tokenizer(vocab_file, uppercase=not lowercase)
    else:
        raise ValueError(f"Unknown tokenizer '{tok_kind}'. Options are 'wordpiece' and 'bpe'")
    mask_token_id = tokenizer.token_to_id("[MASK]")

    dataset = ShardedPretrainingDataset(input_files, mask_token_id, args.max_predictions_per_seq,
                                        args.masked_token_fraction, vocab_size=vocab_size,
                                        seed=args.seed + get_rank())
    sampler = DistributedSampler(dataset, get_world_size(), rank=get_rank(), seed=args.seed)
    if checkpoint is not None and "sampler" in checkpoint:
        sampler.load_state_dict(checkpoint["sampler"])
    loader = BatchedPretrainingLoader(dataset, sampler, args.local_batch_size, depth=args.loader_depth,
                                      pin_memory=args.device_obj.type == "cuda")
    if is_main_process():
        logger.info(f"Samples in dataset: {len(dataset)}")
        logger.info(f"Samples per device: {len(sampler)}")
        logger.info(f"Sampler starting index: {sampler.index}")
        logger.info(f"Batches in dataloader: {len(loader)}")
    return loader, sampler


# ---------------------------------------------------------------------------
# step functions
# ---------------------------------------------------------------------------

def take_optimizer_step(optimizer, preconditioner, model, scaler):
    comm = getattr(model, "comm", None)
    if comm is not None and getattr(comm, "fuses_optimizer", False) and preconditioner is None:
        # one peer-memory kernel: reduce-scatter + unscale + partitioned LAMB + parameter all-gather
        scale = scaler.get_scale() if (scaler is not None and scaler.is_enabled()) else 1.0
        comm.fused_lamb_step(optimizer, loss_scale=scale)
        if scaler is not None and scaler.is_enabled():
            scaler._lazy_init(comm.device)
            scaler.found_inf.copy_(comm.stats[3].clamp(max=1.0))
            scaler.update()
        return
    if preconditioner is not None:
        if scaler is not None:
            scaler.unscale_(optimizer)
        preconditioner.step()
    if scaler is not None:
        scaler.step(optimizer)
        scaler.update()
    else:
        optimizer.step()
    optimizer.zero_grad()        # arena: one memset; keeps the persistent grad views alive


def forward_backward_pass(model, criterion, scaler, batch, divisor, sync_grads=True, compute_dtype=None):
    """One micro-step.  Returns the (unscaled, already divided) loss as a device tensor."""
    input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels = batch
    base = unwrap(model)
    engine = base.pretrain_engine() if hasattr(base, "pretrain_engine") else None
    loss_scale = scaler.get_scale() if (scaler is not None and scaler.is_enabled()) else 1.0
    if engine is not None:
        # fused sm_90a path: forward + backward in one call, grads accumulate into the arena
        comm = getattr(model, "comm", None)
        kf = getattr(base.bert, "_kfac", None) if hasattr(base, "bert") else None
        if kf is not None:                   # K-FAC statistics only where they count; all other micro-steps replay the graph
            kf.capture = kf.wants_data(last_micro_step=sync_grads)
        push = (sync_grads and comm is not None and getattr(model, "defer_reduction", False)
                and hasattr(comm, "begin_push") and comm.begin_push())
        engine.grad_push = bool(push)       # last micro-step: weight-gradient GEMMs reduce-scatter over NVLink
        try:
            loss = engine.forward_backward(input_ids, segment_ids, input_mask, masked_lm_labels,
                                           next_sentence_labels, grad_scale=loss_scale / divisor)
        finally:
            if push:
                comm.end_push()
                engine.grad_push = False
        loss = loss / divisor
    else:
        dev_type = input_ids.device.type
        use_amp = compute_dtype in (torch.float16, torch.bfloat16)
        with torch.autocast(device_type=dev_type, dtype=compute_dtype, enabled=use_amp):
            prediction_scores, seq_relationship_score = model(
                input_ids=input_ids.long(), token_type_ids=segment_ids.long(), attention_mask=input_mask.long())
            loss = criterion(prediction_scores, masked_lm_labels.long(), seq_relationship_score,
                             next_sentence_labels.long())
        loss = loss / divisor
        (scaler.scale(loss) if scaler is not None else loss).backward()
    if sync_grads:
        model.sync_gradients()
    return loss.detach()


# ---------------------------------------------------------------------------
# main loop
# ---------------------------------------------------------------------------

def main(args) -> Tuple[int, float]:
    model, checkpoint, global_step, criterion, args = prepare_model(args)
    optimizer, preconditioner, lr_schedulers, scaler = prepare_optimizers(args, model, checkpoint, global_step)
    loader, sampler = prepare_dataset(args, checkpoint)
    model.train()
    manager = ckpt_utils.CheckpointManager(args.model_output_dir, keep=3)
    device = args.device_obj
    acc = args.accumulation_steps
    epoch = checkpoint["epoch"] if checkpoint is not None and "epoch" in checkpoint else 0
    optimization_steps = 0          # this session
    micro = 0                       # micro-steps inside the current optimizer step
    window_loss = torch.zeros((), device=device)
    last_loss = torch.zeros((), device=device)
    session_seqs = 0
    timer = DeviceTimer(device)
    train_ms = 0.0
    step_t0 = perf_counter()
    pbar = None
    if not args.disable_progress_bar and is_main_process():
        from tqdm import tqdm
        pbar = tqdm(total=int(min(args.steps, args.max_steps - global_step)), desc="train", unit="step")

    def save(step_no: int) -> None:
        if args.skip_checkpoint:
            return
        comm = getattr(model, "comm", None)
        if comm is not None and getattr(model, "defer_reduction", False) and hasattr(comm, "gather_optimizer_state"):
            # peer-memory backend: the LAMB moments (and, with a shard-local master, the fp32 weights) are partitioned;
            # every rank joins the gather so that rank 0 writes the full per-parameter layout (SURVEY.md 5.4)
            comm.gather_optimizer_state()
            comm.gather_master()
        payload: Dict[str, Any] = {
            "model": unwrap(model).state_dict(),
            "optimizer": optimizer.state_dict(),
            "sampler": loader.state_dict(),
            "epoch": epoch,
        }
        if preconditioner is not None:
            payload["preconditioner"] = preconditioner.state_dict()
        if scaler is not None:
            payload["scaler"] = scaler.state_dict()
        if is_main_process():
            path = manager.save(step_no + args.previous_phase_end_step, payload)
            logger.info(f"Saved checkpoint {path}")

    done = global_step >= args.max_steps
    # B200_PROFILE_DIR=<dir>: torch.profiler (CUPTI) trace of optimizer steps 2-3 of this session, one file per rank
    profiler = None
    if os.environ.get("B200_PROFILE_DIR") and device.type == "cuda":
        from torch.profiler import ProfilerActivity, profile, schedule, tensorboard_trace_handler
        profiler = profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA],
                           schedule=schedule(wait=1, warmup=1, active=2, repeat=1),
                           on_trace_ready=tensorboard_trace_handler(os.environ["B200_PROFILE_DIR"]))
        profiler.start()
    timer.start()
    clock = StepClock(device)           # device-side split of every optimizer step: micro-steps | reduction + optimizer
    clock.mark()
    while not done:
        sampler.set_epoch(epoch)
        for batch in loader:
            batch = [t.to(device, non_blocking=True) for t in batch]
            micro += 1
            sync = micro == acc
            with nvtx_range("micro_step_sync" if sync else "micro_step"):
                loss = forward_backward_pass(model, criterion, scaler, batch, acc, sync_grads=sync,
                                             compute_dtype=args.compute_dtype)
            window_loss += loss
            last_loss = loss
            session_seqs += batch[0].size(0)
            if not sync:
                continue
            for lrs in lr_schedulers:
                lrs.step()
            clock.mark()
            with nvtx_range("optimizer_step"):
                take_optimizer_step(optimizer, preconditioner, model, scaler)
            clock.mark()
            if profiler is not None:
                profiler.step()
            global_step += 1
            optimization_steps += 1
            micro = 0
            now = perf_counter()
            step_time = now - step_t0
            step_t0 = now
            average_loss = float(window_loss)          # the one host synchronisation of the step
            micro_ms, opt_ms = clock.intervals()[-2:]      # complete: the read-back above waited for the stream
            clock.reset()
            clock.mark()
            # reference: run_pretraining.py logs step = global_step + previous_phase_end_step, so phase-2 curves
            # continue phase 1's axis in the same output_dir instead of overlapping it (ADVICE r1)
            logger.log(tag="train", step=global_step + args.previous_phase_end_step, epoch=epoch,
                       average_loss=average_loss, step_loss=float(last_loss) * acc,
                       learning_rate=optimizer.param_groups[0]["lr"],
                       samples_per_second=(acc * args.local_batch_size * get_world_size()) / max(step_time, 1e-9),
                       device_step_ms=micro_ms + opt_ms, optimizer_ms=opt_ms)
            window_loss.zero_()
            if pbar is not None:
                pbar.update(1)
            finished = global_step >= args.max_steps or optimization_steps >= args.steps
            if finished or (optimization_steps % args.num_steps_per_checkpoint == 0):
                save(global_step)
            if finished:
                done = True
                break
        else:
            epoch += 1
            continue
        break
    train_ms = timer.stop()
    if profiler is not None:
        profiler.stop()
    loader.close()
    if pbar is not None:
        pbar.close()
    train_s = max_over_ranks(train_ms / 1e3)
    seqs = session_seqs * get_world_size()
    args.train_time_s = train_s
    return global_step, (seqs / train_s if train_s > 0 else 0.0)


def seed_everything(seed: int) -> None:
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)


def cli(argv=None) -> None:
    args = parse_arguments(argv)
    check_required(args)
    seed_everything(args.seed + args.local_rank)
    t0 = perf_counter()
    args = setup_training(args)
    logger.info("TRAINING CONFIG: " + json.dumps({k: v for k, v in vars(args).items()
                                                  if isinstance(v, (int, float, str, bool, list, type(None)))}))
    with open(args.model_config_file) as f:
        logger.info("MODEL CONFIG: " + json.dumps(json.load(f)))
    global_steps, seq_per_sec = main(args)
    runtime = perf_counter() - t0
    logger.info(f"runtime: {runtime:.2f}s  train_time: {getattr(args, 'train_time_s', 0.0):.2f}s  "
                f"training_seq_per_sec: {seq_per_sec:.2f}  global_steps: {global_steps}")
    logger.flush()
    if torch.distributed.is_initialized():
        torch.distributed.destroy_process_group()
