"""Sharded HDF5 pre-training data: dataset, resumable sampler, dynamic masking and a
batched, pinned-memory loader.

Parity targets (reference file:line):
  * ``ShardedPretrainingDataset`` -- src/dataset.py:9-338: sorted file list, per-file
    ``(start, end)`` sample index built by opening every file once, at most two files
    resident with the next one prefetched by a background thread, sequential-access
    contract, dynamic masking or the legacy pre-masked NVIDIA schema, five int64 arrays
    per sample.
  * ``DistributedSampler`` -- src/dataset.py:341-428: one *contiguous* chunk of the
    index space per rank, is its own iterator, ``state_dict`` = ``{epoch, seed,
    num_replicas, total_size, index}`` with the changed-size / changed-world guards.

Design differences (H100-first; an H100 eats ~3k sequences/s so the reference's
per-token Python loop x 4 DataLoader workers per rank cannot feed eight of them):
  * masking is vectorised over the whole micro-batch (:func:`mask_batch`, numpy here,
    multi-threaded C++ in ops/csrc/host.cpp when built) and writes straight into pinned
    staging buffers; one background thread per rank keeps a ring of batches ready
    (:class:`BatchedPretrainingLoader`) and the H2D copies go out on a side stream;
  * quirks fixed on purpose: the cached shard is never mutated (Q3), every producer has
    its own seeded generator (Q5), the sampler position stored in a checkpoint is the
    *consumed* position, not the prefetched one (Q6), ``math`` is imported (Q1), the
    empty-dataset check looks at the verified list (Q2).
"""
from __future__ import annotations

import math
import os
import queue
import threading
import warnings
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import hdf5

# ---------------------------------------------------------------------------
# masking
# ---------------------------------------------------------------------------


def segment_ids_and_input_mask(input_ids: np.ndarray, special_pos: np.ndarray
                               ) -> Tuple[np.ndarray, np.ndarray]:
    """Vectorised ``_get_segment_ids`` / ``_get_input_mask`` for a batch
    (src/dataset.py:224-252).  ``special_pos`` is [B, 2] or [B, 3]."""
    B, S = input_ids.shape
    pos = np.arange(S, dtype=np.int32)[None, :]
    last = special_pos[:, -1:].astype(np.int32)
    input_mask = (pos <= last).astype(input_ids.dtype)
    if special_pos.shape[1] == 3:
        sep1 = special_pos[:, 1:2].astype(np.int32)
        seg = ((pos > sep1) & (pos <= last)).astype(input_ids.dtype)
    else:
        seg = np.zeros_like(input_ids)
    return seg, input_mask


def mask_batch(input_ids: np.ndarray, special_pos: np.ndarray, *, mask_token_index: int,
               max_pred_per_seq: int, masked_lm_prob: float, vocab_size: int,
               original_token_prob: float = 0.1, random_token_prob: float = 0.1,
               rng: Optional[np.random.Generator] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Dynamic masking of a whole batch with the sampling semantics of
    src/dataset.py:277-296: candidates are the positions before the last special token
    that are not special tokens; ``mask_count = min(max_pred, max(1, int(n * p)))`` draws
    *with replacement*; each draw keeps (10%), randomises in ``[0, vocab_size-1)`` (10%) or
    writes ``[MASK]`` (80%); draws are applied in order so a later draw on the same
    position overrides an earlier one exactly like the reference's Python loop.
    Returns new arrays ``(masked_ids, labels)``; ``labels`` is -1 off the drawn set.
    """
    rng = rng or np.random.default_rng()
    B, S = input_ids.shape
    ids = input_ids.copy()
    labels = np.full((B, S), -1, dtype=input_ids.dtype)
    nsp = special_pos.shape[1]
    last = special_pos[:, -1].astype(np.int64)
    n_cand = np.maximum(last - (nsp - 1), 0)                    # specials before `last`: nsp-1
    count = np.minimum(max_pred_per_seq, np.maximum(1, (n_cand * masked_lm_prob).astype(np.int64)))
    count = np.where(n_cand > 0, count, 0)
    max_count = int(count.max()) if B else 0
    if max_count == 0:
        return ids, labels
    rows = np.arange(B)
    draw_k = (rng.random((B, max_count)) * n_cand[:, None]).astype(np.int64)
    draw_k = np.minimum(draw_k, np.maximum(n_cand[:, None] - 1, 0))
    action = rng.random((B, max_count))
    rand_tok = rng.integers(0, max(vocab_size - 1, 1), size=(B, max_count))
    inner = np.sort(special_pos[:, :-1].astype(np.int64), axis=1)   # specials strictly before `last`
    for j in range(max_count):
        live = j < count
        pos = draw_k[:, j].copy()
        for s in range(inner.shape[1]):                       # k-th candidate -> sequence position
            pos += (pos >= inner[:, s]).astype(np.int64)
        pos = np.where(live, pos, 0)
        lab = input_ids[rows, pos]
        labels[rows[live], pos[live]] = lab[live]
        a = action[:, j]
        to_rand = live & (a >= original_token_prob) & (a < original_token_prob + random_token_prob)
        to_mask = live & (a >= original_token_prob + random_token_prob)
        ids[rows[to_rand], pos[to_rand]] = rand_tok[to_rand, j].astype(ids.dtype)
        ids[rows[to_mask], pos[to_mask]] = mask_token_index
    return ids, labels


def labels_from_premasked(input_ids: np.ndarray, masked_lm_positions: np.ndarray,
                          masked_lm_ids: np.ndarray) -> np.ndarray:
    """Legacy NVIDIA schema (src/dataset.py:254-275): positions are zero padded; the first
    zero terminates the list."""
    B, S = input_ids.shape
    labels = np.full((B, S), -1, dtype=input_ids.dtype)
    for b in range(B):
        pos = masked_lm_positions[b]
        zeros = np.nonzero(pos == 0)[0]
        n = int(zeros[0]) if len(zeros) else len(pos)
        labels[b, pos[:n]] = masked_lm_ids[b, :n]
    return labels


# ---------------------------------------------------------------------------
# dataset
# ---------------------------------------------------------------------------

_REQUIRED_KEYS = ("input_ids", "next_sentence_labels")


class ShardedPretrainingDataset(torch.utils.data.Dataset):
    def __init__(self, files, mask_token_index: Optional[int], max_pred_per_seq: int,
                 masked_lm_prob: float, vocab_size: int, original_token_prob: float = 0.1,
                 random_token_prob: float = 0.1, shuffle: bool = False, seed: Optional[int] = None):
        if mask_token_index is not None and not isinstance(mask_token_index, (int, np.integer)):
            raise ValueError("mask_token_index must be an integer")
        if not isinstance(max_pred_per_seq, (int, np.integer)) or max_pred_per_seq < 0:
            raise ValueError("max_pred_per_seq must be an integer >= 0")
        if not 0 <= masked_lm_prob <= 1:
            raise ValueError("masked_lm_prob must be in [0,1]")
        if not isinstance(vocab_size, (int, np.integer)) or vocab_size < 0:
            raise ValueError("vocab_size must be an integer >= 0")
        for name, v in (("original_token_prob", original_token_prob), ("random_token_prob", random_token_prob)):
            if not 0 <= v <= 1:
                raise ValueError(f"{name} must be in [0,1]")
        if original_token_prob + random_token_prob > 1:
            raise ValueError("random_token_prob + original_token_prob > 1")
        if shuffle:
            raise ValueError("shuffling is not supported; pre-shuffle the samples in the input files")
        if isinstance(files, (str, os.PathLike)):
            files = [files]
        files = sorted(os.fspath(f) for f in files)      # every rank sees the same order
        self.files, self.file_idxs = self._verify_and_count_samples(files)
        self.mask_token_index = mask_token_index
        self.max_pred_per_seq = int(max_pred_per_seq)
        self.masked_lm_prob = float(masked_lm_prob)
        self.vocab_size = int(vocab_size)
        self.original_token_prob = original_token_prob
        self.random_token_prob = random_token_prob
        self.shuffle = shuffle
        self.seed = seed
        self.epoch = 0
        self._rng = np.random.default_rng(seed)
        # shard cache: current + prefetched next
        self._lock = threading.Lock()
        self._cur_idx: Optional[int] = None
        self._cur: Optional[Dict[str, np.ndarray]] = None
        self._next_idx: Optional[int] = None
        self._next_thread: Optional[threading.Thread] = None
        self._next_data: Optional[Dict[str, np.ndarray]] = None

    # -- bookkeeping --------------------------------------------------------
    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def reseed(self, seed: int) -> None:
        self.seed = seed
        self._rng = np.random.default_rng(seed)

    def __len__(self) -> int:
        return self.file_idxs[-1][1]

    @staticmethod
    def _verify_and_count_samples(files: Sequence[str]):
        cur = 0
        ok_files: List[str] = []
        idxs: List[Tuple[int, int]] = []
        for fp in files:
            if not os.path.isfile(fp):
                warnings.warn(f"File not found: {fp}. Skipping file")
                continue
            try:
                with hdf5.File(fp, "r") as f:
                    counts = [len(f[k]) for k in _REQUIRED_KEYS]
            except Exception as e:  # noqa: BLE001 - mirror the reference: skip anything unreadable
                warnings.warn(f"Unable to read keys {_REQUIRED_KEYS} from {fp} ({e}). Skipping file")
                continue
            if len(set(counts)) != 1:
                warnings.warn(f"Number of samples per key in {fp} do not match. Skipping file")
                continue
            ok_files.append(fp)
            idxs.append((cur, cur + counts[0]))
            cur += counts[0]
        if not ok_files:
            raise RuntimeError("Unable to open any valid data files")
        return ok_files, idxs

    def file_index_of(self, idx: int) -> int:
        lo, hi = 0, len(self.file_idxs) - 1
        if not 0 <= idx < len(self):
            raise ValueError(f"idx ({idx}) exceeds dataset size ({len(self)})")
        while lo < hi:
            mid = (lo + hi) // 2
            if idx >= self.file_idxs[mid][1]:
                lo = mid + 1
            else:
                hi = mid
        return lo

    # -- shard cache ----------------------------------------------------------
    @staticmethod
    def _load_file(path: str) -> Dict[str, np.ndarray]:
        with hdf5.File(path, "r") as f:
            return {k: np.asarray(f[k][:]) for k in f.keys()}

    def _start_prefetch(self, file_idx: int) -> None:
        def work():
            self._next_data = self._load_file(self.files[file_idx])
        self._next_idx = file_idx
        self._next_data = None
        self._next_thread = threading.Thread(target=work, daemon=True)
        self._next_thread.start()

    def shard(self, file_idx: int) -> Dict[str, np.ndarray]:
        """Arrays of shard ``file_idx`` (read-only); keeps the next shard loading in the
        background.  At most two shards are resident."""
        with self._lock:
            if self._cur_idx == file_idx and self._cur is not None:
                return self._cur
            if self._next_idx == file_idx and self._next_thread is not None:
                self._next_thread.join()
                data = self._next_data
            else:
                if self._next_thread is not None:
                    self._next_thread.join()
                data = self._load_file(self.files[file_idx])
            self._cur, self._cur_idx = data, file_idx
            self._start_prefetch((file_idx + 1) % len(self.files))
            return self._cur

    # -- batch / sample construction --------------------------------------------
    def build_batch(self, file_idx: int, lo: int, hi: int, rng: Optional[np.random.Generator] = None
                    ) -> List[np.ndarray]:
        """Rows ``[lo, hi)`` (file-local) of shard ``file_idx`` as the five model inputs
        ``[input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels]``."""
        d = self.shard(file_idx)
        ids = d["input_ids"][lo:hi]
        nsl = np.asarray(d["next_sentence_labels"][lo:hi])
        if "special_token_positions" in d:
            sp = d["special_token_positions"][lo:hi]
            seg, imask = segment_ids_and_input_mask(ids, sp)
            masked, labels = self._mask(ids, sp, rng or self._rng)
        else:
            seg, imask = d["segment_ids"][lo:hi], d["input_mask"][lo:hi]
            masked = ids
            labels = labels_from_premasked(ids, d["masked_lm_positions"][lo:hi], d["masked_lm_ids"][lo:hi])
            # legacy pre-masked shards carry their own number of targets: the fused MLM head compacts at most
            # max_predictions_per_seq rows per sequence (static shapes), anything beyond would be dropped silently
            # (ADVICE r1) -- refuse instead; the reference criterion would have used every label
            if self.max_pred_per_seq > 0:
                worst = int((labels >= 0).sum(axis=1).max()) if labels.size else 0
                if worst > self.max_pred_per_seq:
                    raise ValueError(f"pre-masked shard has {worst} masked tokens in one sequence but "
                                     f"--max_predictions_per_seq is {self.max_pred_per_seq}; raise the flag")
        return [masked, seg, imask, labels, nsl]

    def _mask(self, ids, sp, rng):
        from ..ops import native_host
        nat = native_host.load_or_none()
        kw = dict(mask_token_index=int(self.mask_token_index), max_pred_per_seq=self.max_pred_per_seq,
                  masked_lm_prob=self.masked_lm_prob, vocab_size=self.vocab_size,
                  original_token_prob=self.original_token_prob, random_token_prob=self.random_token_prob)
        if nat is not None and ids.dtype == np.int32 and sp.dtype == np.int32:
            return native_host.mask_batch(nat, ids, sp, seed=int(rng.integers(0, 2 ** 62)), **kw)
        return mask_batch(ids, sp, rng=rng, **kw)

    def __getitem__(self, idx: int) -> List[np.ndarray]:
        fi = self.file_index_of(idx)
        # sequential-access contract of the reference: only the current or the next shard
        if self._cur_idx is not None and fi not in (self._cur_idx, (self._cur_idx + 1) % len(self.files)):
            raise RuntimeError(
                f"idx ({idx}) is outside the resident shards; samples must be read in order "
                "(e.g. do not use a shuffling sampler)")
        lo = idx - self.file_idxs[fi][0]
        out = self.build_batch(fi, lo, lo + 1)
        return [np.asarray(a[0]).astype(np.int64) for a in out]


# ---------------------------------------------------------------------------
# sampler
# ---------------------------------------------------------------------------


class DistributedSampler(torch.utils.data.Sampler):
    """Contiguous-chunk distributed sampler that is its own (resumable) iterator."""

    def __init__(self, dataset, num_replicas: Optional[int] = None, rank: Optional[int] = None,
                 shuffle: bool = False, seed: int = 0, drop_last: bool = False):
        from ..utils import dist as D
        if num_replicas is None:
            num_replicas = D.get_world_size()
        if rank is None:
            rank = D.get_rank()
        if not 0 <= rank < num_replicas:
            raise ValueError(f"invalid rank {rank} for {num_replicas} replicas")
        self.dataset, self.num_replicas, self.rank = dataset, num_replicas, rank
        self.seed, self.drop_last, self.epoch = seed, drop_last, 0
        self.shuffle = False
        n = len(dataset)
        if drop_last and n % num_replicas != 0:
            self.num_samples = math.ceil((n - num_replicas) / num_replicas)
        else:
            self.num_samples = math.ceil(n / num_replicas)
        self.total_size = self.num_samples * num_replicas
        self._n = n
        self.index = 0
        if hasattr(dataset, "seed") and getattr(dataset, "seed", None) is None:
            dataset.reseed(seed + rank) if hasattr(dataset, "reseed") else setattr(dataset, "seed", seed)

    def global_index(self, i: int) -> int:
        """Dataset index of this rank's ``i``-th sample (padding wraps around, the
        drop_last tail is cut -- src/dataset.py:364-382)."""
        g = i + self.rank * self.num_samples
        return g % self._n if g >= self._n else g

    def __len__(self) -> int:
        return self.num_samples

    def __iter__(self) -> Iterator[int]:
        return self

    def __next__(self) -> int:
        if self.index == self.num_samples:
            self.index = 0
            raise StopIteration
        x = self.global_index(self.index)
        self.index += 1
        return x

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch
        if hasattr(self.dataset, "set_epoch"):
            self.dataset.set_epoch(epoch)

    def state_dict(self) -> Dict[str, int]:
        return {"epoch": self.epoch, "seed": self.seed, "num_replicas": self.num_replicas,
                "total_size": self.total_size, "index": self.index}

    def load_state_dict(self, state: Dict[str, int]) -> None:
        if state["total_size"] != self.total_size:
            warnings.warn(f"The number of samples in the sampler changed (expected {self.total_size}, "
                          f"got {state['total_size']}); not restoring the sampler state. Ignore this "
                          "message if the dataset was changed on purpose (e.g. phase 1 -> phase 2)")
            return
        if state["num_replicas"] != self.num_replicas:
            warnings.warn("The number of replicas changed so the saved sampler index is no longer "
                          "valid; not restoring the sampler state")
            return
        self.epoch, self.seed, self.index = state["epoch"], state["seed"], state["index"]


# ---------------------------------------------------------------------------
# batched loader (the fast path)
# ---------------------------------------------------------------------------


class BatchedPretrainingLoader:
    """Yields micro-batches as five tensors (int32 in pinned host memory when CUDA is
    present; the model casts on device).  One producer thread walks the sampler's
    contiguous range, cuts it at shard boundaries, masks each piece with the vectorised
    kernel and fills a ring of staging buffers ``depth`` deep.

    ``state_dict()['index']`` is the number of samples *handed to the training loop*, so a
    resume neither repeats nor skips samples (fixes reference quirk Q6), and the mask RNG is keyed by
    (seed, rank, epoch, batch position): 5 + 5 steps reproduce 10 steps exactly (tests/test_pretrain_cpu.py).
    """

    def __init__(self, dataset: ShardedPretrainingDataset, sampler: DistributedSampler, batch_size: int,
                 depth: int = 4, pin_memory: Optional[bool] = None, drop_last: bool = False,
                 dtype: torch.dtype = torch.int32):
        self.dataset, self.sampler, self.batch_size = dataset, sampler, int(batch_size)
        self.depth, self.drop_last, self.dtype = depth, drop_last, dtype
        self.pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self._thread: Optional[threading.Thread] = None
        self._q: "queue.Queue" = queue.Queue(maxsize=depth)
        self._stop = threading.Event()
        self._consumed = sampler.index

    def __len__(self) -> int:
        n = len(self.sampler) - self.sampler.index
        return n // self.batch_size if self.drop_last else math.ceil(n / self.batch_size)

    def _pieces(self, start: int, stop: int):
        """Split this rank's sample range [start, stop) into shard-contiguous runs."""
        i = start
        while i < stop:
            g = self.sampler.global_index(i)
            fi = self.dataset.file_index_of(g)
            f_lo, f_hi = self.dataset.file_idxs[fi]
            run = min(stop - i, f_hi - g)
            # the padded tail may wrap to index 0
            yield fi, g - f_lo, g - f_lo + run
            i += run

    def _produce(self, start: int, seed: Sequence[int]) -> None:
        n = len(self.sampler)
        i = start
        try:
            while i < n and not self._stop.is_set():
                j = min(i + self.batch_size, n)
                if self.drop_last and j - i < self.batch_size:
                    break
                # masks are a function of (seed, rank, epoch, first sample of the batch): a run resumed from a
                # checkpoint draws exactly the masks the uninterrupted run would have drawn
                rng = np.random.default_rng([*seed, i])
                parts = [self.dataset.build_batch(fi, lo, hi, rng) for fi, lo, hi in self._pieces(i, j)]
                cols = [np.concatenate([p[c] for p in parts], axis=0) if len(parts) > 1 else parts[0][c]
                        for c in range(5)]
                tensors = []
                for c in cols:
                    t = torch.from_numpy(np.ascontiguousarray(c)).to(self.dtype)
                    if self.pin:
                        t = t.pin_memory()
                    tensors.append(t)
                self._q.put((j - i, tensors))
                i = j
        except BaseException as e:  # noqa: BLE001 - surface in the consumer
            self._q.put(e)
            return
        self._q.put(None)

    def __iter__(self):
        self.close()
        self._stop.clear()
        self._q = queue.Queue(maxsize=self.depth)
        start = self.sampler.index
        self._consumed = start
        seed = (int(self.dataset.seed or 0) & 0x7FFFFFFF, int(self.sampler.rank), int(self.sampler.epoch))
        self._thread = threading.Thread(target=self._produce, args=(start, seed), daemon=True)
        self._thread.start()
        while True:
            item = self._q.get()
            if item is None:
                self.sampler.index = 0
                self._consumed = 0
                return
            if isinstance(item, BaseException):
                raise item
            n, tensors = item
            self._consumed += n
            self.sampler.index = self._consumed
            yield tensors

    def close(self) -> None:
        if self._thread is not None and self._thread.is_alive():
            self._stop.set()
            try:
                while True:
                    self._q.get_nowait()
            except queue.Empty:
                pass
            self._thread.join(timeout=5)
        self._thread = None

    def state_dict(self) -> Dict[str, int]:
        sd = self.sampler.state_dict()
        sd["index"] = self._consumed
        return sd


def _smoke(argv=None) -> int:
    """Loader smoke loop (reference: src/dataset.py:431-505): run under torchrun (gloo) or stand-alone, walk
    ``--epochs`` epochs of this rank's share and report sizes + samples/s.
    ``python -m bert_pytorch_b200.data.dataset --input_dir DIR [--batch_size 8] [--epochs 2]``"""
    import argparse
    import time
    from pathlib import Path

    p = argparse.ArgumentParser(description="Dataloader test")
    p.add_argument("--input_dir", required=True, help="an .hdf5 shard or a directory of shards")
    p.add_argument("--max_predictions_per_seq", default=80, type=int)
    p.add_argument("--masked_lm_prob", type=float, default=0.15)
    p.add_argument("--batch_size", type=int, default=8)
    p.add_argument("--epochs", type=int, default=2)
    p.add_argument("--mask_token_index", type=int, default=103)
    p.add_argument("--vocab_size", type=int, default=30000)
    p.add_argument("--local_rank", type=int, default=0)
    a = p.parse_args(argv)

    import torch.distributed as dist
    if "RANK" in os.environ and not dist.is_initialized():
        dist.init_process_group(backend="gloo", init_method="env://")
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    files = [a.input_dir] if os.path.isfile(a.input_dir) else sorted(
        str(x) for x in Path(a.input_dir).rglob("*.hdf5") if x.is_file())
    dataset = ShardedPretrainingDataset(files, a.mask_token_index, a.max_predictions_per_seq, a.masked_lm_prob,
                                        vocab_size=a.vocab_size)
    sampler = DistributedSampler(dataset, world, rank=rank)
    loader = BatchedPretrainingLoader(dataset, sampler, a.batch_size, pin_memory=False)
    if rank == 0:
        print(f"[rank {rank}] Found {len(files)} input files")
        print(f"[rank {rank}] Dataset size = {len(dataset)}")
        print(f"[rank {rank}] Dataloader size = {len(loader)}")
        print(f"[rank {rank}] Sampler num_samples = {len(sampler)}")
        print(f"[rank {rank}] Sampler total_size = {sampler.total_size}")
    for epoch in range(a.epochs):
        sampler.set_epoch(epoch)
        t0, n = time.time(), 0
        for batch in loader:
            n += batch[0].size(0)
        print(f"[rank {rank}] epoch {epoch}: {n} samples, {n / max(time.time() - t0, 1e-9):.0f} samples/s", flush=True)
    loader.close()
    if dist.is_initialized():
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(_smoke())
