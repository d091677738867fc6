"""GLUE sentence(-pair) classification data: the tab-separated files of each task as ``download_glue_data.py`` writes
them, their features for ``BertForSequenceClassification``, and the task metrics.

Every task directory holds ``train.tsv``, ``dev.tsv`` and ``test.tsv`` (MNLI: ``dev_matched.tsv`` /
``dev_mismatched.tsv`` and ``test_matched.tsv`` / ``test_mismatched.tsv``).  Columns, counted from 0:

=====  ===============================================  ===============================  ==========================
task   train / dev (a, b, label)                        test (index, a, b)               labels
=====  ===============================================  ===============================  ==========================
CoLA   no header; 3, -, 1                               header; 0, 1, -                  0 1
SST-2  header; 0, -, 1                                  header; 0, 1, -                  0 1
MRPC   header; 3, 4, 0                                  header; 0, 3, 4                  0 1
QQP    header; 3, 4, 5                                  header; 0, 1, 2                  0 1
MNLI   header; 8, 9, last                               header; 0, 8, 9                  contradiction entailment
                                                                                         neutral
QNLI   header; 1, 2, 3                                  header; 0, 1, 2                  entailment not_entailment
RTE    header; 1, 2, 3                                  header; 0, 1, 2                  entailment not_entailment
WNLI   header; 1, 2, 3                                  header; 0, 1, 2                  0 1
=====  ===============================================  ===============================  ==========================

The files are read as plain tab-separated lines (no quote processing: GLUE's sentences contain unbalanced quotes).
STS-B is a regression task and is not served here.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class Example:
    guid: str              # "<split>-<line>" for train / dev, the file's index column for test
    text_a: str
    text_b: Optional[str]
    label: Optional[str]   # None for the test split


@dataclass(frozen=True)
class _Layout:
    header: bool
    a: int
    b: Optional[int]
    label: Optional[int]   # None: the last column


@dataclass(frozen=True)
class Task:
    name: str                               # the submission file's stem
    labels: Tuple[str, ...]
    train: _Layout
    test: _Layout                           # ``label`` unused; ``index`` column 0
    dev_files: Tuple[Tuple[str, str], ...]  # (result name, file)
    test_files: Tuple[Tuple[str, str], ...]  # (submission stem, file)
    metrics: Tuple[str, ...]

    @property
    def num_labels(self) -> int:
        return len(self.labels)


def _task(name, labels, train, test, metrics=("acc",), dev=None, tests=None) -> Task:
    return Task(name, tuple(labels), _Layout(*train), _Layout(*test),
                dev or ((name, "dev.tsv"),), tests or ((name, "test.tsv"),), metrics)


_01 = ("0", "1")
_ENT = ("entailment", "not_entailment")
TASKS: Dict[str, Task] = {
    "cola": _task("CoLA", _01, (False, 3, None, 1), (True, 1, None, None), ("mcc",)),
    "sst-2": _task("SST-2", _01, (True, 0, None, 1), (True, 1, None, None)),
    "mrpc": _task("MRPC", _01, (True, 3, 4, 0), (True, 3, 4, None), ("acc", "f1")),
    "qqp": _task("QQP", _01, (True, 3, 4, 5), (True, 1, 2, None), ("acc", "f1")),
    "mnli": _task("MNLI", ("contradiction", "entailment", "neutral"), (True, 8, 9, None), (True, 8, 9, None),
                  dev=(("MNLI-m", "dev_matched.tsv"), ("MNLI-mm", "dev_mismatched.tsv")),
                  tests=(("MNLI-m", "test_matched.tsv"), ("MNLI-mm", "test_mismatched.tsv"))),
    "qnli": _task("QNLI", _ENT, (True, 1, 2, 3), (True, 1, 2, None)),
    "rte": _task("RTE", _ENT, (True, 1, 2, 3), (True, 1, 2, None)),
    "wnli": _task("WNLI", _01, (True, 1, 2, 3), (True, 1, 2, None)),
}


def get_task(name: str) -> Task:
    key = name.lower()
    if key in ("sts-b", "stsb"):
        raise ValueError("STS-B is a regression task; only GLUE's classification tasks are supported "
                         f"({', '.join(sorted(TASKS))})")
    if key not in TASKS:
        raise ValueError(f"unknown GLUE task {name!r}; choose one of {', '.join(sorted(TASKS))}")
    return TASKS[key]


def _rows(path: str, header: bool) -> List[List[str]]:
    with open(path, encoding="utf-8") as f:
        lines = [ln.rstrip("\r\n") for ln in f]
    return [ln.split("\t") for ln in (lines[1:] if header else lines) if ln]


def read_examples(task: Task, path: str, split: str) -> List[Example]:
    """The examples of one file; ``split`` is "train", "dev" or "test".  Lines with too few columns are skipped (QQP's
    training file has a few)."""
    test = split == "test"
    lay = task.test if test else task.train
    need = max(c for c in (lay.a, lay.b, lay.label, 0) if c is not None) + 1
    out = []
    for i, r in enumerate(_rows(path, lay.header)):
        if len(r) < need:
            continue
        label = None if test else (r[-1] if lay.label is None else r[lay.label])
        if label is not None and label not in task.labels:
            raise ValueError(f"{path}, line {i + 1 + lay.header}: label {label!r} is not one of {task.labels}")
        out.append(Example(guid=r[0] if test else f"{split}-{i}", text_a=r[lay.a],
                           text_b=None if lay.b is None else r[lay.b], label=label))
    return out


def train_examples(task: Task, data_dir: str) -> List[Example]:
    return read_examples(task, os.path.join(data_dir, "train.tsv"), "train")


def dev_sets(task: Task, data_dir: str) -> List[Tuple[str, List[Example]]]:
    return [(name, read_examples(task, os.path.join(data_dir, f), "dev")) for name, f in task.dev_files]


def test_sets(task: Task, data_dir: str) -> List[Tuple[str, List[Example]]]:
    return [(name, read_examples(task, os.path.join(data_dir, f), "test")) for name, f in task.test_files]


# ---- features --------------------------------------------------------------------------------------------------------
def truncate_pair(a: List[int], b: Optional[List[int]], budget: int) -> None:
    """Longest-first truncation in place: drop the last token of the longer sequence (of ``b`` on a tie) until both
    fit in ``budget`` tokens."""
    if b is None:
        del a[max(budget, 0):]
        return
    while len(a) + len(b) > budget:
        (a if len(a) > len(b) else b).pop()


def features(ids_a: List[List[int]], ids_b: Optional[List[Optional[List[int]]]], max_seq_length: int, cls_id: int,
             sep_id: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """int64 ``(input_ids, segment_ids, input_mask)`` [N, max_seq_length]: ``[CLS] a [SEP]`` with segment 0, then
    ``b [SEP]`` with segment 1 where there is a ``b``, zero padding (mask 0) to ``max_seq_length``."""
    n = len(ids_a)
    ids = np.zeros((n, max_seq_length), dtype=np.int64)
    seg = np.zeros_like(ids)
    mask = np.zeros_like(ids)
    for i in range(n):
        a = list(ids_a[i])
        b = None if ids_b is None or ids_b[i] is None else list(ids_b[i])
        truncate_pair(a, b, max_seq_length - (3 if b is not None else 2))
        toks = [cls_id] + a + [sep_id]
        n0 = len(toks)
        if b is not None:
            toks += b + [sep_id]
        ids[i, :len(toks)] = toks
        seg[i, n0:len(toks)] = 1
        mask[i, :len(toks)] = 1
    return ids, seg, mask


class Featurizer:
    """Examples -> feature arrays with the repo's WordPiece tokenizer (the native encoder where it applies)."""

    def __init__(self, vocab_file: str, do_lower_case: bool, max_seq_length: int):
        from .tokenization import FastWordPiece
        self.tok = FastWordPiece(vocab_file, do_lower_case=do_lower_case)
        self.cls_id = self.tok.py.vocab["[CLS]"]
        self.sep_id = self.tok.py.vocab["[SEP]"]
        self.max_seq_length = max_seq_length

    def __call__(self, task: Task, examples: Sequence[Example]):
        """(input_ids, segment_ids, input_mask, labels) as int64 numpy arrays; the label is the index into
        ``task.labels``, -1 for an unlabelled (test) example."""
        a = self.tok.encode_batch([e.text_a for e in examples])
        pairs = [i for i, e in enumerate(examples) if e.text_b is not None]
        b: Optional[List[Optional[List[int]]]] = None
        if pairs:
            b = [None] * len(examples)
            for i, ids in zip(pairs, self.tok.encode_batch([examples[i].text_b for i in pairs])):
                b[i] = ids
        ids, seg, mask = features(a, b, self.max_seq_length, self.cls_id, self.sep_id)
        labels = np.array([-1 if e.label is None else task.labels.index(e.label) for e in examples], dtype=np.int64)
        return ids, seg, mask, labels


def fill_batch(ids, seg, mask, labels, batch_size: int):
    """A short batch (torch tensors [n, S], n <= batch_size) filled up to ``batch_size`` rows with inert examples: one
    unmasked [PAD] token (id 0, segment 0) and label -1.  They add nothing to the loss, its mean or any gradient, so one
    static batch shape (one CUDA graph) serves the whole epoch."""
    import torch
    n, S = ids.shape
    k = batch_size - n
    if k <= 0:
        return ids, seg, mask, labels

    def pad(t, first, fill):
        z = torch.full((k,) + tuple(t.shape[1:]), fill, dtype=t.dtype, device=t.device)
        if first is not None:
            z[:, 0] = first
        return torch.cat([t, z])
    return pad(ids, None, 0), pad(seg, None, 0), pad(mask, 1, 0), pad(labels, None, -1)


# ---- metrics ---------------------------------------------------------------------------------------------------------
def accuracy(pred, label) -> float:
    pred, label = np.asarray(pred), np.asarray(label)
    return float((pred == label).mean()) if label.size else 0.0


def f1_positive(pred, label, positive: int = 1) -> float:
    """F1 of class ``positive``: 2 tp / (2 tp + fp + fn), 0 when there is no positive prediction or label."""
    pred, label = np.asarray(pred) == positive, np.asarray(label) == positive
    tp = float(np.sum(pred & label))
    den = 2 * tp + float(np.sum(pred & ~label)) + float(np.sum(~pred & label))
    return 2 * tp / den if den else 0.0


def matthews_corr(pred, label) -> float:
    """Matthews correlation of a binary prediction; 0 when a margin of the confusion matrix is empty (e.g. one class
    predicted throughout)."""
    pred, label = np.asarray(pred) == 1, np.asarray(label) == 1
    tp = float(np.sum(pred & label))
    tn = float(np.sum(~pred & ~label))
    fp = float(np.sum(pred & ~label))
    fn = float(np.sum(~pred & label))
    den = (tp + fp) * (tp + fn) * (tn + fp) * (tn + fn)
    return (tp * tn - fp * fn) / float(np.sqrt(den)) if den > 0 else 0.0


def compute_metrics(task: Task, pred, label) -> Dict[str, float]:
    out = {}
    for m in task.metrics:
        if m == "acc":
            out["acc"] = accuracy(pred, label)
        elif m == "f1":
            out["f1"] = f1_positive(pred, label)
            out["acc_and_f1"] = (out["acc"] + out["f1"]) / 2
        elif m == "mcc":
            out["mcc"] = matthews_corr(pred, label)
    return out


def write_submission(task: Task, path: str, examples: Sequence[Example], pred) -> None:
    """GLUE's submission format: a header ``index\\tprediction``, then one line per test example with its label
    string."""
    with open(path, "w", encoding="utf-8") as f:
        f.write("index\tprediction\n")
        for e, p in zip(examples, pred):
            f.write(f"{e.guid}\t{task.labels[int(p)]}\n")
