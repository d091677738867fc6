"""Held-out evaluation without a GPU: the held-out set (masks independent of world size, batch size and rebuilds,
pre-masked shards kept, inert filler rows, rank slices), the plain PyTorch ``evaluate`` against a direct torch
computation and over a two-rank ``FakeComm`` world, the runtime flags, and the runtime on CPU with ``--eval_dir``."""
import csv
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bert_pytorch_b200 import BertConfig, pretrain
from bert_pytorch_b200.data import HeldOutSet, hdf5, synthetic
from bert_pytorch_b200.models import BertForPreTraining
from bert_pytorch_b200.parallel.comm import FakeComm

V, S, MP = 1000, 64, 10


def _shards(root, num_shards=3, per=20, seed=0):
    return synthetic.write_shards(str(root), num_shards, per, S, V, next_sentence=True, seed=seed)


def _set(files, n=50, seed=0, **kw):
    return HeldOutSet(files, n, 4, MP, 0.2, V, seed=seed, **kw)


def _cat(batches, n_real=None):
    cols = [torch.cat([b[c] for b in batches]) for c in range(5)]
    return cols if n_real is None else [c[:n_real] for c in cols]


# ---- the held-out set --------------------------------------------------------------------------------------------------
def test_masks_do_not_depend_on_world_size_batch_size_or_rebuilds(tmp_path):
    files = _shards(tmp_path / "d")
    a, b = _set(files), _set(list(reversed(files)))
    assert len(a) == 50
    for x, y in zip(a.tensors, b.tensors):
        assert torch.equal(x, y)
    whole = _cat(list(a.batches(7)), 50)
    for c in range(5):
        assert torch.equal(whole[c], a.tensors[c])
    for world in (2, 3):
        for bs in (4, 16):
            parts = []
            for r in range(world):
                lo, hi = a.rank_range(r, world)
                parts.append(_cat(list(a.batches(bs, r, world)), hi - lo))
            for c in range(5):
                assert torch.equal(torch.cat([p[c] for p in parts]), a.tensors[c]), (world, bs, c)
    # a different seed draws different masks; a smaller set is a prefix of a larger one
    assert not torch.equal(_set(files, seed=1).tensors[3], a.tensors[3])
    small = _set(files, n=13)
    for c in range(5):
        assert torch.equal(small.tensors[c], a.tensors[c][:13])


def test_set_holds_int32_labels_inside_the_training_masking_rules(tmp_path):
    s = _set(_shards(tmp_path / "d"))
    ids, seg, mask, labels, nsl = s.tensors
    assert all(t.dtype == torch.int32 for t in s.tensors) and ids.shape == (50, S) and nsl.shape == (50,)
    n = (labels >= 0).sum(dim=1)
    assert (n >= 1).all() and (n <= MP).all()
    assert ((labels < 0) | (mask > 0)).all()          # labels lie inside the attention mask
    assert (labels[:, 0] < 0).all()                   # [CLS] is never a target


def test_more_samples_than_the_shards_hold_takes_them_all(tmp_path):
    assert len(_set(_shards(tmp_path / "d", num_shards=2, per=8), n=1000)) == 16


def _legacy(path, N=6, L=16):
    ids = np.random.default_rng(0).integers(5, 100, size=(N, L), dtype=np.int32)
    pos = np.zeros((N, 4), dtype=np.int32); pos[:, 0] = 3; pos[:, 1] = 7
    mids = np.zeros((N, 4), dtype=np.int32); mids[:, 0] = 11; mids[:, 1] = 12
    with hdf5.File(path, "w") as f:
        for k, v in dict(input_ids=ids, segment_ids=np.zeros_like(ids), input_mask=np.ones_like(ids),
                         masked_lm_positions=pos, masked_lm_ids=mids,
                         next_sentence_labels=np.zeros(N, dtype=np.int8)).items():
            f.create_dataset(k, data=v, compression="gzip")
    return ids


def test_premasked_shard_keeps_its_stored_masks(tmp_path):
    p = str(tmp_path / "legacy.hdf5")
    ids = _legacy(p)
    s = HeldOutSet([p], 4, None, 4, 0.15, 100)
    labels = s.tensors[3].numpy()
    assert (labels[:, 3] == 11).all() and (labels[:, 7] == 12).all()
    assert (np.delete(labels, [3, 7], axis=1) == -1).all()
    assert np.array_equal(s.tensors[0].numpy(), ids[:4])
    with pytest.raises(ValueError, match="max_predictions_per_seq"):
        HeldOutSet([p], 4, None, 1, 0.15, 100)


def test_filler_rows_are_inert(tmp_path):
    s = _set(_shards(tmp_path / "d"), n=10)
    batches = list(s.batches(8))
    assert [b[0].size(0) for b in batches] == [8, 8]
    ids, seg, mask, labels, nsl = (t[2:] for t in batches[-1])
    assert (labels == -1).all() and (nsl == -1).all()
    assert (mask[:, 0] == 1).all() and (mask[:, 1:] == 0).all()
    assert (ids == 0).all() and (seg == 0).all()


def test_rank_slices_cover_every_sample_once(tmp_path):
    s = _set(_shards(tmp_path / "d"), n=37)
    for world in (1, 2, 4, 5, 37, 40):
        seen = []
        for r in range(world):
            lo, hi = s.rank_range(r, world)
            seen += list(range(lo, hi))
        assert seen == list(range(37)), world


# ---- evaluate on the plain PyTorch path --------------------------------------------------------------------------------
def _model(nsp=True):
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=V, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=128, max_position_embeddings=S, next_sentence=nsp)
    cfg.max_predictions_per_seq = MP
    m = BertForPreTraining(cfg)
    m.train()
    return m


def _direct(model, batch):
    """The metrics straight from torch: eval-mode forward, cross-entropy and argmax over the labelled rows."""
    ids, seg, mask, labels, nsl = (t.long() for t in batch)
    model.eval()
    with torch.no_grad():
        scores, nsp = model(ids, seg, mask)
    model.train()
    out = []
    for sc, lab in ((scores.reshape(-1, V), labels.reshape(-1)), (nsp, nsl)):
        if sc is None:
            out += [0.0, 0.0, 0.0]
            continue
        k = lab >= 0
        out += [F.cross_entropy(sc[k].double(), lab[k], reduction="sum").item(),
                float((sc[k].argmax(-1) == lab[k]).sum()), float(k.sum())]
    return out


@pytest.mark.parametrize("nsp", [True, False])
def test_oracle_evaluate_matches_a_direct_torch_computation(tmp_path, nsp):
    s = _set(_shards(tmp_path / "d"), n=20)
    model = _model(nsp)
    acc = torch.zeros(6, dtype=torch.float64)
    want = np.zeros(6)
    for batch in s.batches(8):
        model.evaluate(*batch, acc)
        want += np.array(_direct(model, batch))
    assert model.training                                  # the training flag comes out as it went in
    got = acc.numpy()
    assert got[2] == want[2] == (s.tensors[3] >= 0).sum().item()
    assert got[1] == want[1] and got[4] == want[4] and got[5] == want[5]
    assert abs(got[0] - want[0]) <= 1e-5 * want[0] and abs(got[3] - want[3]) <= 1e-5 * max(want[3], 1.0)
    if nsp:
        assert got[5] == 20
    else:
        assert not got[3:].any()


def test_oracle_evaluate_ties_go_to_the_lowest_index():
    from bert_pytorch_b200.models.modeling import _metric_sums
    scores = torch.tensor([[1.0, 3.0, 3.0, 0.0], [2.0, 2.0, 2.0, 2.0], [0.0, 5.0, 1.0, 5.0]])
    s = _metric_sums(scores, torch.tensor([2, 0, 1]))
    assert s[1].item() == 2 and s[2].item() == 3


def test_two_rank_world_matches_one_rank(tmp_path):
    s = _set(_shards(tmp_path / "d"), n=24)          # each rank's batches are batches of the one-rank run: equal rows
    # the ranks are threads sharing one model: in training mode, one rank's evaluate could switch the training flag
    # (and with it dropout) back on while the other rank's forward runs
    model = _model().eval()

    def run(comm):
        acc = torch.zeros(6, dtype=torch.float64)
        for batch in s.batches(4, comm.rank, comm.world_size):
            model.evaluate(*batch, acc)
        comm.all_reduce_(acc)
        return acc

    one = FakeComm.spawn(1, run)[0]
    two = FakeComm.spawn(2, run)
    assert torch.equal(two[0], two[1])
    for i in (1, 2, 4, 5):
        assert two[0][i].item() == one[i].item()
    for i in (0, 3):
        assert abs(two[0][i].item() - one[i].item()) <= 1e-12 * abs(one[i].item())


# ---- flags and runtime -------------------------------------------------------------------------------------------------
def test_flag_defaults_json_keys_and_help(tmp_path):
    a = pretrain.parse_arguments(["--output_dir", "o"])
    assert (a.eval_dir, a.num_eval_examples, a.eval_batch_size, a.eval_interval, a.eval_seed) == (None, 10000, None, 0, 0)
    cfg = tmp_path / "c.json"
    cfg.write_text(json.dumps({"eval_dir": "e", "num_eval_examples": 64, "eval_batch_size": 16, "eval_interval": 5,
                               "eval_seed": 3}))
    a = pretrain.parse_arguments(["--output_dir", "o", "--config_file", str(cfg), "--eval_seed", "7"])
    assert (a.eval_dir, a.num_eval_examples, a.eval_batch_size, a.eval_interval, a.eval_seed) == ("e", 64, 16, 5, 7)
    helps = {a.dest: a.help for a in pretrain.build_parser()._actions}
    for k in ("eval_dir", "num_eval_examples", "eval_batch_size", "eval_interval", "eval_seed"):
        assert helps[k], k


def _workspace(root):
    data, model_json, _ = synthetic.make_workspace(
        str(root / "ws"), num_shards=2, samples_per_shard=40, seq_len=S, vocab_size=V, hidden_size=64,
        num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, max_position_embeddings=S,
        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    eval_dir = str(root / "eval")
    synthetic.write_shards(eval_dir, 2, 12, S, V, next_sentence=True, seed=99)
    return data, model_json, eval_dir


def _argv(data, model_json, out, steps, extra=()):
    return ["--input_dir", data, "--output_dir", out, "--model_config_file", model_json, "--steps", str(steps),
            "--max_steps", "10", "--global_batch_size", "16", "--local_batch_size", "8", "--max_predictions_per_seq",
            str(MP), "--num_steps_per_checkpoint", "2", "--disable_progress_bar", "--device", "cpu",
            "--learning_rate", "1e-3", *extra]


def test_runtime_on_cpu_logs_eval_rows(tmp_path):
    data, model_json, eval_dir = _workspace(tmp_path)
    out = str(tmp_path / "out")
    pretrain.cli(_argv(data, model_json, out, 3, ["--eval_dir", eval_dir, "--num_eval_examples", "20",
                                                  "--eval_batch_size", "6", "--eval_interval", "2"]))
    rows = list(csv.DictReader(open(os.path.join(out, "logfile_metrics.csv"))))
    ev = [r for r in rows if r["tag"] == "eval"]
    assert [int(r["step"]) for r in ev] == [2, 3]
    for r in ev:
        assert np.isfinite(float(r["eval_mlm_loss"])) and np.isfinite(float(r["eval_nsp_loss"]))
        assert 0.0 <= float(r["eval_mlm_accuracy"]) <= 1.0 and 0.0 <= float(r["eval_nsp_accuracy"]) <= 1.0
        assert int(float(r["eval_samples"])) == 20 and float(r["eval_seconds"]) > 0
    assert [int(r["step"]) for r in rows if r["tag"] == "train"] == [1, 2, 3]

    plain = str(tmp_path / "plain")
    pretrain.cli(_argv(data, model_json, plain, 3))
    rows = list(csv.DictReader(open(os.path.join(plain, "logfile_metrics.csv"))))
    assert all(r["tag"] == "train" for r in rows) and "eval_mlm_loss" not in rows[0]
