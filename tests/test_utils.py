import csv
import json
import os

import pytest
import torch

from bert_pytorch_b200.data import tokenization as T
from bert_pytorch_b200.utils import checkpoint as ck
from bert_pytorch_b200.utils import logging as L
from bert_pytorch_b200.utils.dist import format_step, get_rank, get_world_size, is_main_process
from bert_pytorch_b200.utils.file_utils import cached_path, url_to_filename


def test_logger_four_sinks(tmp_path):
    L.init(handlers=[L.StreamHandler(verbose=False), L.FileHandler(str(tmp_path / "log.txt")),
                     L.CSVHandler(str(tmp_path / "m.csv")), L.TorchTensorboardHandler(str(tmp_path / "tb"))])
    L.info("hello")
    L.log(tag="train", step=1, loss=2.5, lr=0.1)
    L.log(tag="train", step=2, loss=2.0, lr=0.1, extra=7)
    L.flush(); L.close()
    assert "hello" in open(tmp_path / "log.txt").read()
    rows = list(csv.DictReader(open(tmp_path / "m.csv")))
    assert rows[0]["loss"] == "2.5" and rows[1]["extra"] == "7" and rows[0]["extra"] == ""
    assert os.path.isdir(tmp_path / "tb")
    L.init(handlers=[L.CSVHandler(str(tmp_path / "m.csv"))])            # append on resume
    L.log(tag="train", step=3, loss=1.0, lr=0.1, extra=1)
    L.close()
    assert len(list(csv.DictReader(open(tmp_path / "m.csv")))) == 3


def test_dllogger_facade(tmp_path):
    L.dllogger.init([L.JSONStreamBackend(L.Verbosity.VERBOSE, str(tmp_path / "squad_log.json"))])
    L.dllogger.log(step=(0, 5), data={"step_loss": 1.5})
    L.dllogger.log(step="PARAMETER", data={"lr": 1e-5})
    L.dllogger.flush()
    lines = open(tmp_path / "squad_log.json").read().strip().splitlines()
    rec = json.loads(lines[0][5:])
    assert rec["step"] == [0, 5] and rec["data"]["step_loss"] == 1.5
    assert format_step((1, 20)) == "Training Epoch: 1 Training Iteration: 20 "


def test_checkpoint_manager(tmp_path):
    d = str(tmp_path / "pretrain_ckpts")
    m = ck.CheckpointManager(d, keep=3)
    for s in (200, 400, 600, 800):
        m.save(s, {"x": s})
    assert [s for s, _ in ck.list_checkpoints(d)] == [400, 600, 800]
    open(os.path.join(d, "notes.txt"), "w").close()
    payload, step = ck.load_latest(d)
    assert step == 800 and payload["x"] == 800
    assert ck.load_latest(str(tmp_path / "none")) == (None, 0)
    c = {"optimizer": {"state": {0: {"exp_avg": 1}}, "param_groups": [{"lr": 9.0, "step": 7038, "initial_lr": 9.0}]}}
    ck.override_optimizer_hparams(c, global_steps=0, max_steps=1563, warmup=0.128, lr=4e-3)
    g = c["optimizer"]["param_groups"][0]
    assert g == {"lr": 4e-3, "step": 0, "t_total": 1563, "warmup": 0.128} and c["optimizer"]["state"][0]["step"] == 0


def test_dist_helpers_without_init():
    assert get_rank() == 0 and get_world_size() == 1 and is_main_process()


def test_file_utils(tmp_path):
    f = tmp_path / "a.bin"; f.write_bytes(b"x")
    assert cached_path(str(f)) == str(f)
    with pytest.raises(FileNotFoundError):
        cached_path(str(tmp_path / "missing"))
    assert url_to_filename("http://a", "e") != url_to_filename("http://a")


def test_tokenizers(tmp_path):
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "un", "##aff", "##able", "hello", ",", "world", "the", "##s"]
    vf = tmp_path / "vocab.txt"; vf.write_text("\n".join(vocab) + "\n")
    tok = T.BertTokenizer(str(vf))
    assert tok.tokenize("Hello, UNAFFABLE worlds!") == ["hello", ",", "un", "##aff", "##able", "world", "##s", "[UNK]"]
    assert tok.convert_tokens_to_ids(["[CLS]", "hello", "[SEP]"]) == [2, 8, 3]
    assert tok.convert_ids_to_tokens([4]) == ["[MASK]"]
    b = T.BasicTokenizer(do_lower_case=True)
    assert b.tokenize("Héllo  [MASK] 中文") == ["hello", "[MASK]", "中", "文"]
    assert T.BasicTokenizer(do_lower_case=False).tokenize("A.b") == ["A", ".", "b"]
    hf = T.get_wordpiece_tokenizer(str(vf))
    assert hf.token_to_id("[MASK]") == 4
    assert hf.encode("hello world").tokens == ["[CLS]", "hello", "world", "[SEP]"]


def test_downloaders_with_local_urls(tmp_path, monkeypatch, capsys):
    """utils/download.py back end against file:// URLs: SQuAD files land under v1.1 / v2.0, the weights archive is
    extracted and its files are checked against the recorded SHA-256 digests (a doctored archive is reported)."""
    import zipfile
    from bert_pytorch_b200.data import corpus
    src = tmp_path / "src"; src.mkdir()
    (src / "train.json").write_text('{"data": []}')
    monkeypatch.setattr(corpus, "SQUAD_URLS", {(src / "train.json").as_uri(): "v1.1/train-v1.1.json"})
    corpus.download("squad", str(tmp_path / "dl"))
    assert (tmp_path / "dl" / "squad" / "v1.1" / "train-v1.1.json").read_text() == '{"data": []}'
    corpus.download("squad", str(tmp_path / "dl"))                    # second call: already there
    assert "already exists" in capsys.readouterr().out

    zpath = src / "uncased_L-24_H-1024_A-16.zip"
    with zipfile.ZipFile(zpath, "w") as z:
        z.writestr("uncased_L-24_H-1024_A-16/vocab.txt", "[PAD]\n")
        z.writestr("uncased_L-24_H-1024_A-16/bert_config.json", "{}")
    monkeypatch.setattr(corpus, "WEIGHT_URLS", {"bert_large_uncased": zpath.as_uri()})
    corpus.download("weights", str(tmp_path / "dl"))
    out = capsys.readouterr().out
    assert "SHA256sum does not match on file: vocab.txt" in out and "bert_model.ckpt.index" in out
    assert (tmp_path / "dl" / "weights" / "uncased_L-24_H-1024_A-16" / "vocab.txt").is_file()
    assert set(corpus.WEIGHT_SHA256) == set(corpus.WEIGHT_URLS) | {"bert_base_uncased", "bert_base_cased", "bert_large_cased"}
    with pytest.raises(ValueError):
        corpus.download("imagenet", str(tmp_path / "dl"))



def test_host_keep_bits_pack_the_keep_mask_little_endian():
    """utils/philox.keep_bits is the host twin of dropout_mask_kernel: bit t of byte j = element 8 j + t."""
    import numpy as np
    from bert_pytorch_b200.utils import philox
    rows, cols, p = 5, 64, 0.1
    keep = philox.keep_mask(1234, 19, rows * cols, p).reshape(rows, cols)
    bits = philox.keep_bits(1234, 19, rows, cols, p)
    assert bits.shape == (rows, cols // 8) and bits.dtype == np.uint8
    for r in range(rows):
        for c in range(cols):
            assert bool((bits[r, c // 8] >> (c % 8)) & 1) == bool(keep[r, c])
    assert philox.keep_bits(1, 2, 3, 16, 0.0).min() == 255          # p = 0 keeps everything
    frac = 1.0 - philox.keep_mask(7, 3, 1 << 16, 0.1).mean()
    assert abs(frac - 0.1) < 0.01
