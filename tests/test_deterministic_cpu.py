"""Deterministic mode, the switches (no GPU needed): ``ops.api.deterministic()`` under the environment variable and
under torch's flag, ``--deterministic`` and the JSON key on the three runners, the mode's place in the CUDA-graph
key of ``FusedPretrainer``, and the [CLS] row indices that captured graphs keep reading."""
import json
import os

import pytest
import torch


@pytest.fixture
def torch_flag():
    prev = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(prev)


def test_predicate_follows_the_environment_and_torch(monkeypatch, torch_flag):
    from bert_pytorch_b200.ops import api as K
    monkeypatch.delenv("B200_DETERMINISTIC", raising=False)
    torch.use_deterministic_algorithms(False)
    assert not K.deterministic()
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    assert not K.deterministic()
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    assert K.deterministic()
    monkeypatch.delenv("B200_DETERMINISTIC")
    torch.use_deterministic_algorithms(True)
    assert K.deterministic()


def test_use_deterministic_sets_torch_and_cublas(monkeypatch, torch_flag):
    from bert_pytorch_b200 import ops
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    torch.use_deterministic_algorithms(False)
    fill = torch.utils.deterministic.fill_uninitialized_memory
    try:
        ops.use_deterministic()
        assert torch.are_deterministic_algorithms_enabled() and ops.deterministic()
        assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":4096:8"
        assert torch.utils.deterministic.fill_uninitialized_memory is False
        monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":16:8")       # a user's own setting stays
        ops.use_deterministic()
        assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":16:8"
    finally:
        torch.utils.deterministic.fill_uninitialized_memory = fill


def _help(parser, flag):
    return next(a.help for a in parser._actions if flag in a.option_strings)


def test_pretraining_flag_and_json_key(tmp_path):
    from bert_pytorch_b200 import pretrain
    base = ["--input_dir", "x", "--output_dir", "y", "--model_config_file", "z"]
    assert pretrain.parse_arguments(base).deterministic is False
    assert pretrain.parse_arguments(base + ["--deterministic"]).deterministic is True
    cfg = tmp_path / "c.json"
    cfg.write_text(json.dumps({"deterministic": True}))
    assert pretrain.parse_arguments(base + ["--config_file", str(cfg)]).deterministic is True
    assert "bitwise" in _help(pretrain.build_parser(), "--deterministic")


def test_pretraining_setup_switches_the_mode_on(monkeypatch, torch_flag):
    from bert_pytorch_b200 import ops, pretrain
    calls = []
    monkeypatch.setattr(ops.api, "use_deterministic", lambda: calls.append(1))

    class Stop(Exception):
        pass
    monkeypatch.setattr(torch.cuda, "is_available", lambda: (_ for _ in ()).throw(Stop()))
    args = pretrain.parse_arguments(["--input_dir", "x", "--output_dir", "y", "--model_config_file", "z",
                                     "--deterministic"])
    with pytest.raises(Stop):
        pretrain.setup_training(args)
    assert calls == [1]


def test_pretraining_refuses_the_peer_memory_backend(monkeypatch, torch_flag):
    """The fused backend pushes weight-gradient tiles to their owner rank with atomics: not one GPU, not fixed order."""
    from bert_pytorch_b200 import ops, pretrain
    monkeypatch.setattr(ops.api, "use_deterministic", lambda: None)
    args = pretrain.parse_arguments(["--input_dir", "x", "--output_dir", "y", "--model_config_file", "z",
                                     "--deterministic", "--backend", "fused"])
    with pytest.raises(ValueError, match="backend fused"):
        pretrain.setup_training(args)


def test_fine_tuning_flags():
    from bert_pytorch_b200 import finetune_ner, finetune_squad
    req = ["--train_file", "t", "--labels", "B", "--model_config_file", "c", "--model_checkpoint", "m"]
    assert finetune_ner.parse_arguments(req + ["--deterministic"]).deterministic is True
    assert finetune_ner.parse_arguments(req).deterministic is False
    p = finetune_squad.build_parser()
    assert "bitwise" in _help(p, "--deterministic")
    assert p.get_default("deterministic") is False


def test_graph_key_holds_the_mode(monkeypatch):
    """The captured program differs between the modes: a switch must capture a new graph, not replay the old one."""
    from bert_pytorch_b200.models import fused

    keys = []

    class Pt(fused.FusedPretrainer):
        def __init__(self):
            pass

        def _bucket(self, *a):
            return None

        def _graph_ok(self):
            return True

    pt = Pt()
    pt.model = type("M", (), {"training": True, "bert": type("B", (), {"encoder": object()})()})()
    pt.engine = type("E", (), {"fp8": False, "wgrad_side": True, "_fp8_calibrated": True})()
    pt.grad_push, pt.graph_warmup = False, 10

    class Graphs(dict):
        def setdefault(self, k, v):
            keys.append(k)
            return super().setdefault(k, v)
    pt._graphs = Graphs()
    monkeypatch.setattr(pt, "_program", lambda *a, **k: None, raising=False)
    t = torch.zeros(2, 8, dtype=torch.int32)
    for flag in ("0", "1"):
        monkeypatch.setenv("B200_DETERMINISTIC", flag)
        pt.forward_backward(t, t, t, t, torch.zeros(2, dtype=torch.int32))
    assert len(keys) == 2 and keys[0] != keys[1]
    assert keys[0][-2] is False and keys[1][-2] is True           # the last entry is the token bucket


def test_cls_rows_stay_one_tensor_per_batch_shape():
    """A captured graph reads the padded [CLS] row indices of its batch shape through a raw pointer: requesting other
    shapes must neither replace nor free that tensor.  A packed batch brings its own indices."""
    from types import SimpleNamespace

    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    from bert_pytorch_b200.models.fused import FusedPretrainer
    cfg = BertConfig(vocab_size_or_config_json_file=64, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                     intermediate_size=128, max_position_embeddings=16)
    pt = FusedPretrainer(BertForPreTraining(cfg))
    cpu = torch.device("cpu")
    first = pt._cls_rows(None, 4, 16, cpu)
    assert first.dtype == torch.int32 and first.tolist() == [0, 16, 32, 48]
    for B, S in ((3, 16), (4, 8), (8, 16)):
        assert pt._cls_rows(None, B, S, cpu).tolist() == [b * S for b in range(B)]
    assert pt._cls_rows(None, 4, 16, cpu) is first
    pk = SimpleNamespace(cls_rows=torch.tensor([0, 5, 9], dtype=torch.int32))
    assert pt._cls_rows(pk, 3, 16, cpu) is pk.cls_rows
