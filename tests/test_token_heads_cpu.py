"""SQuAD and NER ``train_step`` / ``predict`` where the fused program cannot run (CPU): the loss semantics (clamp and
ignore, all ignored gives 0), gradients equal to ``forward`` + the loss, the inert-row fill of a short batch, and the
runners keeping the module path on the CPU."""
import argparse

import pytest
import torch
import torch.nn.functional as F

from bert_pytorch_b200 import BertConfig
from bert_pytorch_b200.models import BertForQuestionAnswering, BertForTokenClassification
from bert_pytorch_b200.models.modeling import span_loss, token_loss


def _cfg():
    return BertConfig(vocab_size_or_config_json_file=64, hidden_size=32, num_hidden_layers=1, num_attention_heads=2,
                      intermediate_size=64, max_position_embeddings=32, hidden_dropout_prob=0.0,
                      attention_probs_dropout_prob=0.0)


def _batch(B=4, S=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 64, (B, S), generator=g)
    mask = torch.ones(B, S, dtype=torch.long)
    mask[1, 10:] = 0
    mask[2, 3] = 0                                              # a hole
    seg = torch.zeros_like(ids)
    return ids, seg, mask


def _grads(m):
    return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def test_span_loss_clamps_ignores_and_is_zero_when_everything_is_ignored():
    g = torch.Generator().manual_seed(1)
    s, e = torch.randn(4, 16, generator=g), torch.randn(4, 16, generator=g)
    sp, ep = torch.tensor([-3, 5, 16, 40]), torch.tensor([2, 16, 16, 7])
    ce = lambda lg, y: F.cross_entropy(lg, y)                   # noqa: E731
    want = (ce(s[[0, 1]], torch.tensor([0, 5])) + ce(e[[0, 3]], torch.tensor([2, 7]))) / 2
    assert torch.allclose(span_loss(s, e, sp, ep), want)
    s.requires_grad_(True)
    loss = span_loss(s, e, torch.full((4,), 16), torch.full((4,), 99))
    loss.backward()
    assert loss.item() == 0.0 and (s.grad == 0).all()


def test_token_loss_counts_mask_one_and_labels_in_range():
    g = torch.Generator().manual_seed(2)
    logits = torch.randn(2, 6, 5, generator=g)
    labels = torch.tensor([[0, -100, 4, 5, -1, 2], [1, 1, 3, 0, 2, 4]])
    mask = torch.tensor([[1, 1, 1, 1, 1, 1], [1, 1, 0, 0, 2, 1]])
    keep = torch.tensor([True, False, True, False, False, True, True, True, False, False, False, True])
    want = F.cross_entropy(logits.view(-1, 5)[keep], labels.view(-1)[keep])
    assert torch.allclose(token_loss(logits, labels, mask), want)
    logits.requires_grad_(True)
    loss = token_loss(logits, torch.full_like(labels, -100), mask)
    loss.backward()
    assert loss.item() == 0.0 and (logits.grad == 0).all()


def test_qa_train_step_and_predict_fall_back_on_cpu():
    torch.manual_seed(0)
    m = BertForQuestionAnswering(_cfg())
    ids, seg, mask = _batch()
    sp, ep = torch.tensor([3, -1, 16, 20]), torch.tensor([5, 2, 16, 8])
    m.train()
    loss = m.train_step(ids, seg, mask, sp, ep, grad_scale=0.5)
    got = _grads(m)
    m.zero_grad()
    s, e = m(ids, seg, mask)
    want = span_loss(s, e, sp, ep)
    (want * 0.5).backward()
    assert torch.allclose(loss, want.detach())
    for n, g in _grads(m).items():
        assert torch.allclose(got[n], g, atol=1e-7), n
    m.zero_grad()
    assert m.train_step(ids, seg, mask, torch.full((4,), 16), torch.full((4,), 16)).item() == 0.0
    assert all((p.grad is None) or (p.grad == 0).all() for p in m.parameters())
    ps, pe = m.predict(ids, seg, mask)
    assert m.training and ps.dtype == torch.float32 and ps.shape == (4, 16) and pe.shape == (4, 16)


def test_token_train_step_and_predict_fall_back_on_cpu():
    torch.manual_seed(0)
    m = BertForTokenClassification(_cfg(), num_labels=5)
    ids, seg, mask = _batch()
    labels = torch.randint(0, 5, ids.shape)
    labels[:, 0] = -100
    labels[3, 4] = -1
    labels[0, 7] = 9
    m.train()
    loss = m.train_step(ids, seg, mask, labels)
    got = _grads(m)
    m.zero_grad()
    want = token_loss(m(ids, seg, mask), labels, mask)
    want.backward()
    assert torch.allclose(loss, want.detach())
    for n, g in _grads(m).items():
        assert torch.allclose(got[n], g, atol=1e-7), n
    m.zero_grad()
    assert m.train_step(ids, seg, mask, torch.full_like(labels, -100)).item() == 0.0
    m.eval()
    lg = m.predict(ids, seg, mask)
    assert not m.training and lg.shape == (4, 16, 5) and lg.dtype == torch.float32


def test_short_batches_are_filled_with_inert_rows():
    from bert_pytorch_b200 import finetune_ner, finetune_squad
    ids, seg, mask = _batch(B=3)
    sp, ep = torch.tensor([1, 2, 3]), torch.tensor([4, 5, 6])
    f = finetune_squad.fill_batch((ids, mask, seg, sp, ep), 8, 16)
    assert [t.size(0) for t in f] == [8] * 5
    assert (f[3][3:] == 16).all() and (f[4][3:] == 16).all()       # S: ignored after the clamp (-1 would be target 0)
    assert (f[1][3:, 0] == 1).all() and (f[1][3:, 1:] == 0).all() and (f[0][3:] == 0).all()
    torch.manual_seed(0)
    m = BertForQuestionAnswering(_cfg())
    m.train()
    real = m.train_step(ids, seg, mask, sp, ep)
    full = m.train_step(f[0], f[2], f[1], f[3], f[4])
    assert torch.allclose(real, full, rtol=1e-6)
    p = finetune_squad.fill_batch((ids, mask, seg), 8, 16)
    assert [t.size(0) for t in p] == [8] * 3

    labels = torch.randint(0, 5, ids.shape)
    s2, l2, m2 = finetune_ner.fill_batch(ids, labels, mask, 8)
    assert s2.shape == l2.shape == m2.shape == (8, 16)
    assert (l2[3:] == -100).all() and (m2[3:, 0] == 1).all() and (m2[3:, 1:] == 0).all()
    tm = BertForTokenClassification(_cfg(), num_labels=5)
    tm.train()
    assert torch.allclose(tm.train_step(ids, seg, mask, labels), tm.train_step(s2, torch.zeros_like(s2), m2, l2),
                          rtol=1e-6)


def test_runners_keep_the_module_path_on_cpu():
    from bert_pytorch_b200 import finetune_ner, finetune_squad
    m = BertForQuestionAnswering(_cfg())
    assert not finetune_squad.fused_program(m, 16, torch.device("cpu"), torch.bfloat16)
    assert not finetune_squad.fused_program(m, 16, torch.device("cpu"), torch.float32)
    tm = BertForTokenClassification(_cfg(), num_labels=5)
    assert not finetune_ner.fused_program(tm, argparse.Namespace(cuda=False, bf16=True, max_seq_len=16))


def test_token_engine_refuses_more_than_64_labels():
    assert BertForTokenClassification(_cfg(), num_labels=65).token_engine() is None
