"""Model variants next to the flagship config: the no-NSP (RoBERTa-style) model on the fused engine
and configurations the kernel program does not implement, which must fall back to the plain
PyTorch path instead of raising."""
import copy
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("vocab", [1000, 1024])
def test_fused_pretrainer_without_next_sentence_task(vocab):
    """RoBERTa-style model (config/roberta_large_cased_config.json: ``next_sentence: false`` -> no token-type
    embeddings, no pooler, no NSP head; vocabulary with a tail tile): loss and gradients vs fp32 autograd."""
    from test_gpu_kernels import _batch, _tiny_model
    from bert_pytorch_b200.models import BertPretrainingCriterion
    from bert_pytorch_b200.models.arena import ParamArena
    model = _tiny_model(vocab=vocab, nsp=False).cuda()
    assert not any("token_type" in n or "pooler" in n or "seq_relationship" in n for n, _ in model.named_parameters())
    arena = ParamArena(model)
    ids, seg, mask, labels, nsl = _batch(V=vocab)
    oracle = copy.deepcopy(model)
    for p in oracle.parameters():
        p.data = p.data.to(torch.bfloat16).float()
    oracle.bert.use_fused = False
    crit = BertPretrainingCriterion(model.config.vocab_size)
    scores, nsp = oracle(ids, seg, mask)
    assert nsp is None
    ref_loss = crit(scores, labels, nsp, nsl)
    ref_loss.backward()
    eng = model.pretrain_engine()
    for it in range(4):                                   # eager calls, then the captured graph
        arena.zero_grad()
        loss = eng.forward_backward(ids, seg, mask, labels, nsl, grad_scale=1.0)
        assert abs(loss.item() - ref_loss.item()) < 3e-2 * abs(ref_loss.item()), (it, loss.item(), ref_loss.item())
        gmax = max(po.grad.abs().max().item() for po in oracle.parameters())
        bad = []
        for (n, p), po in zip(model.named_parameters(), oracle.parameters()):
            denom = max(po.grad.abs().max().item(), 1e-3 * gmax)
            rel = (p.grad.float() - po.grad.float()).abs().max().item() / denom
            if rel > 8e-2:
                bad.append((n, rel))
        assert not bad, (it, bad[:8])



@pytest.mark.parametrize("act,H,heads", [("relu", 128, 2), ("swish", 128, 2), ("gelu", 128, 4)])
def test_non_fusable_configs_train_on_the_oracle_path(act, H, heads):
    """relu / swish FFN or head_dim != 64 (reference: any ACT2FN entry, any head size -- src/modeling.py:118-139): on a
    CUDA box with the extension loaded these used to raise NotImplementedError from the engine constructor; now
    ``BertModel.fusable_config()`` routes them to the autograd path and they train."""
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining, BertPretrainingCriterion
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=512, hidden_size=H, num_hidden_layers=2, num_attention_heads=heads,
                     intermediate_size=4 * H, max_position_embeddings=64, hidden_act=act)
    model = BertForPreTraining(cfg).cuda()
    assert not model.bert.fusable_config() and model.pretrain_engine() is None
    crit = BertPretrainingCriterion(cfg.vocab_size)
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    ids = torch.randint(5, 512, (4, 32), device="cuda")
    labels = torch.full_like(ids, -1)
    labels[:, 3:9] = ids[:, 3:9]
    nsl = torch.randint(0, 2, (4,), device="cuda")
    losses = []
    for _ in range(5):
        scores, nsp = model(ids, torch.zeros_like(ids), torch.ones_like(ids))
        loss = crit(scores, labels, nsp, nsl)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses
