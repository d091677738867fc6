"""GLUE fine-tuning on the H100: the ``cls_head`` kernel against an fp64 reference fed the kernel's own dropout keep bits,
the fused classification program (``FusedClassifier``) against the plain PyTorch module, padded against unpadded,
across token buckets and under CUDA-graph replay, the inert rows of a short batch, the training state an evaluation must
leave alone, and ``run_glue.py --bf16`` reproducible under ``--deterministic`` and learning a synthetic task."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_glue_cpu import VOCAB, _config_file, write_synthetic_sst2

pytestmark = pytest.mark.gpu

V = 512


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernel against fp64
# ---------------------------------------------------------------------------------------------------------------------
def _head_case(B, H, C, seed):
    g = torch.Generator().manual_seed(seed)
    pooled = torch.tanh(torch.randn(B, H, generator=g) * 1.5).to(torch.bfloat16)
    w = (torch.randn(C, H, generator=g) * 0.1).to(torch.bfloat16)
    bias = torch.randn(C, generator=g) * 0.1
    y = torch.randint(0, C, (B,), generator=g)
    y[::5] = -1                                                    # ignored rows
    return pooled, w, bias, y


def _ref_head(pooled, w, bias, y, keep, scale, grad_scale):
    """fp64: loss, dW, db, dz of cross-entropy(classifier(dropout(pooled))) averaged over the valid rows."""
    x = pooled.double()
    xd = (x * keep.double() * scale).requires_grad_(True)
    wd = w.double().requires_grad_(True)
    bd = bias.double().requires_grad_(True)
    logits = xd @ wd.t() + bd
    valid = y >= 0
    if valid.any():
        loss = F.cross_entropy(logits[valid], y[valid], reduction="mean")
    else:
        loss = (logits * 0).sum()
    (loss * grad_scale).backward()
    dz = xd.grad * keep.double() * scale * (1 - x * x)
    return loss.item(), wd.grad, bd.grad, dz


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("C", [2, 3])
def test_cls_head_matches_fp64(C, p, det, monkeypatch):
    from bert_pytorch_b200.ops import api as K
    from bert_pytorch_b200.utils import philox
    monkeypatch.setenv("B200_DETERMINISTIC", "1" if det else "0")
    B, H, seed, stream, gs = 37, 1024, 12345, 8188, 0.5
    for case, all_ignored in ((0, False), (1, True)):
        pooled, w, bias, y = _head_case(B, H, C, seed=C * 10 + case)
        if all_ignored:
            y[:] = -1
        bits = philox.keep_bits(seed, stream, B, H, p)
        keep = torch.from_numpy(np.unpackbits(bits, axis=1, bitorder="little").astype(np.float32))
        loss_ref, dw_ref, db_ref, dz_ref = _ref_head(pooled, w, bias, y, keep, philox.keep_scale(p), gs)
        loss = torch.zeros(1, device="cuda")
        dw = torch.full((C, H), 0.25, device="cuda")                   # the kernel accumulates
        db = torch.full((C,), 0.25, device="cuda")
        dz = K.cls_head_(pooled.cuda(), w.cuda(), bias.cuda(), y.cuda(), gs, loss, dw, db, p_drop=p, seed=seed,
                         stream=stream)
        torch.cuda.synchronize()
        assert torch.isfinite(dz).all() and torch.isfinite(loss).all()
        assert abs(loss.item() - loss_ref) <= 1e-5 * max(1.0, abs(loss_ref)), (loss.item(), loss_ref)
        assert (dw.cpu().double() - 0.25 - dw_ref).abs().max().item() <= 1e-5
        assert (db.cpu().double() - 0.25 - db_ref).abs().max().item() <= 1e-6
        err = (dz.cpu().double() - dz_ref).abs()
        assert (err <= 1e-2 * dz_ref.abs() + 1e-7).all(), err.max().item()     # bf16 rounding of dz
        if all_ignored:
            assert loss.item() == 0.0 and (dz == 0).all() and (dw == 0.25).all() and (db == 0.25).all()
        if det:                                                        # fixed order: the same bits again
            loss2, dw2, db2 = torch.zeros(1, device="cuda"), torch.full_like(dw, 0.25), torch.full_like(db, 0.25)
            dz2 = K.cls_head_(pooled.cuda(), w.cuda(), bias.cuda(), y.cuda(), gs, loss2, dw2, db2, p_drop=p, seed=seed,
                              stream=stream)
            assert torch.equal(loss, loss2) and torch.equal(dw, dw2) and torch.equal(db, db2) and torch.equal(dz, dz2)


def test_cls_logits_and_class_count_refusal():
    from bert_pytorch_b200.ops import api as K
    pooled, w, bias, _ = _head_case(9, 256, 3, seed=1)
    lg = K.cls_logits(pooled.cuda(), w.cuda(), bias.cuda()).cpu().double()
    ref = pooled.double() @ w.double().t() + bias.double()
    assert lg.shape == (9, 3) and (lg - ref).abs().max().item() <= 1e-5
    with pytest.raises(ValueError, match="classes"):
        K.cls_logits(pooled.cuda(), torch.zeros(4, 256, dtype=torch.bfloat16, device="cuda"), torch.zeros(4).cuda())


# ---------------------------------------------------------------------------------------------------------------------
# 2.-5. the fused program
# ---------------------------------------------------------------------------------------------------------------------
def _model(C=2, p_drop=0.0, seed=0, layers=2):
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForSequenceClassification
    torch.manual_seed(seed)
    cfg = BertConfig(vocab_size_or_config_json_file=V, hidden_size=256, num_hidden_layers=layers, num_attention_heads=4,
                     intermediate_size=1024, max_position_embeddings=128, hidden_dropout_prob=p_drop,
                     attention_probs_dropout_prob=p_drop)
    m = BertForSequenceClassification(cfg, C)
    with torch.no_grad():
        for n, prm in m.named_parameters():
            if "LayerNorm.weight" in n:
                prm.uniform_(0.5, 1.5)
            elif "bias" in n:
                prm.normal_(0, 0.1)
            elif "classifier.weight" in n:
                prm.normal_(0, 0.2)
            prm.copy_(prm.to(torch.bfloat16).float())                  # weights the bf16 program holds exactly
    return m


def _fused(m):
    from bert_pytorch_b200.models.arena import ParamArena
    m = m.cuda()
    arena = ParamArena(m)
    m.train()
    return m, arena


def _batch(B, S, C, seed=0, pair=True):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(8, S // 2, (B,), generator=g)
    lens[0] = S
    ids = torch.randint(5, V, (B, S), generator=g)
    ids[:, 0] = 2
    pos = torch.arange(S)[None]
    mask = (pos < lens[:, None]).long()
    seg = ((pos >= lens[:, None] // 2) & (mask > 0)).long() if pair else torch.zeros_like(ids)
    ids = ids * mask
    y = torch.randint(0, C, (B,), generator=g)
    return [t.cuda() for t in (ids, seg, mask, y)], int(mask.sum())


def _grad_errors(got, ref):
    bad = []
    for n, r in ref.items():
        if n.endswith("attention.self.key.bias"):                    # zero in exact arithmetic: rounding noise
            continue
        gt = got[n].double()
        r = r.double()
        cos = F.cosine_similarity(gt.flatten(), r.flatten(), dim=0).item()
        rel = ((gt - r).norm() / r.norm().clamp_min(1e-12)).item()
        if not (cos >= 0.9995 and rel <= 1e-2):
            bad.append((n, round(cos, 6), round(rel, 5)))
    return bad


@pytest.mark.parametrize("unpad", [False, True])
@pytest.mark.parametrize("C", [2, 3])
def test_fused_step_matches_the_module_path(C, unpad):
    ref = _model(C).cuda()
    ref.bert.use_fused = False
    m, arena = _fused(_model(C))
    m.bert.unpad = unpad
    (ids, seg, mask, y), tok = _batch(16, 128, C)
    y[3] = -1
    ref.train()
    logits = ref(ids, seg, mask)
    loss_ref = F.cross_entropy(logits.float(), y, ignore_index=-1)
    loss_ref.backward()
    arena.zero_grad()
    loss = m.train_step(ids, seg, mask, y, tokens=tok)
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) <= 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    got = {s.name: arena.grad(s.name).float().clone() for s in arena.slots}
    want = {n: p.grad for n, p in ref.named_parameters()}
    assert not _grad_errors(got, want), _grad_errors(got, want)


def test_logits_padded_unpadded_across_buckets_and_replayed_are_bitwise_equal():
    m, arena = _fused(_model(3))
    eng = m.classifier_engine()
    assert eng.use_graphs
    (ids, seg, mask, _), tok = _batch(32, 128, 3, seed=4)
    padded = [m.predict(ids, seg, mask) for _ in range(eng.graph_warmup + 2)]   # eager, eager, capture, replay
    m.bert.unpad = True
    unpadded = [m.predict(ids, seg, mask, tokens=tok) for _ in range(eng.graph_warmup + 2)]
    wide = m.predict(ids, seg, mask, tokens=32 * 128)                          # the largest bucket
    for t in padded + unpadded + [wide]:
        assert t.dtype == torch.float32 and torch.equal(t, padded[0])
    assert sum(k[0] == "cls-eval" and "graph" in e for k, e in eng._graphs.items()) == 2


def test_train_replay_equals_eager_and_draws_new_masks(monkeypatch):
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    m, arena = _fused(_model(2, p_drop=0.1))
    m.bert.unpad = True
    eng = m.classifier_engine()
    (ids, seg, mask, y), tok = _batch(32, 128, 2, seed=5)
    for _ in range(eng.graph_warmup):
        m.train_step(ids, seg, mask, y, tokens=tok)
    arena.zero_grad()
    loss_r = m.train_step(ids, seg, mask, y, tokens=tok).clone()                 # capture + first replay
    g_r = arena.flat_grad.clone()
    arena.zero_grad()
    loss_e = eng._program(ids, seg, mask, y, 1.0, seed=eng.engine._seed_base, bucket=eng._bucket(mask, tok))
    assert torch.equal(loss_r, loss_e) and torch.equal(g_r, arena.flat_grad)
    loss_2 = m.train_step(ids, seg, mask, y, tokens=tok).clone()                 # the next replay: new masks
    assert loss_2.item() != loss_r.item()


def test_short_batch_filled_with_inert_rows():
    from bert_pytorch_b200.data.glue import fill_batch
    ref = _model(2).cuda()
    ref.bert.use_fused = False
    m, arena = _fused(_model(2))
    (ids, seg, mask, y), _ = _batch(32, 128, 2, seed=6)
    n = 11
    real = [t[:n] for t in (ids, seg, mask, y)]
    full = fill_batch(*real, 32)
    ref.train()
    loss_ref = F.cross_entropy(ref(*real[:3]).float(), real[3])
    for unpad in (False, True):
        m.bert.unpad = unpad
        arena.zero_grad()
        loss = m.train_step(*full, tokens=int(full[2].sum()))
        assert abs(loss.item() - loss_ref.item()) <= 1e-2 * loss_ref.item(), (unpad, loss.item(), loss_ref.item())
        logits = m.predict(*full[:3], tokens=int(full[2].sum()))
        assert torch.equal(logits[:n], m.predict(*[t[:n] for t in full[:3]], tokens=int(real[2].sum())))


def test_evaluation_leaves_the_training_state_alone():
    from bert_pytorch_b200.optim import Adam
    m, arena = _fused(_model(2, p_drop=0.1))
    opt = Adam([{"params": list(m.parameters()), "weight_decay": 0.01}], lr=1e-4, bias_correction=False)
    arena.bind_optimizer(opt)
    eng = m.classifier_engine()
    (ids, seg, mask, y), tok = _batch(32, 128, 2, seed=7)
    for _ in range(eng.graph_warmup + 1):                                         # training graph captured
        m.train_step(ids, seg, mask, y, tokens=tok)
        opt.step()
    m.train_step(ids, seg, mask, y, tokens=tok)
    torch.cuda.synchronize()
    state = lambda: [t.clone() for t in (arena.flat_param, arena.flat_grad, arena.flat_shadow, arena.exp_avg,  # noqa
                                         arena.exp_avg_sq, eng._seed_step)] + [eng.engine._calls]
    before = state()
    for unpad in (False, True):
        m.bert.unpad = unpad
        for _ in range(eng.graph_warmup + 2):
            m.predict(ids, seg, mask, tokens=tok)
    torch.cuda.synchronize()
    after = state()
    assert m.training
    for a, b in zip(before[:-1], after[:-1]):
        assert torch.equal(a, b)
    assert before[-1] == after[-1]


# ---------------------------------------------------------------------------------------------------------------------
# 6.-7. run_glue.py --bf16
# ---------------------------------------------------------------------------------------------------------------------
def _run(tmp_path, tag, data, cj, *extra):
    from bert_pytorch_b200 import finetune_glue
    out = tmp_path / tag
    finetune_glue.main(["--task_name", "SST-2", "--data_dir", str(data), "--config_file", str(cj), "--output_dir",
                        str(out), "--do_train", "--do_eval", "--do_lower_case", "--max_seq_length", "64",
                        "--train_batch_size", "32", "--bf16", "--log_freq", "1", *extra])
    return out


def _files(tmp_path):
    vf = tmp_path / "vocab.txt"
    vf.write_text("\n".join(VOCAB) + "\n")
    data = tmp_path / "SST-2"
    write_synthetic_sst2(str(data), 512, 256, 8, max_words=40)
    cj = _config_file(tmp_path, vf, hidden_size=256, num_attention_heads=4, num_hidden_layers=2,
                      intermediate_size=1024, max_position_embeddings=64, hidden_dropout_prob=0.1,
                      attention_probs_dropout_prob=0.1)
    return data, cj


def test_run_glue_deterministic_twice_gives_the_same_bits(tmp_path):
    from bert_pytorch_b200 import ops
    data, cj = _files(tmp_path)
    outs = []
    try:
        for i in range(2):
            ops.extension().set_seed_step(None)      # a graph of the previous run left its step counter set
            outs.append(_run(tmp_path, f"d{i}", data, cj, "--deterministic", "--unpad", "--num_train_epochs", "1",
                             "--learning_rate", "1e-4"))
    finally:
        torch.use_deterministic_algorithms(False)

    def losses(o):
        return [ln for ln in open(o / "glue_log.json") if "step_loss" in ln]
    a, b = (torch.load(o / "pytorch_model.bin", weights_only=False)["model"] for o in outs)
    assert all(torch.equal(a[k], b[k]) for k in a)
    strip = lambda lines: [json.loads(ln.split("DLLL", 1)[-1].strip())["data"] for ln in lines]   # noqa: E731
    assert strip(losses(outs[0])) == strip(losses(outs[1])) and len(losses(outs[0])) == 16
    assert open(outs[0] / "eval_results.json").read() == open(outs[1] / "eval_results.json").read()


@pytest.mark.parametrize("unpad", [False, True])
def test_run_glue_learns_a_synthetic_task(tmp_path, unpad):
    data, cj = _files(tmp_path)
    out = _run(tmp_path, "o", data, cj, "--num_train_epochs", "4", "--learning_rate", "1e-4",
               *(["--unpad"] if unpad else []))
    res = json.load(open(out / "eval_results.json"))["SST-2"]
    assert res["eval_samples"] == 256 and res["acc"] >= 0.95, res
