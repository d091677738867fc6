"""Held-out evaluation on the H100: the ``mlm_eval`` / ``nsp_eval`` kernels against an fp64 reference of their own bf16
inputs, ``FusedPretrainer.evaluate`` against the training loss, the plain PyTorch model, the unpadded program, its own
CUDA-graph replay and the deterministic mode, the training state it must leave untouched, and the runtime flags.

Every sum of the evaluation is taken in a fixed order (``ordered_sum``, no atomics), so repeated and replayed
evaluations are compared bitwise."""
import csv
import json
import os

import numpy as np
import pytest
import torch

from test_gpu_pretrain_unpad import MP, V, _batch, _model, _tokens

pytestmark = pytest.mark.gpu


def _bf16(x):
    return x.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the metric kernels against fp64
# ---------------------------------------------------------------------------------------------------------------------
def _mlm_case(Vc, seed=0):
    """Rows: random, large-magnitude, planted ties below / at / above the target, all-equal, ignored."""
    g = torch.Generator().manual_seed(seed)
    R = 40
    x = torch.randn(R, Vc, generator=g) * 3.0
    x[5:10] *= 30.0                                                # large magnitudes (|x| up to ~450)
    t = torch.randint(0, Vc, (R,), generator=g)
    t[10:13] = Vc // 2
    # planted maxima: around the target (not correct), at the target with a lower duplicate (not correct), at the
    # target as the lowest of the duplicates (correct)
    for r, dup in ((10, [3, Vc // 2 + 5]), (11, [3, Vc // 2]), (12, [Vc // 2, Vc - 2])):
        x[r, dup] = 50.0
    x[13] = 0.25                                                   # all equal: argmax 0
    t[13] = 0
    x[14] = -7.0
    t[14] = 3
    t[15:20] = -1                                                  # ignored
    t[20] = Vc - 1                                                 # target at the last column
    x[20, Vc - 1] = x[20].max() + 1
    return _bf16(x).cuda(), t.to(torch.int32).cuda()


def _ref_rows(x64, t):
    out = np.zeros((x64.shape[0], 3))
    for r in range(x64.shape[0]):
        if t[r] < 0:
            continue
        m = x64[r].max()
        out[r] = (m + np.log(np.exp(x64[r] - m).sum()) - x64[r, t[r]], float(np.argmax(x64[r]) == t[r]), 1.0)
    return out


@pytest.mark.parametrize("Vc", [1000, 2048, 30528])
def test_mlm_eval_matches_fp64(Vc):
    from bert_pytorch_b200.ops import api as K
    x, t = _mlm_case(Vc)
    acc = torch.zeros(3, dtype=torch.float64, device="cuda")
    rows = K.mlm_eval(x, t, acc).cpu().numpy()
    ref = _ref_rows(x.float().double().cpu().numpy(), t.cpu().numpy())
    assert np.array_equal(rows[:, 1:], ref[:, 1:]), np.nonzero(rows[:, 1] != ref[:, 1])
    # __expf is within 2 ulp (+ a term in |x|) of expf: relative 1e-6 per term on the arguments <= 0 it gets here,
    # so the log of the sum moves by ~1e-6; the rest is fp32 rounding of lse at |lse| <= 512 (half an ulp: 3e-5)
    err = np.abs(rows[:, 0] - ref[:, 0])
    assert err.max() <= 1e-4, (err.argmax(), err.max())
    assert rows[10, 1] == 0 and rows[11, 1] == 0 and rows[12, 1] == 1 and rows[13, 1] == 1
    a = acc.cpu().numpy()
    assert a[1] == ref[:, 1].sum() and a[2] == ref[:, 2].sum() == 35
    assert abs(a[0] - ref[:, 0].sum()) <= 1e-5 * ref[:, 0].sum()
    # the logits are only read, and a second call gives the same bits
    x0 = x.clone()
    assert torch.equal(K.mlm_eval(x, t).cpu(), torch.from_numpy(rows)) and torch.equal(x, x0)


def test_mlm_eval_on_a_strided_view():
    from bert_pytorch_b200.ops import api as K
    x, t = _mlm_case(1024, seed=3)
    wide = torch.zeros(x.size(0), 1024 + 64, dtype=torch.bfloat16, device="cuda")
    wide[:, :1024] = x
    assert torch.equal(K.mlm_eval(wide[:, :1024], t), K.mlm_eval(x, t))


@pytest.mark.parametrize("H", [256, 1024])
def test_nsp_eval_matches_fp64(H):
    from bert_pytorch_b200.ops import api as K
    g = torch.Generator().manual_seed(H)
    B = 70
    pooled = _bf16(torch.tanh(torch.randn(B, H, generator=g))).cuda()
    w = _bf16(torch.randn(2, H, generator=g) * 0.05).cuda()
    bias = torch.tensor([0.1, -0.2]).cuda()
    y = torch.randint(0, 2, (B,), generator=g)
    y[::9] = -1
    pooled[5] = 0                                                  # a tie: l0 == l1 after the bias below
    tie_bias = torch.tensor([0.3, 0.3]).cuda()
    acc = torch.zeros(3, dtype=torch.float64, device="cuda")
    rows = K.nsp_eval(pooled, w, bias, y.cuda(), acc).cpu().numpy()
    lg = pooled.double().cpu().numpy() @ w.double().cpu().numpy().T + bias.double().cpu().numpy()
    yn = y.numpy()
    for b in range(B):
        if yn[b] < 0:
            assert (rows[b] == 0).all()
            continue
        m = lg[b].max()
        lse = m + np.log(np.exp(lg[b] - m).sum())
        assert abs(rows[b, 0] - (lse - lg[b, yn[b]])) <= 1e-5, b
        assert rows[b, 1] == float(int(lg[b, 1] > lg[b, 0]) == yn[b]) and rows[b, 2] == 1.0
    a = acc.cpu().numpy()
    assert a[1] == rows[:, 1].sum() and a[2] == (yn >= 0).sum()
    tie = K.nsp_eval(pooled[5:6].contiguous(), w, tie_bias, torch.tensor([0, 1]).cuda()[:1]).cpu()
    assert tie[0, 1].item() == 1.0                                  # a tie goes to class 0


# ---------------------------------------------------------------------------------------------------------------------
# 2.-6. the evaluation program
# ---------------------------------------------------------------------------------------------------------------------
def _eval(pt, batch, tokens=None):
    acc = torch.zeros(6, dtype=torch.float64, device="cuda")
    pt.evaluate(*batch, acc, tokens=tokens)
    return acc.cpu()


def _loader_batch(B, S, seed=0):
    g = np.random.default_rng(seed)
    lens = g.integers(S // 4, S + 1, B)
    lens[0] = S
    ids, seg, mask, labels, nsl = _batch(B, S, list(lens), seed=seed)
    labels[:, 0] = -1                                              # [CLS] is never masked
    return ids, seg, mask, labels, nsl


def test_eval_losses_equal_the_training_loss():
    model, arena, pt = _model(p_drop=0.0)
    pt.use_graphs = False
    batch = _loader_batch(8, 128)
    a = _eval(pt, batch)
    loss = float(pt.forward_backward(*batch))
    ev = a[0].item() / a[2].item() + a[3].item() / a[5].item()
    assert abs(ev - loss) <= 1e-6 * abs(loss), (ev, loss)


def test_eval_against_plain_pytorch_fp32_on_bf16_weights():
    model, arena, pt = _model(p_drop=0.0, layers=2)
    pt.use_graphs = False
    batch = _loader_batch(16, 128, seed=4)
    a = _eval(pt, batch)
    ref, _, _ = _model(p_drop=0.0, layers=2)                      # the same seed: the same weights
    ref.bert.use_fused = False
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    ref.eval()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            scores, nsp = ref(*(t.long() for t in batch[:3]))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    lab = batch[3].long().view(-1)
    k = lab >= 0
    s = scores.view(-1, V)[k].double()
    t = lab[k]
    loss = torch.nn.functional.cross_entropy(s, t, reduction="sum").item()
    correct = (s.argmax(-1) == t).sum().item()
    top2 = s.topk(2, dim=-1).values
    mx = top2[:, 0].abs()
    res = torch.exp2(torch.floor(torch.log2(mx.clamp(min=1e-30)))) * 2.0 ** -7      # bf16 spacing at the row max
    close = int(((top2[:, 0] - top2[:, 1]) < res).sum())
    assert a[2].item() == k.sum().item()
    assert abs(a[0].item() - loss) <= 1e-2 * abs(loss), (a[0].item(), loss)
    assert abs(a[1].item() - correct) <= close, (a[1].item(), correct, close)
    nl = batch[4].long()
    nloss = torch.nn.functional.cross_entropy(nsp.double(), nl, reduction="sum").item()
    assert abs(a[3].item() - nloss) <= 1e-2 * abs(nloss) and a[5].item() == 16


@pytest.mark.parametrize("S", [128, 512])
@pytest.mark.parametrize("nsp", [True, False])
def test_padded_and_unpadded_sums_are_bitwise_equal(S, nsp):
    model, arena, pt = _model(S=S, nsp=nsp)
    pt.use_graphs = False
    batch = _loader_batch(8 if S == 128 else 4, S, seed=S)
    padded = _eval(pt, batch)
    model.bert.unpad = True
    unpadded = _eval(pt, batch, tokens=_tokens(batch[2]))
    assert torch.equal(padded, unpadded), (padded, unpadded)
    assert (padded[3:] == 0).all() != nsp


@pytest.mark.parametrize("unpad", [False, True])
def test_graph_replay_equals_the_eager_program_in_the_shared_pool(unpad):
    model, arena, pt = _model(p_drop=0.1)
    model.bert.unpad = unpad
    assert pt.use_graphs
    train, ev = _loader_batch(8, 128, seed=1), _loader_batch(8, 128, seed=2)
    tok = _tokens(train[2]) if unpad else None
    for _ in range(3):
        pt.forward_backward(*train, tokens=tok)
    graphs = lambda: [e for e in pt._graphs.values() if "graph" in e]      # noqa: E731
    n_train = len(graphs())
    assert n_train == 1
    etok = _tokens(ev[2]) if unpad else None
    runs = [_eval(pt, ev, etok) for _ in range(pt.graph_warmup + 2)]        # eager, eager, capture + replay, replay
    for r in runs[1:]:
        assert torch.equal(r, runs[0])
    assert len(graphs()) == n_train + 1
    assert len({e["graph"].pool() for e in graphs()}) == 1
    assert any(k[0] == "eval" for k in pt._graphs)
    pt.forward_backward(*train, tokens=tok)                                 # training still replays its graph
    assert len(graphs()) == n_train + 1


def test_two_evaluations_and_the_deterministic_mode_agree(monkeypatch):
    model, arena, pt = _model(p_drop=0.1)
    pt.use_graphs = False
    batch = _loader_batch(8, 128, seed=7)
    a, b = _eval(pt, batch), _eval(pt, batch)
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    c = _eval(pt, batch)
    assert torch.equal(a, b) and torch.equal(a, c)


# ---------------------------------------------------------------------------------------------------------------------
# 7. evaluations leave the training state as it was
# ---------------------------------------------------------------------------------------------------------------------
def _train(kind, with_eval):
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.optim import Lamb
    # the device step counter is process-wide: detach the previous run's, so that both runs start from the same seeds
    ops.extension().set_seed_step(None)
    model, arena, pt = _model(p_drop=0.1)
    if kind == "fp8":
        model.bert.fused_engine().enable_fp8()
    model.bert.unpad = kind == "unpad"
    opt = Lamb([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-3)
    arena.bind_optimizer(opt)
    ev = _loader_batch(8, 128, seed=11)
    losses = []
    for step in range(3):
        for micro in range(3):
            batch = _loader_batch(8, 128, seed=100 + 3 * step + micro)
            tok = _tokens(batch[2]) if kind == "unpad" else None
            losses.append(float(pt.forward_backward(*batch, grad_scale=1.0 / 3, tokens=tok)))
            if with_eval and micro == 1:
                eng = pt.engine
                before = (eng._calls, None if pt._seed_step is None else pt._seed_step.clone(), model.training)
                for _ in range(3):                                     # eager, eager, captured
                    _eval(pt, ev, _tokens(ev[2]) if kind == "unpad" else None)
                after = (eng._calls, None if pt._seed_step is None else pt._seed_step.clone(), model.training)
                assert before[0] == after[0] and before[2] == after[2]
                assert (before[1] is None) == (after[1] is None) and (before[1] is None or torch.equal(before[1], after[1]))
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    return losses, arena.flat_param.clone(), arena.exp_avg.clone(), arena.exp_avg_sq.clone()


@pytest.mark.parametrize("kind", ["bf16", "unpad", "fp8"])
def test_evaluations_do_not_perturb_deterministic_training(kind, monkeypatch):
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    ref = _train(kind, False)
    got = _train(kind, True)
    assert got[0] == ref[0], (got[0], ref[0])
    for name, a, b in zip(("weights", "exp_avg", "exp_avg_sq"), got[1:], ref[1:]):
        assert torch.equal(a, b), name


# ---------------------------------------------------------------------------------------------------------------------
# 8. the runtime
# ---------------------------------------------------------------------------------------------------------------------
def _run(tmp_path, steps, eval_dir=None, out_name="out"):
    from bert_pytorch_b200 import pretrain
    from bert_pytorch_b200.data import synthetic
    root = tmp_path / "w"
    if not (root / "model_config.json").exists():
        synthetic.make_workspace(str(root), num_shards=2, samples_per_shard=128, seq_len=128, vocab_size=1024,
                                 hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
                                 max_position_embeddings=128)
        synthetic.write_shards(str(tmp_path / "eval"), 2, 40, 128, 1024, next_sentence=True, seed=5)
    data = str(root / "sequences_lowercase_max_seq_len_128_next_seq_task_true")
    out = str(tmp_path / out_name)
    cfg = {"model_config_file": str(root / "model_config.json"), "max_predictions_per_seq": 20, "learning_rate": 1e-3,
           "global_batch_size": 16, "local_batch_size": 8, "max_steps": 8, "num_steps_per_checkpoint": 2,
           "log_prefix": "log", "disable_progress_bar": True}
    if eval_dir:
        cfg.update(eval_dir=eval_dir, num_eval_examples=50, eval_batch_size=16, eval_interval=2)
    path = str(tmp_path / f"{out_name}.json")
    with open(path, "w") as f:
        json.dump(cfg, f)
    pretrain.cli(["--config_file", path, "--input_dir", data, "--output_dir", out, "--steps", str(steps)])
    return out


def _rows(out, tag):
    return [r for r in csv.DictReader(open(os.path.join(out, "log_metrics.csv"))) if r["tag"] == tag]


def test_runtime_eval_rows_resume_and_no_eval_without_the_flag(tmp_path):
    from bert_pytorch_b200.utils import checkpoint as ck
    out = _run(tmp_path, 4, eval_dir=str(tmp_path / "eval"))
    ev = _rows(out, "eval")
    assert [int(r["step"]) for r in ev] == [2, 4]
    for r in ev:
        assert np.isfinite(float(r["eval_mlm_loss"])) and np.isfinite(float(r["eval_nsp_loss"]))
        assert 0 <= float(r["eval_mlm_accuracy"]) <= 1 and 0 <= float(r["eval_nsp_accuracy"]) <= 1
        assert int(float(r["eval_samples"])) == 50
    out = _run(tmp_path, 2, eval_dir=str(tmp_path / "eval"))               # resumes from step 4
    assert [int(r["step"]) for r in _rows(out, "eval")] == [2, 4, 6]
    assert [int(r["step"]) for r in _rows(out, "train")] == list(range(1, 7))
    plain = _run(tmp_path, 4, out_name="plain")
    assert not _rows(plain, "eval")
    keys = []
    for o in (out, plain):
        _, path = ck.find_latest(os.path.join(o, "pretrain_ckpts"))
        keys.append(set(torch.load(path, map_location="cpu", weights_only=False)))
    assert keys[0] == keys[1] == {"model", "optimizer", "sampler", "epoch", "scaler"}
