"""Unpadded pre-training on the H100: the device packing kernel and the remapped MLM compaction against a numpy oracle,
``FusedPretrainer`` unpadded against padded, the inertness of the pad tail, one CUDA graph per token bucket replayed in
data order, the packed-row dropout numbering against an fp32 oracle, the runtime with ``--unpad``, and the padded
fallbacks (fp8, K-FAC taps).

Two sums in the program are fp32 atomics whose order varies from run to run: the loss (``softmax_ce`` /
``nsp_head`` add per row) and the split-K weight-gradient GEMMs.  Where the same program runs twice, the loss is
therefore compared to 1e-6 relative (a different dropout seed moves it by far more) and the gradients to the bound
of the existing graph-replay test; the sequence output, which has no such sum, is compared bitwise."""
import csv
import json
import os

import numpy as np
import pytest
import torch

from test_pretrain_unpad_cpu import masks, np_pack

pytestmark = pytest.mark.gpu

V, MP = 2048, 20


def _model(S=128, layers=2, p_drop=0.0, nsp=True, seed=0):
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    from bert_pytorch_b200.models.arena import ParamArena
    torch.manual_seed(seed)
    cfg = BertConfig(vocab_size_or_config_json_file=V, hidden_size=256, num_hidden_layers=layers, num_attention_heads=4,
                     intermediate_size=1024, max_position_embeddings=S, hidden_dropout_prob=p_drop,
                     attention_probs_dropout_prob=p_drop, next_sentence=nsp)
    cfg.max_predictions_per_seq = MP
    model = BertForPreTraining(cfg).cuda()
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "LayerNorm.weight" in n:
                p.uniform_(0.5, 1.5)
            elif "bias" in n:
                p.normal_(0, 0.1)
    arena = ParamArena(model)
    model.train()
    return model, arena, model.pretrain_engine()


def _batch(B, S, lens, seed=0, holes=False):
    """int32 batch like the loader's: prefix masks of ``lens`` (0 = an empty row), labels inside the mask."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(5, V, (B, S), device="cuda", generator=g, dtype=torch.int32)
    L = torch.tensor(lens, device="cuda")
    pos = torch.arange(S, device="cuda")[None, :]
    mask = (pos < L[:, None]).int()
    if holes:
        mask[0, 3:9] = 0
    seg = ((pos > L[:, None] // 2) & (mask > 0)).int()
    labels = torch.full((B, S), -1, dtype=torch.int32, device="cuda")
    for b in range(B):
        n = max(int(lens[b]), 1) if lens[b] > 0 else S
        p = torch.randperm(n, device="cuda", generator=g)[:MP]
        p = p[mask[b, p] > 0] if lens[b] > 0 else p
        labels[b, p] = ids[b, p]
    nsl = torch.randint(0, 2, (B,), device="cuda", generator=g, dtype=torch.int32)
    return ids, seg, mask, labels, nsl


def _grads(arena):
    return {s.name: arena.grad(s.name).float().clone() for s in arena.slots}


def _grad_errors(got, ref, bound=1e-3):
    """Parameters whose max abs error exceeds ``bound`` x the norm of the reference gradient.  The key bias is left
    out: its gradient is zero in exact arithmetic (softmax is invariant to it), so both are rounding noise."""
    bad = []
    for n, r in ref.items():
        if n.endswith("attention.self.key.bias"):
            continue
        err = (got[n] - r).abs().max().item()
        if not err <= bound * r.norm().item():
            bad.append((n, err, r.norm().item()))
    return bad


def _tokens(mask):
    from bert_pytorch_b200.models.fused import packed_tokens
    return packed_tokens(mask.cpu())


# ---------------------------------------------------------------------------------------------------------------------
# 1. the packing kernel and the remapped MLM compaction
# ---------------------------------------------------------------------------------------------------------------------
def _mask_cases():
    from bert_pytorch_b200.models.fused import token_bucket
    B, S = 12, 128
    M = B * S
    g = 128 * -(-M // (128 * 16))
    cases = [("random", masks(B, S, 0)), ("random2", masks(B, S, 5)),
             ("full", np.ones((B, S), np.int32)), ("empty", np.zeros((B, S), np.int32))]
    for name, T in (("edge", 2 * g), ("edge-1", 2 * g - 1), ("edge+1", 2 * g + 1), ("last", M - 1), ("one-per-row", B)):
        lens = np.full(B, T // B)
        lens[: T % B] += 1
        cases.append((name, (np.arange(S)[None, :] < lens[:, None]).astype(np.int32)))
    holes = masks(B, S, 3)
    holes[:, 0] = 1
    cases.append(("holes", holes))
    out = []
    for name, m in cases:
        T = np_pack(m, m, m, M, B)["T"]
        out.append((name, m, *token_bucket(T, B, S)))
    out.append(("cap=B*S", masks(B, S, 7), M, B))
    return out


@pytest.mark.parametrize("case", _mask_cases(), ids=lambda c: c[0])
def test_pack_tokens_matches_numpy_oracle(case):
    from bert_pytorch_b200.ops import api as K
    name, m, T_cap, D = case
    B, S = m.shape
    g = np.random.default_rng(1)
    ids = g.integers(5, V, (B, S)).astype(np.int32)
    seg = g.integers(0, 2, (B, S)).astype(np.int32)
    want = np_pack(m, ids, seg, T_cap, D)
    dev = lambda a: torch.from_numpy(a).cuda()           # noqa: E731
    # outputs start as garbage: every element must be written
    got = K.pack_tokens(dev(m), dev(ids), dev(seg), T_cap, D)
    for k, t in zip(("ids", "seg", "pos", "cu", "cls", "row_map"), got):
        assert np.array_equal(t.cpu().numpy(), want[k]), (name, k)
    cu = got[3].cpu().numpy()
    assert cu[-1] == T_cap and (np.diff(cu[B:]) <= S).all()
    # no segments (RoBERTa-style configs): zeros
    assert not K.pack_tokens(dev(m), dev(ids), None, T_cap, D)[1].any()
    # remapped MLM compaction: labels at masked tokens are dropped; the rest name packed rows
    labels = np.full((B, S), -1, np.int32)
    for b in range(B):
        p = g.choice(S, 10, replace=False)
        labels[b, p] = ids[b, p]
    idx, tgt, count = K.mlm_compact(dev(labels), 8, row_map=got[5])
    rm = want["row_map"].reshape(B, S)
    w_idx, w_tgt = np.full((B, 8), -1), np.full((B, 8), -1)
    n = 0
    for b in range(B):
        s = [s for s in range(S) if labels[b, s] >= 0 and rm[b, s] >= 0][:8]
        w_idx[b, :len(s)], w_tgt[b, :len(s)] = rm[b, s], labels[b, s]
        n += len(s)
    assert np.array_equal(idx.cpu().numpy().reshape(B, 8), w_idx) and np.array_equal(tgt.cpu().numpy().reshape(B, 8), w_tgt)
    assert count.item() == n


def test_mlm_compact_without_row_map_is_unchanged():
    from bert_pytorch_b200.ops import api as K
    labels = torch.full((3, 64), -1, dtype=torch.int32, device="cuda")
    labels[0, [1, 5, 9]] = 7
    labels[2, 10:40] = 3
    idx, tgt, count = K.mlm_compact(labels, 16)
    assert idx.view(3, 16)[0, :4].tolist() == [1, 5, 9, -1] and idx.view(3, 16)[2, 0].item() == 2 * 64 + 10
    assert count.item() == 3 + 16


# ---------------------------------------------------------------------------------------------------------------------
# 2. unpadded against padded FusedPretrainer (dropout 0)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ckpt", [False, True], ids=["saved", "ckpt"])
@pytest.mark.parametrize("nsp", [True, False], ids=["nsp", "mlm-only"])
@pytest.mark.parametrize("S", [128, 512])
def test_unpadded_matches_padded(S, nsp, ckpt):
    model, arena, pt = _model(S=S, nsp=nsp)
    pt.use_graphs = False
    model.checkpoint_activations(ckpt)
    B = 8
    lens = [S, S // 3, 1, 0, S - 1, 65, S // 2 + 3, 129 if S > 128 else 100]
    batch = _batch(B, S, lens)
    res = []
    for unpad in (False, True):
        model.bert.unpad = unpad
        arena.zero_grad()
        loss = pt.forward_backward(*batch, tokens=_tokens(batch[2]) if unpad else None).item()
        torch.cuda.synchronize()
        res.append((loss, _grads(arena)))
    assert abs(res[1][0] - res[0][0]) <= 1e-5 * abs(res[0][0]), (res[0][0], res[1][0])
    bad = _grad_errors(res[1][1], res[0][1])
    assert not bad, bad
    # the device count (no tokens given) picks the same bucket
    assert pt._bucket(batch[2], None) == pt._bucket(batch[2], _tokens(batch[2]))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the pad tail is inert
# ---------------------------------------------------------------------------------------------------------------------
def test_pad_tail_is_inert():
    from bert_pytorch_b200.models.fused import pack_device, token_bucket
    S, B = 128, 8
    model, arena, pt = _model(S=S, p_drop=0.1)
    batch = _batch(B, S, [100, 7, 128, 0, 33, 64, 90, 12])
    T = _tokens(batch[2])
    bucket = token_bucket(T, B, S)
    full = (B * S, -(-(B * S - T) // S))
    assert bucket[0] < B * S
    seed = 0x1234567
    res = []
    for bk in (bucket, full):
        pk = pack_device(batch[2], batch[0], batch[1], *bk)
        seq, _ = pt.engine.forward(batch[0], batch[1], batch[2], training=True, seed=seed, dropout=True, pack=pk)
        assert torch.isfinite(seq.float()).all()
        arena.zero_grad()
        loss = pt._program(*batch, 1.0, seed=seed, bucket=bk).item()
        torch.cuda.synchronize()
        res.append((seq[:T].clone(), loss, _grads(arena)))
    assert torch.equal(res[0][0], res[1][0])               # real rows do not depend on T_cap
    assert abs(res[0][1] - res[1][1]) <= 1e-6 * abs(res[0][1])
    assert all(torch.isfinite(g).all() for g in res[1][2].values())
    bad = _grad_errors(res[1][2], res[0][2])
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# 4. one graph per bucket, replayed in data order
# ---------------------------------------------------------------------------------------------------------------------
def test_graphs_per_bucket_replay_like_the_eager_program():
    from bert_pytorch_b200.models.fused import token_bucket
    S, B = 128, 8
    model, arena, pt = _model(S=S, p_drop=0.1)
    model.bert.unpad = True
    assert pt.use_graphs
    batches = {"A": _batch(B, S, [128] * 8, seed=1), "B": _batch(B, S, [64] * 8, seed=2),
               "C": _batch(B, S, [20, 3, 0, 9, 30, 11, 5, 1], seed=3)}
    buckets = {k: token_bucket(_tokens(b[2]), B, S) for k, b in batches.items()}
    assert len(set(buckets.values())) == 3
    for k in "ABC":                                       # the warm-up calls run eagerly
        for _ in range(pt.graph_warmup):
            pt.forward_backward(*batches[k], tokens=_tokens(batches[k][2]))
    torch.cuda.synchronize()
    eng = pt.engine
    for k in "ABACB":
        b = batches[k]
        step0 = pt._seed_step.clone() if pt._seed_step is not None else torch.zeros(1, dtype=torch.int64, device="cuda")
        arena.zero_grad()
        loss_g = pt.forward_backward(*b, tokens=_tokens(b[2])).item()
        torch.cuda.synchronize()
        grads_g = _grads(arena)
        # the eager program at the same seed counter
        pt._seed_step.copy_(step0)
        pt._seed_step.add_(1)
        arena.zero_grad()
        loss_e = pt._program(*b, 1.0, seed=eng._seed_base, bucket=buckets[k]).item()
        torch.cuda.synchronize()
        assert abs(loss_g - loss_e) <= 1e-6 * abs(loss_e), (k, loss_g, loss_e)
        grads_e = _grads(arena)
        for n, r in grads_e.items():
            scale = r.abs().max().item() + 1e-12
            assert (grads_g[n] - r).abs().max().item() <= 1e-4 * scale, (k, n)
    graphs = [key for key, ent in pt._graphs.items() if "graph" in ent]
    assert len(graphs) == 3 and {key[-1] for key in graphs} == set(buckets.values())


# ---------------------------------------------------------------------------------------------------------------------
# 5. packed-row dropout numbering against an fp32 oracle fed the kernels' keep bits
# ---------------------------------------------------------------------------------------------------------------------
def test_device_packing_with_dropout_matches_fp32_oracle():
    import test_gpu_unpadded as U
    from bert_pytorch_b200.models.fused import pack_device, pack_rows, token_bucket
    P_DROP, SEED = 0.1, 0x5EED1234ABC
    model, arena = U._model(layers=1, p_drop=P_DROP, S=256)
    eng = model.fused_engine()
    B, S = 8, 256
    ids, seg, mask = U._batch(B, S, [256, 33, 128, 129, 1, 200, 64, 250], holes=True)
    ref_pk = pack_rows(mask)
    T = ref_pk.T
    pk = pack_device(mask, ids, seg, *token_bucket(T, B, S))
    assert pk.T > T                                       # a real pad tail
    d_out = torch.zeros(pk.T, 1024, dtype=torch.bfloat16, device="cuda")
    d_out[:T] = (torch.randn(T, 1024, device="cuda") * 0.1).bfloat16()
    params = {s.name: (arena.shadow(s.name).float() if "LayerNorm" not in s.name else arena.view(s.name).clone()
                       ).requires_grad_(True) for s in arena.slots}
    model.train()
    arena.zero_grad()
    seq, sv = eng.forward(ids, seg, mask, training=True, seed=SEED, dropout=True, pack=pk)
    eng.backward(sv, d_out)
    torch.cuda.synchronize()
    rows = ref_pk.rows.long()
    ref_out = U._oracle_packed(params, ids.view(-1)[rows], seg.view(-1)[rows], ref_pk, B, S, 16, P_DROP, SEED,
                               d_out[:T])
    assert ((seq[:T].float() - ref_out).norm() / ref_out.norm()).item() < 1e-2
    bad = []
    for name, t in params.items():
        if t.grad is None or "pooler" in name:
            continue
        g, g_ref = arena.grad(name).float(), t.grad
        if name.endswith("attention.self.key.bias"):
            continue
        cos = U._cos(g, g_ref)
        rel = ((g - g_ref).norm() / g_ref.norm().clamp_min(1e-12)).item()
        if not (cos >= 0.9995 and rel <= 1e-2):
            bad.append((name, round(cos, 6), round(rel, 5)))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# 6. the runtime
# ---------------------------------------------------------------------------------------------------------------------
def _run(tmp_path, steps, extra=()):
    from bert_pytorch_b200 import pretrain
    from bert_pytorch_b200.data import synthetic
    data, model_json, _ = synthetic.make_workspace(
        str(tmp_path / "w"), num_shards=2, samples_per_shard=256, seq_len=128, vocab_size=1024, hidden_size=128,
        num_hidden_layers=2, num_attention_heads=2, intermediate_size=512, max_position_embeddings=128)
    out = str(tmp_path / "run" / "out")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cfg = {"model_config_file": model_json, "max_predictions_per_seq": 20, "learning_rate": 1e-3,
           "global_batch_size": 32, "local_batch_size": 8, "max_steps": 8, "num_steps_per_checkpoint": 4,
           "log_prefix": "log", "disable_progress_bar": True, "unpad": True}
    path = os.path.join(os.path.dirname(out), "train.json")
    with open(path, "w") as f:
        json.dump(cfg, f)
    pretrain.cli(["--config_file", path, "--input_dir", data, "--output_dir", out, "--steps", str(steps), *extra])
    return out


def test_runtime_with_unpad_graphs_and_resume(tmp_path):
    from bert_pytorch_b200.ops import api as K
    from bert_pytorch_b200.utils import checkpoint as ck
    n0 = K.KERNEL_LAUNCHES
    out = _run(tmp_path, 4)
    out = _run(tmp_path, 4)                               # resumes from step 4
    assert K.KERNEL_LAUNCHES - n0 > 8 * 4 * 50
    rows = list(csv.DictReader(open(os.path.join(out, "log_metrics.csv"))))
    assert [int(r["step"]) for r in rows] == list(range(1, 9))
    assert all(np.isfinite(float(r["average_loss"])) for r in rows)
    step, path = ck.find_latest(os.path.join(out, "pretrain_ckpts"))
    assert step == 8
    payload = torch.load(path, map_location="cpu", weights_only=False)
    assert set(payload) == {"model", "optimizer", "sampler", "epoch", "scaler"}
    assert "bert.encoder.layer.0.attention.self.query.weight" in payload["model"]


# ---------------------------------------------------------------------------------------------------------------------
# 7. fallbacks
# ---------------------------------------------------------------------------------------------------------------------
def test_fp8_warns_once_and_runs_padded():
    import warnings
    S, B = 128, 8
    res = []
    for unpad in (False, True):
        model, arena, pt = _model(S=S)
        pt.use_graphs = False
        pt.engine.enable_fp8()
        model.bert.unpad = unpad
        batch = _batch(B, S, [100, 7, 128, 0, 33, 64, 90, 12])
        losses = []
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            for _ in range(3):
                arena.zero_grad()
                losses.append(pt.forward_backward(*batch, tokens=_tokens(batch[2])).item())
        torch.cuda.synchronize()
        hits = sum("no unpadded pre-training path" in str(w.message) for w in rec)
        assert hits == (1 if unpad else 0)
        res.append((losses, _grads(arena)))
    # the same padded program from the same weights: the loss up to the order of its fp32 atomics
    assert all(abs(a - b) <= 1e-6 * abs(a) for a, b in zip(res[0][0], res[1][0])), res
    assert not _grad_errors(res[1][1], res[0][1], bound=1e-4)


def test_kfac_tapped_micro_steps_run_padded():
    model, arena, pt = _model(S=128)
    model.bert.unpad = True

    class Taps:
        capture = True
    batch = _batch(8, 128, [100, 7, 128, 0, 33, 64, 90, 12])
    model.bert._kfac = Taps()
    try:
        assert pt._bucket(batch[2], 500) is None
        Taps.capture = False
        assert pt._bucket(batch[2], 500) is not None
    finally:
        del model.bert._kfac
