"""Deterministic mode on the H100 (``B200_DETERMINISTIC=1`` / ``torch.use_deterministic_algorithms``): every site that
sums in a scheduling-dependent order by default gives the same bits on a second call, the fixed-order forms still meet
the fp64 reference tests of their kernels, and whole training steps -- padded and unpadded, S = 128 and 512, NSP,
activation checkpointing, fp8 operands -- repeat bit for bit, also across the scheduling choices (weight-gradient side
stream, CUDA-graph replay) that only change when kernels run, and a replayed graph repeats its loss after batches of
another shape."""
import os

import pytest
import torch

import test_gpu_attention_reference as attn_ref
import test_gpu_optim_loss as optim_ref
from test_gpu_pretrain_unpad import _batch, _grad_errors, _grads, _model, _tokens

pytestmark = pytest.mark.gpu


@pytest.fixture
def det(monkeypatch):
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    from bert_pytorch_b200.ops import api as K
    assert K.deterministic()
    return K


def _twice(fn):
    """fn() twice; each call returns a tuple of tensors computed from the same inputs"""
    a = [t.clone() for t in fn()]
    b = [t.clone() for t in fn()]
    torch.cuda.synchronize()
    return a, b


def _assert_equal(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i, (x.double() - y.double()).abs().max().item())


def _rel(got, ref):
    return ((got.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item()


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernel sites: bitwise repeat (many waves of CTAs) and accuracy
# ---------------------------------------------------------------------------------------------------------------------
def test_wgrad_split_k_is_fixed_order(det):
    g = torch.Generator(device="cuda").manual_seed(1)
    dy = torch.randn(12288, 1024, device="cuda", generator=g).bfloat16()
    x = torch.randn(12288, 1024, device="cuda", generator=g).bfloat16()
    assert det.wgrad_splits(1024, 1024, 12288) > 1          # the default mode splits this shape
    base = torch.randn(1024, 1024, device="cuda", generator=g)

    def run():
        grad = base.clone()
        det.wgrad_accumulate(dy, x, grad, alpha=0.5)
        return (grad,)
    a, b = _twice(run)
    _assert_equal(a, b, "wgrad")
    ref = base.double() + 0.5 * dy.double().t() @ x.double()
    assert _rel(a[0], ref) < 1e-4


def test_fp8_wgrad_is_fixed_order(det, monkeypatch):
    meta = det.Fp8Meta(["dy", "x"], [True, False], "cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    dy = torch.randn(8192, 1024, device="cuda", generator=g).bfloat16()
    x = torch.randn(8192, 1024, device="cuda", generator=g).bfloat16()
    qdy = meta.quantize(dy, "dy", calibrate=True)
    qx = meta.quantize(x, "x", calibrate=True)

    def run():
        grad = torch.zeros(1024, 1024, device="cuda")
        det.wgrad_accumulate(qdy, qx, grad, scale_a=meta.inv_scale("dy"), scale_b=meta.inv_scale("x"), a_e5m2=True)
        return (grad,)
    a, b = _twice(run)
    _assert_equal(a, b, "fp8 wgrad")
    # the same sum as the default mode's split-K GEMM (checked against fp64 by test_gpu_fp8_reference), in one pass
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    assert _rel(a[0], run()[0].double()) < 1e-5


def test_gemm_colsum_is_fixed_order(det):
    g = torch.Generator(device="cuda").manual_seed(3)
    dy = torch.randn(12288, 1024, device="cuda", generator=g).bfloat16()
    w = (torch.randn(1024, 4096, device="cuda", generator=g) * 0.05).bfloat16()
    y1 = torch.rand(12288, 4096, device="cuda", generator=g).bfloat16()

    def run():
        cs = torch.ones(4096, device="cuda")
        out = det.gemm(dy, w, layout=det.NN, epi=det.EPI_MUL, res=y1, colsum=cs)
        return out, cs
    a, b = _twice(run)
    _assert_equal(a, b, "EPI_MUL colsum")
    assert _rel(a[1], 1.0 + a[0].double().sum(0)) < 1e-6          # the column sums of the bf16 output


def test_colsum_and_dgelu_dbias_are_fixed_order(det, monkeypatch):
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(12288, 4096, device="cuda", generator=g).bfloat16()
    dy = torch.randn(12288, 4096, device="cuda", generator=g).bfloat16()

    def run():
        cs, db = torch.zeros(4096, device="cuda"), torch.zeros(4096, device="cuda")
        det.colsum_accumulate(x, cs)
        dx = det.dgelu_bwd(dy, x, db)
        return cs, dx, db
    a, b = _twice(run)
    _assert_equal(a, b, "colsum / dgelu dbias")
    assert _rel(a[0], x.double().sum(0)) < 1e-6
    # dbias sums the fp32 products dy * gelu'(x) before their bf16 rounding, as the default kernel does
    xd = x.double()
    dgelu = 0.5 * (1 + torch.erf(xd / 2 ** 0.5)) + xd * torch.exp(-0.5 * xd * xd) / (2 * torch.pi) ** 0.5
    assert _rel(a[2], (dy.double() * dgelu).sum(0)) < 1e-5
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    assert _rel(a[2], run()[2].double()) < 1e-6


def test_layer_norm_bwd_is_fixed_order(det, monkeypatch):
    M, H = 12288, 1024
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, H, device="cuda", generator=g).bfloat16()
    gamma = torch.rand(H, device="cuda", generator=g) + 0.5
    beta = torch.randn(H, device="cuda", generator=g)
    _, mean, rstd = det.layer_norm_fwd(x, gamma, beta)
    dy = torch.randn(M, H, device="cuda", generator=g).bfloat16()

    def run():
        dg, db, dbias = (torch.zeros(H, device="cuda") for _ in range(3))
        dx, dxd = det.layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True,
                                     p_drop=0.1, seed=7, drop_stream=3)
        return dx, dxd, dg, db, dbias
    a, b = _twice(run)
    _assert_equal(a, b, "LN backward")
    xhat = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    assert _rel(a[2], (dy.double() * xhat).sum(0)) < 1e-5
    assert _rel(a[3], dy.double().sum(0)) < 1e-5
    # dbias: the kernel sums the dropped gradient before its bf16 rounding; the default mode sums the same values
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    assert _rel(a[4], run()[4].double()) < 1e-6


@pytest.mark.parametrize("form", ["padded", "packed", "no-seg", "chunked"])
def test_embedding_scatter_is_fixed_order(det, form):
    B, S, H, V = (320 if form == "chunked" else 96), 128, 1024, 30528      # 40960 rows: two sorted chunks
    M = B * S
    g = torch.Generator(device="cuda").manual_seed(6)
    ids = torch.randint(0, 200, (M,), device="cuda", generator=g, dtype=torch.int32)     # many repeats
    ids[M // 2:M // 2 + 3000] = 0                                                      # a long [PAD] run
    seg = torch.randint(0, 2, (M,), device="cuda", generator=g, dtype=torch.int32)
    if form == "no-seg":                                   # no segment ids: every row is token type 0
        seg = None
    pos_ids = torch.randint(0, S, (M,), device="cuda", generator=g, dtype=torch.int32) if form == "packed" else None
    de = torch.randn(M, H, device="cuda", generator=g).bfloat16()
    base = [torch.randn(n, H, device="cuda", generator=g) for n in (V, S, 2)]

    def run():
        gw, gp, gt = (t.clone() for t in base)
        det.embedding_bwd_scatter(de, ids, seg, gw, gp, gt, S, pos_ids=pos_ids)
        return gw, gp, gt
    a, b = _twice(run)
    _assert_equal(a, b, "embedding scatter")
    pos = pos_ids.long() if pos_ids is not None else torch.arange(M, device="cuda") % S
    tkey = seg.long() if seg is not None else torch.zeros(M, dtype=torch.long, device="cuda")
    for got, t0, key in zip(a, base, (ids.long(), pos, tkey)):
        ref = t0.double().index_add(0, key, de.double())
        assert (got.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


@pytest.mark.parametrize("form", ["padded", "varlen"])
def test_attention_dq_is_fixed_order_at_s512(det, form):
    B, S, heads, H = 16, 512, 16, 1024
    g = torch.Generator(device="cuda").manual_seed(8)
    lens = [S, 500, 129, 200, 511, 77, 384, 257, 300, 1, 450, 128, 640, 0, 256, 333]       # ends inside key blocks
    qkv, dctx = attn_ref._inputs("n0.5", B, S, H, lens, g)
    kw = dict(p_drop=0.1, seed=attn_ref.SEED, stream=9)
    if form == "padded":
        seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
        ctx, lse = det.attention_fwd(qkv, seqlens, heads, **kw)
        run = lambda: (det.attention_bwd(qkv, seqlens, ctx, dctx, lse, heads, **kw),)      # noqa: E731
    else:
        n = [min(max(x, 0), S) or S for x in lens]
        rows = torch.cat([torch.arange(b * S, b * S + n[b], device="cuda") for b in range(B)])
        pq, pd = qkv.view(B * S, -1)[rows].contiguous(), dctx.view(B * S, -1)[rows].contiguous()
        cu = torch.tensor([0] + list(torch.tensor(n).cumsum(0)), dtype=torch.int32, device="cuda")
        ctx, lse = det.attention_fwd(pq, None, heads, cu_seqlens=cu, S=S, **kw)
        run = lambda: (det.attention_bwd(pq, None, ctx, pd, lse, heads, cu_seqlens=cu, S=S, **kw),)   # noqa: E731
    a, b = _twice(run)
    _assert_equal(a, b, "attention dqkv")


@pytest.mark.parametrize("S", [128, 200, 512])
def test_attention_meets_the_fp64_reference_in_deterministic_mode(det, S):
    attn_ref.test_attention_matches_fp64_reference(S, 0.1, 16)
    attn_ref.test_attention_matches_fp64_reference_many_waves(S)


@pytest.mark.parametrize("S", [200, 512])
def test_varlen_attention_meets_the_fp64_reference_in_deterministic_mode(det, S):
    attn_ref.test_varlen_attention_matches_fp64_reference(S, 0.1)


def test_losses_are_fixed_order(det):
    g = torch.Generator(device="cuda").manual_seed(9)
    R, V = 1920, 30528
    x0, tgt = optim_ref._ce_rows(R, V, g)
    count = torch.tensor([int((tgt >= 0).sum())], dtype=torch.int32, device="cuda")
    B, H = 256, 1024
    pooled = torch.tanh(torch.randn(B, H, device="cuda", generator=g)).bfloat16()
    w = (torch.randn(2, H, device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn(2, device="cuda", generator=g) * 0.1
    labels = torch.randint(-1, 2, (B,), device="cuda", generator=g)

    def run():
        x, loss = x0.clone(), torch.zeros(1, device="cuda")
        det.softmax_ce_(x, tgt, count, 1.0, loss)
        dw, db = torch.zeros(2, H, device="cuda"), torch.zeros(2, device="cuda")
        dz = det.nsp_head_(pooled, w, bias, labels, 1.0, loss, dw, db)
        return x, loss, dz, dw, db
    a, b = _twice(run)
    _assert_equal(a, b, "losses")


@pytest.mark.parametrize("V,R", [(30528, 640), (2048, 80)])
def test_softmax_ce_meets_the_fp64_reference_in_deterministic_mode(det, V, R):
    optim_ref.test_softmax_ce_matches_fp64(V, R, 65536.0)
    optim_ref.test_softmax_ce_count_zero(V)


@pytest.mark.parametrize("B,H", [(7, 200), (256, 1024)])
def test_nsp_head_meets_the_fp64_reference_in_deterministic_mode(det, B, H):
    optim_ref.test_nsp_head_matches_fp64(B, H, 1024.0)
    optim_ref.test_nsp_head_all_ignored(B)


@pytest.mark.parametrize("case", optim_ref.LAMB_CASES[:4] + optim_ref.ADAM_CASES[-1:], ids=optim_ref._case_id)
def test_arena_optimizers_meet_the_fp64_reference_in_deterministic_mode(det, case):
    optim_ref.test_arena_optimizer_matches_fp64(case)


@pytest.mark.parametrize("opt", ["lamb", "adam"])
def test_loss_scaler_skip_in_deterministic_mode(det, opt):
    optim_ref.test_overflow_skips_the_step(opt)


def test_optimizer_norms_are_fixed_order(det):
    from bert_pytorch_b200.optim import GradientClipper, Lamb
    model, arena, _ = _model(S=128, layers=2)
    opt = Lamb([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-3)
    arena.bind_optimizer(opt)
    g = torch.Generator(device="cuda").manual_seed(10)
    grads = torch.randn(arena.flat_grad.shape, device="cuda", generator=g)
    p0, m0, v0 = arena.flat_param.clone(), arena.exp_avg.clone(), arena.exp_avg_sq.clone()
    tensors = [torch.randn(n, device="cuda", generator=g) for n in (5, 65536 * 3 + 7, 1 << 20, 1000)]

    def run():
        arena.flat_param.copy_(p0); arena.exp_avg.copy_(m0); arena.exp_avg_sq.copy_(v0)
        arena.flat_grad.copy_(grads)
        for gr in opt.param_groups:
            gr["step"] = 0
        opt.step()
        total, per = det.multi_tensor_l2norm(tensors, per_tensor=True)
        ps = [torch.nn.Parameter(torch.zeros_like(t)) for t in tensors]
        for p, t in zip(ps, tensors):
            p.grad = t.clone()
        GradientClipper(max_grad_norm=1.0).step(ps)
        return (arena.flat_param, arena.exp_avg, arena.exp_avg_sq, opt.last_grad_norm.reshape(1), total.reshape(1), per,
                *[p.grad for p in ps])
    a, b = _twice(run)
    _assert_equal(a, b, "LAMB / l2norm / clip")
    ref = torch.stack([t.double().norm() for t in tensors])
    assert _rel(a[5], ref) < 1e-6 and abs(a[4].item() - ref.norm().item()) <= 1e-6 * ref.norm().item()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the engine: whole micro-steps and optimizer steps
# ---------------------------------------------------------------------------------------------------------------------
def _train(S, unpad, *, ckpt=False, fp8=False, graphs=False, side=True, steps=2, seed=0):
    """Two micro-steps + arena-LAMB steps of a fresh dropout-0.1 NSP model; returns the loss and gradients of the first
    micro-step and the weights and moments at the end."""
    from bert_pytorch_b200.optim import Lamb
    model, arena, pt = _model(S=S, p_drop=0.1, seed=seed)
    model.bert.unpad = unpad
    model.checkpoint_activations(ckpt)
    if fp8:
        pt.engine.enable_fp8()
    pt.engine.wgrad_side = side
    pt.use_graphs = graphs
    pt.graph_warmup = 1
    opt = Lamb([{"params": list(model.parameters()), "weight_decay": 0.01}], lr=1e-3)
    arena.bind_optimizer(opt)
    B = 8
    lens = [S, S // 3, 1, 0, S - 1, 65, S // 2 + 3, 129 if S > 128 else 100]
    out = {}
    for step in range(max(steps, 3 if graphs else 1)):
        batch = _batch(B, S, lens, seed=step)
        loss = pt.forward_backward(*batch, tokens=_tokens(batch[2]) if unpad else None)
        torch.cuda.synchronize()
        if step == 0:
            out["loss"] = loss.clone()
            out.update({"g." + k: v for k, v in _grads(arena).items()})
        opt.step()
        opt.zero_grad()
    out.update(param=arena.flat_param.clone(), m=arena.exp_avg.clone(), v=arena.exp_avg_sq.clone())
    torch.cuda.synchronize()
    return out


def _same(a, b, what):
    bad = [(k, (a[k].double() - b[k].double()).abs().max().item()) for k in a if not torch.equal(a[k], b[k])]
    assert not bad, (what, len(bad), bad[:8])


@pytest.mark.parametrize("unpad", [False, True], ids=["padded", "unpadded"])
@pytest.mark.parametrize("S", [128, 512])
def test_two_fresh_runs_are_bitwise_equal(det, S, unpad):
    _same(_train(S, unpad), _train(S, unpad), (S, unpad))


@pytest.mark.parametrize("variant", ["ckpt", "fp8"])
def test_checkpointed_and_fp8_runs_are_bitwise_equal(det, variant):
    kw = {"ckpt": True} if variant == "ckpt" else {"fp8": True}
    _same(_train(128, False, **kw), _train(128, False, **kw), variant)
    if variant == "ckpt":
        _same(_train(512, True, **kw), _train(512, True, **kw), "ckpt unpadded")


@pytest.mark.parametrize("unpad", [False, True], ids=["padded", "unpadded"])
def test_scheduling_does_not_change_the_bits(det, unpad):
    """The weight-gradient side stream and CUDA-graph replay only change when kernels run.  A replay draws its dropout
    seed from the device step counter: the eager program is run at the same counter."""
    _same(_train(512, unpad, steps=3), _train(512, unpad, side=False, steps=3), "side stream off")
    S, B = 512, 8
    model, arena, pt = _model(S=S, p_drop=0.1)
    model.bert.unpad = unpad
    assert pt.use_graphs
    batch = _batch(B, S, [S, S // 3, 1, 0, S - 1, 65, S // 2 + 3, 129], seed=1)
    tok = _tokens(batch[2]) if unpad else None
    for _ in range(pt.graph_warmup):
        pt.forward_backward(*batch, tokens=tok)
    for _ in range(2):                                   # the capture, then a replay
        step0 = pt._seed_step.clone() if pt._seed_step is not None else torch.zeros(1, dtype=torch.int64, device="cuda")
        arena.zero_grad()
        replay = {"loss": pt.forward_backward(*batch, tokens=tok).clone()}
        torch.cuda.synchronize()
        replay.update(_grads(arena))
        pt._seed_step.copy_(step0)
        pt._seed_step.add_(1)
        arena.zero_grad()
        eager = {"loss": pt._program(*batch, 1.0, seed=pt.engine._seed_base, bucket=pt._bucket(batch[2], tok)).clone()}
        torch.cuda.synchronize()
        eager.update(_grads(arena))
        _same(replay, eager, "graph replay")


def test_nsp_graph_replays_alike_after_a_batch_of_another_size(det):
    """The graph of a batch shape reads the [CLS] row indices of the NSP head through the pointer it was captured with:
    a batch of another size (the short last batch of an epoch) must leave that tensor alive.  Dropout 0 and no
    optimizer step, so every replay of the same batch gives the same loss."""
    S = 128
    model, arena, pt = _model(S=S)
    assert pt.use_graphs and pt.has_nsp
    full = _batch(8, S, [S, S // 3, 1, 0, S - 1, 65, S // 2 + 3, 100], seed=1)
    short = _batch(5, S, [S, 3, 64, 0, 99], seed=2)

    def captured(batch):                             # the eager calls, the capture, then one more replay
        losses = [pt.forward_backward(*batch).clone() for _ in range(pt.graph_warmup + 2)]
        torch.cuda.synchronize()
        return losses[-1]
    before = captured(full)
    captured(short)
    assert sum("graph" in e for e in pt._graphs.values()) == 2
    after = pt.forward_backward(*full).clone()
    torch.cuda.synchronize()
    assert torch.equal(before, after), (before.item(), after.item())


def test_deterministic_mode_agrees_with_the_default_mode(monkeypatch):
    from bert_pytorch_b200.ops import api as K
    runs = []
    for flag in ("0", "1"):
        monkeypatch.setenv("B200_DETERMINISTIC", flag)
        assert K.deterministic() == (flag == "1")
        runs.append(_train(512, False, steps=1))
    assert abs(runs[0]["loss"].item() - runs[1]["loss"].item()) <= 1e-5 * abs(runs[0]["loss"].item())
    grads = [{k[2:]: v for k, v in r.items() if k.startswith("g.")} for r in runs]
    bad = _grad_errors(grads[1], grads[0])
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# 3. fine-tuning under torch's flag, and the pre-training runtime
# ---------------------------------------------------------------------------------------------------------------------
def _ner_step():
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForTokenClassification
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Adam, GradientClipper
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=2048, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=1024, max_position_embeddings=512)
    model = BertForTokenClassification(cfg, num_labels=9).cuda()
    model.bert.unpad = True
    arena = ParamArena(model)
    opt = Adam(model.parameters(), lr=1e-3, bias_correction=False)
    arena.bind_optimizer(opt)
    clip = GradientClipper(max_grad_norm=1.0)
    g = torch.Generator(device="cuda").manual_seed(1)
    B, S = 16, 512
    ids = torch.randint(5, 2048, (B, S), device="cuda", generator=g)
    lens = torch.tensor([S, 500, 129, 200, 511, 77, 384, 257, 300, 1, 450, 128, 33, 0, 256, 333], device="cuda")
    mask = (torch.arange(S, device="cuda")[None, :] < lens[:, None]).long()
    labels = torch.randint(0, 9, (B, S), device="cuda", generator=g)
    model.train()
    loss = model(ids, torch.zeros_like(ids), mask, labels)
    loss.backward()
    clip.step(model.parameters())
    opt.step()
    torch.cuda.synchronize()
    return [loss.detach().clone()] + [p.detach().clone() for p in model.parameters()]


def test_token_classification_step_repeats_under_torch_flag():
    from bert_pytorch_b200.ops import api as K
    prev = torch.are_deterministic_algorithms_enabled()
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        assert K.deterministic()
        a, b = _ner_step(), _ner_step()
    finally:
        torch.use_deterministic_algorithms(prev)
    _assert_equal(a, b, "NER step")


def test_pretraining_runtime_checkpoints_are_bitwise_equal(tmp_path):
    from test_gpu_e2e import _run
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.utils import checkpoint as ck
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for extra in ((), ("--unpad",)):
            payloads = []
            for i in range(2):
                ops.extension().set_seed_step(None)      # a graph of the previous run left its step counter set
                out, _ = _run(tmp_path / f"{len(extra)}-{i}", ("--deterministic", *extra))
                _, path = ck.find_latest(os.path.join(out, "pretrain_ckpts"))
                payloads.append(torch.load(path, map_location="cpu", weights_only=False))
            a, b = payloads
            assert a["model"].keys() == b["model"].keys()
            for k in a["model"]:
                assert torch.equal(a["model"][k], b["model"][k]), (extra, k)
            sa, sb = a["optimizer"]["state"], b["optimizer"]["state"]
            assert sa.keys() == sb.keys() and sa
            for k in sa:
                for n in sa[k]:
                    if torch.is_tensor(sa[k][n]):
                        assert torch.equal(sa[k][n], sb[k][n]), (extra, k, n)
    finally:
        torch.use_deterministic_algorithms(prev)
