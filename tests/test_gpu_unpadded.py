"""Unpadded fused encoder on the H100: variable-length attention on packed rows against the padded kernels, embeddings
with explicit position ids, the engine with packed rows against the padded engine and an fp32 oracle, and the
fine-tuning models with ``BertModel.unpad``."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GUARD = 64                      # rows of a sentinel-filled guard region after the T packed rows


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _lens(S):
    return sorted({n for n in (1, 63, 64, 65, 127, 128, 129, S - 1, S) if n <= S}, key=lambda n: (n * 7919) % 13)


def _pack(lens, S):
    mask = torch.zeros(len(lens), S, dtype=torch.long, device="cuda")
    for b, n in enumerate(lens):
        mask[b, :n] = 1
    from bert_pytorch_b200.models.fused import pack_rows
    return mask, pack_rows(mask)


def _cos(a, b):
    return F.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0).item()


def _varlen(C, qkv_p, cu, lse_shape, heads, dctx_p, p_drop, seed=7, stream=3):
    """The varlen kernels with every output followed by a guard region -> (ctx, lse, dqkv, guards intact)."""
    T, H = qkv_p.size(0), qkv_p.size(1) // 3
    scale = 1.0 / math.sqrt(H // heads)
    ctx_buf = torch.full((T + GUARD, H), -7.0, dtype=torch.bfloat16, device="cuda")
    dqkv_buf = torch.full((T + GUARD, 3 * H), -7.0, dtype=torch.bfloat16, device="cuda")
    acc_buf = torch.full(((T + GUARD) * H,), -7.0, dtype=torch.float32, device="cuda")
    lse = torch.empty(*lse_shape, dtype=torch.float32, device="cuda")
    S = lse_shape[2]
    C.attention_fwd(qkv_p, None, ctx_buf[:T], lse, heads, scale, p_drop, seed, stream, None, None, False, cu, S)
    C.attention_bwd(qkv_p, None, ctx_buf[:T], dctx_p, lse, dqkv_buf[:T], torch.empty_like(lse), acc_buf[:T * H], heads,
                    scale, p_drop, seed, stream, None, None, False, cu, S)
    torch.cuda.synchronize()
    intact = bool((ctx_buf[T:] == -7.0).all() and (dqkv_buf[T:] == -7.0).all() and (acc_buf[T * H:] == -7.0).all())
    return ctx_buf[:T], lse, dqkv_buf[:T], intact


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("S", [128, 384, 512])
def test_varlen_attention_matches_padded_kernels(S, p_drop):
    K = _api()
    from bert_pytorch_b200.ops import extension
    C = extension()
    torch.manual_seed(S)
    heads = 2
    H = heads * 64
    lens = _lens(S)
    B = len(lens)
    mask, pk = _pack(lens, S)
    valid = mask.view(-1).bool()
    rows = pk.rows.long()
    qkv = (torch.randn(B, S, 3 * H, device="cuda") * 0.7).to(torch.bfloat16)
    dctx = (torch.randn(B, S, H, device="cuda") * 0.5).to(torch.bfloat16) * mask[:, :, None].to(torch.bfloat16)
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ctx, lse = K.attention_fwd(qkv, seqlens, heads, p_drop=p_drop, seed=7, stream=3)
    dqkv = K.attention_bwd(qkv, seqlens, ctx, dctx, lse, heads, p_drop=p_drop, seed=7, stream=3).view(B * S, 3 * H)

    qkv_p = qkv.view(B * S, 3 * H)[rows].contiguous()
    dctx_p = dctx.view(B * S, H)[rows].contiguous()
    ctx_p, lse_p, dqkv_p, intact = _varlen(C, qkv_p, pk.cu_seqlens, (B, heads, S), heads, dctx_p, p_drop)
    assert intact, "a varlen kernel wrote past row T"
    assert torch.equal(ctx_p, ctx.view(B * S, H)[rows])
    lse_valid = valid.view(B, 1, S).expand(B, heads, S)
    assert torch.equal(lse_p[lse_valid], lse[lse_valid])
    assert torch.equal(dqkv_p[:, H:], dqkv[rows, H:])                       # dK and dV
    dq, dq_ref = dqkv_p[:, :H].float(), dqkv[rows, :H].float()              # fp32 atomics: reduction order only
    assert _cos(dq, dq_ref) >= 0.99999
    assert ((dq - dq_ref).abs() <= dq_ref.abs() * 2 ** -7 + 1e-3 * dq_ref.abs().max()).all()

    if p_drop == 0.0:                                                        # each sequence alone = inside the batch
        cu = pk.cu_seqlens.tolist()
        for b, n in enumerate(lens):
            sl = slice(cu[b], cu[b + 1])
            one = torch.tensor([0, n], dtype=torch.int32, device="cuda")
            c1, l1, d1, ok = _varlen(C, qkv_p[sl].contiguous(), one, (1, heads, S), heads, dctx_p[sl].contiguous(), 0.0)
            assert ok
            assert torch.equal(c1, ctx_p[sl]), (b, n)
            assert torch.equal(l1[0, :, :n], lse_p[b, :, :n]), (b, n)
            assert torch.equal(d1[:, H:], dqkv_p[sl, H:]), (b, n)


def test_embeddings_with_position_ids_match_padded():
    K = _api()
    torch.manual_seed(1)
    B, S, H, V = 6, 128, 1024, 512
    lens = [128, 1, 77, 64, 127, 9]
    mask, pk = _pack(lens, S)
    mask[2, 40:50] = 0                                  # a hole: positions keep their original index
    from bert_pytorch_b200.models.fused import pack_rows
    pk = pack_rows(mask)
    rows = pk.rows.long()
    ids = torch.randint(0, V, (B * S,), device="cuda", dtype=torch.int32)
    seg = torch.randint(0, 2, (B * S,), device="cuda", dtype=torch.int32)
    word = (torch.randn(V, H, device="cuda") * 0.1).bfloat16()
    pos = (torch.randn(S, H, device="cuda") * 0.1).bfloat16()
    typ = (torch.randn(2, H, device="cuda") * 0.1).bfloat16()
    g = torch.rand(H, device="cuda") + 0.5
    b = torch.randn(H, device="cuda") * 0.1
    ref = K.embedding_fwd(ids, seg, word, pos, typ, g, b, S)
    got = K.embedding_fwd(ids[rows].contiguous(), seg[rows].contiguous(), word, pos, typ, g, b, S, pos_ids=pk.pos_ids)
    for r, t in zip(ref, got):
        assert torch.equal(r[rows], t)
    de = (torch.randn(B * S, H, device="cuda") * 0.1).bfloat16() * mask.view(-1, 1).bfloat16()
    grads = []
    for args in ((de, ids, seg, None), (de[rows].contiguous(), ids[rows].contiguous(), seg[rows].contiguous(), pk.pos_ids)):
        gw, gp, gt = (torch.zeros(n, H, device="cuda") for n in (V, S, 2))
        K.embedding_bwd_scatter(args[0], args[1], args[2], gw, gp, gt, S, pos_ids=args[3])
        grads.append((gw, gp, gt))
    torch.cuda.synchronize()
    for r, t in zip(*grads):
        assert torch.allclose(t, r, rtol=1e-5, atol=1e-5 * r.abs().max().item()), (t - r).abs().max().item()


# ------------------------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------------------------
def _model(cls=None, layers=2, p_drop=0.0, S=512, num_labels=None, seed=0):
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertModel
    from bert_pytorch_b200.models.arena import ParamArena
    torch.manual_seed(seed)
    cfg = BertConfig(vocab_size_or_config_json_file=2048, hidden_size=1024, num_hidden_layers=layers,
                     num_attention_heads=16, intermediate_size=4096, max_position_embeddings=S,
                     hidden_dropout_prob=p_drop, attention_probs_dropout_prob=p_drop)
    cls = cls or BertModel
    model = (cls(cfg, num_labels) if num_labels else cls(cfg)).cuda()
    with torch.no_grad():                               # O(1) LayerNorm gains / biases, not the init values
        for n, p in model.named_parameters():
            if "LayerNorm.weight" in n:
                p.uniform_(0.5, 1.5)
            elif "bias" in n:
                p.normal_(0, 0.1)
    return model, ParamArena(model)


def _batch(B, S, lens, holes=False, V=2048, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(5, V, (B, S), device="cuda", generator=g)
    seg = (torch.arange(S, device="cuda")[None, :] >= torch.tensor(lens, device="cuda")[:, None] // 2).long()
    mask = (torch.arange(S, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]).long()
    if holes:
        mask[0, 3:9] = 0
        mask[-1, 1::3] = 0
    return ids, seg, mask


def _grads(arena):
    return {s.name: arena.grad(s.name).float().clone() for s in arena.slots}


def test_engine_eval_and_gradients_match_padded_engine():
    from bert_pytorch_b200.models.fused import pack_rows
    model, arena = _model()
    eng = model.fused_engine()
    B, S = 6, 384
    lens = [384, 17, 200, 64, 129, 1]
    ids, seg, mask = _batch(B, S, lens)
    valid = mask.view(-1).bool()
    model.eval()
    ref, _ = eng.forward(ids, seg, mask, training=False)
    pk = pack_rows(mask)
    got, _ = eng.forward(ids, seg, mask, training=False, pack=pk)
    assert torch.equal(got, ref[valid])
    model.unpad = True
    with torch.no_grad():
        enc = model(ids, seg, mask)[0][-1].view(B * S, -1)
    assert torch.equal(enc[valid], ref[valid].float()) and not enc[~valid].any()
    model.unpad = False

    d_out = ((torch.randn(B * S, 1024, device="cuda") * 0.1).bfloat16() * mask.view(-1, 1).bfloat16()).contiguous()
    model.train()
    for ckpt in (False, True):
        model.checkpoint_activations(ckpt)
        res = []
        for pack in (None, pk):
            arena.zero_grad()
            seq, sv = eng.forward(ids, seg, mask, training=True, seed=11, dropout=False, pack=pack)
            eng.backward(sv, d_out if pack is None else d_out[valid].contiguous())
            torch.cuda.synchronize()
            res.append(_grads(arena))
        bad = []
        for name, r in res[0].items():
            if "pooler" in name or name.endswith("attention.self.key.bias"):   # no gradient / softmax-invariant noise
                continue
            c = _cos(res[1][name], r)
            if not c >= 0.99999:
                bad.append((name, c))
        assert not bad, (ckpt, bad)
    model.checkpoint_activations(False)


def _mask_t(seed, stream, shape, p):
    from bert_pytorch_b200.utils import philox
    n = int(np.prod(shape))
    keep = torch.from_numpy(philox.keep_mask(seed, stream, n, p)).cuda().view(*shape)
    return keep.float() * philox.keep_scale(p)


def _oracle_packed(P, ids, seg, pk, B, S, heads, p, seed, d_out):
    """fp32 embeddings + one post-LN layer on the packed rows, fed the kernels' dropout masks (packed-row counters for
    the hidden sites, in-sequence positions for the attention probabilities)."""
    H = P["embeddings.word_embeddings.weight"].size(1)
    T, pre, d = pk.T, "encoder.layer.0.", 64
    e = P["embeddings.word_embeddings.weight"][ids] + P["embeddings.position_embeddings.weight"][pk.pos_ids.long()] \
        + P["embeddings.token_type_embeddings.weight"][seg]
    e = e + (e.bfloat16().float() - e).detach()
    x = F.layer_norm(e, (H,), P["embeddings.LayerNorm.weight"], P["embeddings.LayerNorm.bias"], 1e-12)
    x = x * _mask_t(seed, 1023 * 8 + 0, (T, H), p)
    qkv_w = torch.cat([P[pre + f"attention.self.{n}.weight"] for n in ("query", "key", "value")], 0)
    qkv_b = torch.cat([P[pre + f"attention.self.{n}.bias"] for n in ("query", "key", "value")], 0)
    qkv = x @ qkv_w.t() + qkv_b
    pmask = _mask_t(seed, 0 * 8 + 1, (B, heads, S, S), p)
    cu = pk.cu_seqlens.tolist()
    ctx = []
    for b in range(B):
        n = cu[b + 1] - cu[b]
        q, k, v = (t.view(n, heads, d).transpose(0, 1) for t in qkv[cu[b]:cu[b + 1]].split(H, dim=1))
        probs = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), -1) * pmask[b, :, :n, :n]
        ctx.append((probs @ v).transpose(0, 1).reshape(n, H))
    ctx = torch.cat(ctx)
    a = ctx @ P[pre + "attention.output.dense.weight"].t() + P[pre + "attention.output.dense.bias"]
    x1 = F.layer_norm(a * _mask_t(seed, 2, (T, H), p) + x, (H,), P[pre + "attention.output.LayerNorm.weight"],
                      P[pre + "attention.output.LayerNorm.bias"], 1e-12)
    h = F.gelu(x1 @ P[pre + "intermediate.dense_act.weight"].t() + P[pre + "intermediate.dense_act.bias"])
    o = h @ P[pre + "output.dense.weight"].t() + P[pre + "output.dense.bias"]
    x2 = F.layer_norm(o * _mask_t(seed, 3, (T, H), p) + x1, (H,), P[pre + "output.LayerNorm.weight"],
                      P[pre + "output.LayerNorm.bias"], 1e-12)
    x2.backward(d_out.float())
    return x2.detach()


@pytest.mark.parametrize("holes", [False, True])
def test_engine_with_dropout_matches_fp32_oracle(holes):
    from bert_pytorch_b200.models.fused import pack_rows
    P_DROP, SEED = 0.1, 0x5EED1234ABC
    model, arena = _model(layers=1, p_drop=P_DROP, S=256)
    eng = model.fused_engine()
    B, S = 8, 256
    ids, seg, mask = _batch(B, S, [256, 33, 128, 129, 1, 200, 64, 250], holes=holes)
    pk = pack_rows(mask)
    rows = pk.rows.long()
    d_out = ((torch.randn(pk.T, 1024, device="cuda") * 0.1).bfloat16()).contiguous()
    params = {s.name: (arena.shadow(s.name).float() if "LayerNorm" not in s.name else arena.view(s.name).clone()
                       ).requires_grad_(True) for s in arena.slots}
    model.train()
    arena.zero_grad()
    seq, sv = eng.forward(ids, seg, mask, training=True, seed=SEED, dropout=True, pack=pk)
    eng.backward(sv, d_out)
    torch.cuda.synchronize()
    ref_out = _oracle_packed(params, ids.view(-1)[rows], seg.view(-1)[rows], pk, B, S, 16, P_DROP, SEED, d_out)
    assert ((seq.float() - ref_out).norm() / ref_out.norm()).item() < 1e-2
    bad = []
    for name, t in params.items():
        if t.grad is None or "pooler" in name:
            continue
        g, g_ref = arena.grad(name).float(), t.grad
        if name.endswith("attention.self.key.bias"):
            qn = params[name.replace("key.bias", "query.bias")].grad.norm().item()
            assert g.norm().item() <= 2e-2 * qn and g_ref.norm().item() <= 2e-2 * qn
            continue
        cos = _cos(g, g_ref)
        rel = ((g - g_ref).norm() / g_ref.norm().clamp_min(1e-12)).item()
        if not (cos >= 0.9995 and rel <= 1e-2):
            bad.append((name, round(cos, 6), round(rel, 5)))
    assert not bad, bad

    if holes:                                           # a mask with holes: the plain PyTorch path agrees (eval)
        model.eval()
        with torch.no_grad():
            model.unpad = True
            got = model(ids, seg, mask)[0][-1]
            model.use_fused = False
            ref = model(ids, seg, mask)[0][-1]
        model.use_fused, model.unpad = True, False
        v = mask.bool()
        assert _cos(got[v], ref[v]) >= 0.9995
        assert ((got[v] - ref[v]).norm() / ref[v].norm()).item() <= 1e-2
        assert not got[~v].any()


# ------------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------------
def test_token_classification_unpadded_matches_padded():
    from bert_pytorch_b200.models import BertForTokenClassification
    model, arena = _model(BertForTokenClassification, num_labels=9)
    B, S = 32, 512
    g = torch.Generator().manual_seed(3)
    lens = (torch.randint(8, 60, (B,), generator=g)).tolist()
    ids, seg, mask = _batch(B, S, lens)
    labels = torch.randint(0, 9, (B, S), device="cuda")
    model.train()
    out = []
    for unpad in (False, True):
        model.bert.unpad = unpad
        arena.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = model(ids, torch.zeros_like(mask), mask, labels=labels)
        loss.backward()
        torch.cuda.synchronize()
        out.append((loss.item(), _grads(arena)))
    assert abs(out[0][0] - out[1][0]) <= 1e-4 * abs(out[0][0])
    bad = [(n, _cos(out[1][1][n], r)) for n, r in out[0][1].items()
           if "pooler" not in n and not n.endswith("attention.self.key.bias") and r.abs().max() > 0
           and not _cos(out[1][1][n], r) >= 0.9999]
    assert not bad, bad


@pytest.mark.parametrize("B", [8, 48])
def test_question_answering_prediction_unpadded_matches_padded(B):
    from bert_pytorch_b200.models import BertForQuestionAnswering
    model, _ = _model(BertForQuestionAnswering, S=384)
    S = 384
    g = torch.Generator().manual_seed(B)
    lens = torch.randint(40, S + 1, (B,), generator=g).tolist()
    ids, seg, mask = _batch(B, S, lens)
    model.eval()
    res = []
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for unpad in (False, True):
            model.bert.unpad = unpad
            res.append([t.float() for t in model(ids, seg, mask)])
    v = mask.bool()
    for r, t in zip(*res):
        assert torch.allclose(t[v], r[v], rtol=0, atol=2e-2 * r[v].abs().max().item()), (t[v] - r[v]).abs().max().item()


def test_empty_batch_returns_zeros():
    model, _ = _model(layers=1, S=128)
    model.eval()
    model.unpad = True
    ids, seg, mask = _batch(2, 128, [0, 0])
    with torch.no_grad():
        out = model(ids, seg, mask)[0][-1]
    assert out.shape == (2, 128, 1024) and not out.any()
