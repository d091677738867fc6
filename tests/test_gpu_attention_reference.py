"""Fused attention (ops/csrc/attention_sm90.cu) against an fp64 reference of the same operation, forward and backward,
under the kernels' own Philox dropout masks (utils/philox.py), in the padded and the varlen form.

The reference reads exactly the bf16 qkv and dctx the kernels read, and its keep decisions are the host evaluation of
the kernels' Philox stream: element ((b * heads + head) * S + q) * S + k, kept iff its 16 bits >= round(p * 65536), a
kept probability scaled by philox.keep_scale(p).  With P = softmax of the scaled scores over the valid keys and
P~ = P * keep * inv_keep:

    ctx = P~ V                 lse = natural-log LSE of the scaled scores (before dropout)
    delta = <dO, ctx>          (ctx: the kernel's bf16 output, which is what the kernel's backward reads)
    dV = P~^T dO               dP = (dO V^T) * keep * inv_keep          dS = P * (dP - delta)
    dQ = scale dS K            dK = scale dS^T Q

The valid keys of sequence b are its first min(seqlens[b], S); a sequence of length 0 (an all-zero attention-mask row)
attends to all S keys, as the model's additive -10000 mask does.  Every query row of the padded form is computed.

Error bound per output: |out - ref| <= c E + R |ref| elementwise and ||out - ref|| / ||ref|| <= eps, where E is the
same chain on absolute values (|P~| |V| for ctx, |P~|^T |dO| for dV, scale (P * (keep inv_keep |dO| |V|^T + |delta|))
|K| for dQ and the same with |Q| for dK) and R = 2^-8 is the rounding of the bf16 output.  Where E is zero (keys
past the sequence, for instance) the output must be exactly zero."""
import math

import numpy as np
import pytest
import torch

from bert_pytorch_b200.utils import philox

HD = 64
SCALE = 1.0 / math.sqrt(HD)
R = 2.0 ** -8                      # unit roundoff of a bf16 output
# Measured on an H100 SXM (80 GB HBM3, 700 W power limit) over every case of this file, worst (c, eps):
# ctx (3.5e-3, 2.9e-3), dQ (2.5e-3, 6.2e-3), dK (1.8e-3, 2.6e-3), dV (3.3e-3, 2.6e-3); lse 5.2e-6 absolute.  c comes
# from rounding P~ and dS to bf16 for the tensor-core products (at most 2^-8 of E); eps is mostly the bf16 rounding of
# the outputs, except for dQ of rows whose probability mass sits in one key block, where dS cancels.  Each bound is
# 2.5-4x its measured worst case.
C_BOUND = {"ctx": 1e-2, "dq": 8e-3, "dk": 6e-3, "dv": 1e-2}
EPS_BOUND = {"ctx": 8e-3, "dq": 1.6e-2, "dk": 8e-3, "dv": 8e-3}
LSE_BOUND = 2e-5
SEED = 0x3A5C9E3779B9              # 46 bits: the high word of the Philox key is not zero, as for the engine's seeds
STREAMS = (1, 9, 185)              # layer * 8 + 1: the engine's attention-probability streams (layers 0, 1 and 23)
SEQ = (64, 128, 136, 200, 256, 384, 504, 512)
WORST = {}


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
def key_lengths(lens, S):
    """The kernels' valid key count per sequence: clamped to S, and 0 (a fully masked sequence) means all S keys."""
    return [S if n <= 0 else min(n, S) for n in lens]


_M32 = 0xFFFFFFFF


def keep_mask_torch(seed, stream, numel, p_drop, device):
    """philox.keep_mask on ``device`` in int64 tensor arithmetic (a 32 x 32-bit product wraps modulo 2^64, so its low and
    high words come out right), for the sites of 10^7 - 10^8 elements that the big cases need."""
    if p_drop <= 0.0:
        return torch.ones(numel, dtype=torch.bool, device=device)
    groups = (numel + 7) // 8
    x = torch.arange(groups, dtype=torch.int64, device=device)
    y = torch.zeros_like(x)
    z = torch.full_like(x, stream & _M32)
    w = torch.full_like(x, 0x5EED)
    k0, k1 = seed & _M32, (seed >> 32) & _M32
    for _ in range(7):
        p0, p1 = x * 0xD2511F53, z * 0xCD9E8D57
        x, z = ((p1 >> 32) & _M32) ^ y ^ k0, ((p0 >> 32) & _M32) ^ w ^ k1
        y, w = p1 & _M32, p0 & _M32
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    words = torch.stack([x, y, z, w], dim=-1)                                   # [G, 4]
    fields = torch.stack([words & 0xFFFF, words >> 16], dim=-1).reshape(-1)     # element t: word t // 2, low half first
    return (fields >= int(p_drop * 65536.0 + 0.5))[:numel]


def keep_tensor(B, heads, S, p_drop, seed, stream, device):
    """[B, heads, S, S] fp64 keep * inv_keep of the attention-probability dropout site."""
    keep = keep_mask_torch(seed, stream, B * heads * S * S, p_drop, device)
    return keep.view(B, heads, S, S).double() * philox.keep_scale(p_drop)


def _heads(t, B, S, heads):
    return t.double().view(B, S, heads, HD).transpose(1, 2)          # [B, h, S, d]


def _merge(t):
    B, h, S, d = t.shape
    return t.transpose(1, 2).reshape(B, S, h * d)


def attention_ref(qkv, dctx, ctx_k, lens, heads, p_drop, seed, stream):
    """fp64 forward and backward of the padded form.  qkv [B, S, 3H], dctx [B, S, H], ctx_k: the ctx the backward reads
    (for delta).  Returns {name: (ref, E)} for ctx [B, S, H], dqkv [B, S, 3H], and lse [B, h, S] (E None)."""
    B, S, H3 = qkv.shape
    H = H3 // 3
    q, k, v = (_heads(t, B, S, heads) for t in qkv.split(H, dim=-1))
    do = _heads(dctx, B, S, heads)
    n = torch.tensor(key_lengths(lens, S), device=qkv.device)
    valid = (torch.arange(S, device=qkv.device)[None, :] < n[:, None])[:, None, None, :]
    s = (q @ k.transpose(-1, -2)) * SCALE
    s = s.masked_fill(~valid, -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    P = torch.exp(s - lse[..., None])
    del s
    ks = keep_tensor(B, heads, S, p_drop, seed, stream, qkv.device)
    Pt = P * ks
    ctx = _merge(Pt @ v)
    ctx_E = _merge(Pt.abs() @ v.abs())
    delta = (do * _heads(ctx_k, B, S, heads)).sum(-1, keepdim=True)
    dv, dv_E = Pt.transpose(-1, -2) @ do, Pt.abs().transpose(-1, -2) @ do.abs()
    del Pt
    dS = P * ((do @ v.transpose(-1, -2)) * ks - delta)
    dq, dk = SCALE * (dS @ k), SCALE * (dS.transpose(-1, -2) @ q)
    del dS
    dS_E = P * (ks * (do.abs() @ v.abs().transpose(-1, -2)) + delta.abs())
    dq_E, dk_E = SCALE * (dS_E @ k.abs()), SCALE * (dS_E.transpose(-1, -2) @ q.abs())
    del dS_E, P, ks
    dqkv = torch.cat([_merge(dq), _merge(dk), _merge(dv)], dim=-1)
    dqkv_E = torch.cat([_merge(dq_E), _merge(dk_E), _merge(dv_E)], dim=-1)
    return {"ctx": (ctx, ctx_E), "lse": (lse, None), "dqkv": (dqkv, dqkv_E)}


# ---------------------------------------------------------------------------------------------------------------------
# reference self-checks (CPU): the formulas against autograd of softmax attention, the masks against Philox itself
# ---------------------------------------------------------------------------------------------------------------------
def _autograd_attention(qkv, dctx, lens, heads, keep):
    B, S, H3 = qkv.shape
    H = H3 // 3
    leaf = qkv.double().clone().requires_grad_(True)
    q, k, v = (_heads(t, B, S, heads) for t in leaf.split(H, dim=-1))
    n = torch.tensor(key_lengths(lens, S))
    scores = (q @ k.transpose(-1, -2)) / math.sqrt(HD)
    scores = scores.masked_fill(~(torch.arange(S)[None, :] < n[:, None])[:, None, None, :], -math.inf)
    ctx = _merge((torch.softmax(scores, dim=-1) * keep) @ v)
    ctx.backward(dctx.double())
    return ctx.detach(), torch.logsumexp(scores, -1).detach(), leaf.grad


@pytest.mark.parametrize("p_drop", [0.0, 0.5])
def test_reference_matches_autograd_softmax_attention(p_drop):
    torch.manual_seed(0)
    B, S, heads = 4, 24, 2
    lens = [24, 5, 0, 40]
    qkv = torch.randn(B, S, 3 * heads * HD).bfloat16()
    dctx = torch.randn(B, S, heads * HD).bfloat16()
    keep = keep_tensor(B, heads, S, p_drop, SEED, 9, "cpu")
    ctx, lse, grad = _autograd_attention(qkv, dctx, lens, heads, keep)
    ref = attention_ref(qkv, dctx, ctx, lens, heads, p_drop, SEED, 9)
    assert torch.allclose(ref["ctx"][0], ctx, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["lse"][0], lse, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["dqkv"][0], grad, rtol=1e-10, atol=1e-12)
    # the 0-length sequence attends to all S keys: its lse is finite, and its keys get gradients
    assert torch.isfinite(ref["lse"][0]).all() and ref["dqkv"][0][2].abs().sum() > 0
    assert (ref["dqkv"][0][1, 5:, heads * HD:] == 0).all()          # keys past a sequence: exactly zero dK / dV
    for t, e in (ref["ctx"], ref["dqkv"]):
        assert ((t.abs() <= e * (1 + 1e-12)) | (e == 0) & (t == 0)).all()


def test_reference_keep_mask_is_the_kernels_element_indexing():
    """Each keep decision re-derived from one Philox draw: group e >> 3 of element e, 32-bit word (e & 7) >> 1, half
    e & 1 -- at the corners of a [B, h, S, S] site and beyond 2^32 bits."""
    B, heads, S, p = 3, 16, 504, 0.5
    keep = keep_tensor(B, heads, S, p, SEED, 185, "cpu") > 0
    thresh = int(p * 65536 + 0.5)
    pts = [(0, 0, 0, 0), (0, 0, 0, 7), (0, 0, 1, 0), (1, 3, 200, 131), (2, 15, 503, 503), (2, 15, 503, 496),
           (1, 0, 0, 503), (2, 7, 77, 1)]
    for b, h, q, k in pts:
        e = ((b * heads + h) * S + q) * S + k
        word = philox.philox4x32_7(SEED, np.array([e >> 3], dtype=np.uint64), 185)[0, (e & 7) >> 1]
        bits = (int(word) >> (16 * (e & 1))) & 0xFFFF
        assert bool(keep[b, h, q, k]) == (bits >= thresh), (b, h, q, k)
    assert 0.45 < keep.double().mean().item() < 0.55


@pytest.mark.parametrize("p_drop", [0.1, 0.5])
def test_torch_keep_mask_matches_host_philox(p_drop):
    n = 1 << 16
    for seed, stream in ((SEED, 185), ((1 << 47) - 1, 1), (12345, 9)):
        want = philox.keep_mask(seed, stream, n, p_drop)
        assert np.array_equal(keep_mask_torch(seed, stream, n, p_drop, "cpu").numpy(), want), (seed, stream)


# ---------------------------------------------------------------------------------------------------------------------
# kernels against the reference (GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _check(out, ref, E, name, tag, fails, rows=None):
    """Elementwise |out - ref| <= c E + R |ref| and relative L2 eps, over ``rows`` (bool, broadcastable) if given; a
    failure is appended to ``fails``, so that one case reports every output that is off."""
    out = out.double()
    if rows is not None:
        out, ref, E = out[rows], ref[rows], E[rows]
    if not torch.isfinite(out).all():
        fails.append((name, "non-finite", int((~torch.isfinite(out)).sum())))
        return
    err = (out - ref).abs()
    slack = err - R * ref.abs()
    pos = E > 0
    if not (slack[~pos] <= 0).all():
        fails.append((name, "non-zero where the reference is exactly zero", int((slack[~pos] > 0).sum())))
    c = (slack[pos] / E[pos]).max().clamp_min(0).item() if pos.any() else 0.0
    eps = ((out - ref).norm() / ref.norm().clamp_min(1e-300)).item()
    w = WORST.setdefault(name, [0.0, 0.0])
    w[0], w[1] = max(w[0], c), max(w[1], eps)
    print(f"[attn ref] {tag} {name}: c = {c:.3e}, eps = {eps:.3e}  (worst so far {w[0]:.3e}, {w[1]:.3e})")
    if not (c <= C_BOUND[name] and eps <= EPS_BOUND[name]):
        fails.append((name, c, eps))


def _check_lse(lse, ref, tag, fails, rows=None):
    if rows is not None:
        lse, ref = lse[rows], ref[rows]
    if not torch.isfinite(lse).all():
        fails.append(("lse", "non-finite", int((~torch.isfinite(lse)).sum())))
        return
    err = (lse.double() - ref).abs().max().item()
    w = WORST.setdefault("lse", [0.0, 0.0])
    w[0] = max(w[0], err)
    print(f"[attn ref] {tag} lse: max abs err = {err:.3e}  (worst so far {w[0]:.3e})")
    if not err <= LSE_BOUND:
        fails.append(("lse", err))


def _check_all(K, qkv, dctx, lens, heads, p, stream, tag):
    """Padded kernels against the reference: every query row of every sequence."""
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kw = dict(p_drop=p, seed=SEED, stream=stream)
    ctx, lse = K.attention_fwd(qkv, seqlens, heads, **kw)
    dqkv = K.attention_bwd(qkv, seqlens, ctx, dctx, lse, heads, **kw)
    torch.cuda.synchronize()
    ref = attention_ref(qkv, dctx, ctx, lens, heads, p, SEED, stream)
    H = qkv.size(-1) // 3
    fails = []
    _check(ctx, *ref["ctx"], "ctx", tag, fails)
    _check_lse(lse, ref["lse"][0], tag, fails)
    for i, name in enumerate(("dq", "dk", "dv")):
        sl = slice(i * H, (i + 1) * H)
        _check(dqkv[..., sl], ref["dqkv"][0][..., sl], ref["dqkv"][1][..., sl], name, tag, fails)
    assert not fails, (tag, fails)
    return ctx, ref


def _lens(S):
    """1, 7, 63-65, 127-129, S - 1, S, a length above S (the kernels clamp it) and 0 (a fully masked sequence)."""
    base = sorted({n for n in (1, 7, 63, 64, 65, 127, 128, 129, S - 1, S) if n <= S})
    return base + [S + 24, 0]


def _inputs(family, B, S, H, lens, g):
    """qkv and dctx [bf16] of an input family.  'n0.5' / 'n2': N(0, sigma^2) (sigma 2: logits of tens);  'last': every
    row's largest scores lie in the last key block of its sequence, so the online softmax rescales by alpha << 1."""
    sigma = {"n0.5": 0.5, "n2": 2.0, "last": 0.5}[family]
    qkv = torch.randn(B, S, 3 * H, device="cuda", generator=g) * sigma
    if family == "last":
        u = torch.full((HD,), 12.0 / 8.0, device="cuda").repeat(H // HD)        # 12 u, |u| = 1, in every head
        qkv[..., :H] += u
        for b, n in enumerate(key_lengths(lens, S)):
            k0 = (n - 1) // 128 * 128
            qkv[b, k0:n, H:2 * H] += u                 # about +18 on the scaled scores of the last block's keys
    dctx = torch.randn(B, S, H, device="cuda", generator=g) * 0.5
    return qkv.bfloat16(), dctx.bfloat16()


FAMILIES = ("n0.5", "n2", "last")


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 2, 16])
@pytest.mark.parametrize("p_drop", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("S", SEQ)
def test_attention_matches_fp64_reference(S, p_drop, heads):
    K = _api()
    i = SEQ.index(S) + (0.0, 0.1, 0.5).index(p_drop) + (1, 2, 16).index(heads)
    family, stream = FAMILIES[i % 3], STREAMS[i % 3]
    g = torch.Generator(device="cuda").manual_seed(1000 * S + 10 * heads + int(p_drop * 10))
    lens = _lens(S)
    qkv, dctx = _inputs(family, len(lens), S, heads * HD, lens, g)
    _check_all(K, qkv, dctx, lens, heads, p_drop, stream, f"S={S} p={p_drop} h={heads} {family}")


def _bert_batch(S):
    """B * heads * S^2 = 2^25 (the fp64 reference stays near 3 GB): many waves of CTAs, and at S = 128 and 512 the
    BERT-large pre-training shapes of phase 1 and phase 2 (16 heads)."""
    return max(1, (1 << 25) // (16 * S * S))


@pytest.mark.gpu
@pytest.mark.parametrize("S", SEQ)
def test_attention_matches_fp64_reference_many_waves(S):
    K = _api()
    B, heads = _bert_batch(S), 16
    g = torch.Generator(device="cuda").manual_seed(S)
    lens = torch.randint(1, S + 1, (B,), device="cuda", generator=g).tolist()
    lens[0] = S
    qkv, dctx = _inputs("n0.5", B, S, heads * HD, lens, g)
    _check_all(K, qkv, dctx, lens, heads, 0.1, 185, f"S={S} B={B} h=16 p=0.1")


@pytest.mark.gpu
@pytest.mark.parametrize("p_drop", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("S", SEQ)
def test_attention_uniform_probabilities_exact(S, p_drop):
    """Q = 0: every probability is 1 / n, P~ = bf16(inv_keep) on kept keys, and with V small integers the forward is
    exact up to the division by l and the bf16 store: ctx must be within one bf16 ulp of
    bf16(inv_keep) * sum(kept v) / n.  One wrong keep decision moves a row by at least 1 / n."""
    K = _api()
    heads, H = 2, 128
    lens = _lens(S)
    B = len(lens)
    stream = STREAMS[SEQ.index(S) % 3]
    g = torch.Generator(device="cuda").manual_seed(S + 7)
    qkv = torch.randn(B, S, 3 * H, device="cuda", generator=g) * 0.5
    qkv[..., :H] = 0.0
    mag = torch.randint(1, 4, (B, S, H), device="cuda", generator=g).float()
    sign = torch.randint(0, 2, (B, S, H), device="cuda", generator=g).float() * 2 - 1
    qkv[..., 2 * H:] = mag * sign
    qkv = qkv.bfloat16()
    dctx = (torch.randn(B, S, H, device="cuda", generator=g) * 0.5).bfloat16()
    tag = f"Q=0 S={S} p={p_drop}"
    ctx, ref = _check_all(K, qkv, dctx, lens, heads, p_drop, stream, tag)

    inv_keep_bf16 = float(torch.tensor(philox.keep_scale(p_drop)).bfloat16())
    keep = keep_tensor(B, heads, S, p_drop, SEED, stream, "cuda") > 0
    n = torch.tensor(key_lengths(lens, S), device="cuda")
    valid = (torch.arange(S, device="cuda")[None, :] < n[:, None])[:, None, None, :]
    v = _heads(qkv[..., 2 * H:], B, S, heads)
    exact = _merge(((keep & valid).double() @ v) * inv_keep_bf16 / n.double()[:, None, None, None])
    ulp = torch.where(exact == 0, torch.zeros_like(exact), torch.exp2(torch.floor(torch.log2(exact.abs())) - 7))
    bad = (ctx.double() - exact).abs() > ulp
    assert not bad.any(), (tag, int(bad.sum()), bad.nonzero()[:4].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("S", [128, 200])
def test_fully_masked_sequence_attends_to_every_key(S, p_drop):
    """seqlens[b] == 0 (an all-zero attention-mask row): every key is valid, as under the model's additive mask, and
    lse, ctx and all three gradients are finite and equal the full-length reference."""
    K = _api()
    heads, H = 2, 128
    lens = [0, S // 2, 0]
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv, dctx = _inputs("n0.5", len(lens), S, H, lens, g)
    ctx, _ = _check_all(K, qkv, dctx, lens, heads, p_drop, 9, f"len 0 S={S} p={p_drop}")
    full, _ = K.attention_fwd(qkv, torch.tensor([S, S // 2, S], dtype=torch.int32, device="cuda"), heads,
                              p_drop=p_drop, seed=SEED, stream=9)
    assert torch.equal(ctx, full)


def _varlen_lens(S):
    return [n for n in (1, 64, 65, 128, 129, S) if n <= S]


@pytest.mark.gpu
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("S", [128, 200, 512])
def test_varlen_attention_matches_fp64_reference(S, p_drop):
    """The varlen kernels on packed rows against the same reference per sequence (its padding query rows get a zero
    dO, so they add nothing to dK / dV)."""
    K = _api()
    from bert_pytorch_b200.models.fused import pack_rows
    heads, H = 2, 128
    lens = _varlen_lens(S)
    B = len(lens)
    mask = (torch.arange(S, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None])
    pk = pack_rows(mask.long())
    rows = pk.rows.long()
    g = torch.Generator(device="cuda").manual_seed(S + 3)
    qkv, dctx = _inputs("n0.5", B, S, H, lens, g)
    dctx = dctx * mask[..., None].bfloat16()
    kw = dict(p_drop=p_drop, seed=SEED, stream=185, cu_seqlens=pk.cu_seqlens, S=S)
    qkv_p = qkv.view(B * S, 3 * H)[rows].contiguous()
    ctx_p, lse = K.attention_fwd(qkv_p, None, heads, **kw)
    dqkv_p = K.attention_bwd(qkv_p, None, ctx_p, dctx.view(B * S, H)[rows].contiguous(), lse, heads, **kw)
    torch.cuda.synchronize()
    ctx = torch.zeros(B * S, H, dtype=torch.bfloat16, device="cuda")
    ctx[rows] = ctx_p
    ref = attention_ref(qkv, dctx, ctx.view(B, S, H), lens, heads, p_drop, SEED, 185)
    tag = f"varlen S={S} p={p_drop}"
    flat = {k: (r.reshape(B * S, -1)[rows], None if e is None else e.reshape(B * S, -1)[rows])
            for k, (r, e) in ref.items() if k != "lse"}
    fails = []
    _check(ctx_p, *flat["ctx"], "ctx", tag, fails)
    _check_lse(lse, ref["lse"][0], tag, fails, rows=mask[:, None, :].expand(B, heads, S))
    for i, name in enumerate(("dq", "dk", "dv")):
        sl = slice(i * H, (i + 1) * H)
        _check(dqkv_p[:, sl], flat["dqkv"][0][:, sl], flat["dqkv"][1][:, sl], name, tag, fails)
    assert not fails, (tag, fails)


# ---------------------------------------------------------------------------------------------------------------------
# the engine with an all-zero attention-mask row
# ---------------------------------------------------------------------------------------------------------------------
def _cos(a, b):
    return torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0).item()


@pytest.mark.gpu
def test_engine_with_a_fully_masked_row():
    """A batch whose second row has an all-zero attention mask: the fused eval output matches the PyTorch path (whose
    additive mask makes that row attend to every key), and a training backward gives finite gradients."""
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertModel
    from bert_pytorch_b200.models.arena import ParamArena
    torch.manual_seed(0)
    B, S = 4, 200
    cfg = BertConfig(vocab_size_or_config_json_file=2048, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                     intermediate_size=1024, max_position_embeddings=S)
    model = BertModel(cfg).cuda()
    arena = ParamArena(model)
    ids = torch.randint(5, 2048, (B, S), device="cuda")
    seg = torch.zeros_like(ids)
    mask = (torch.arange(S, device="cuda")[None, :] < torch.tensor([S, 0, 77, 130], device="cuda")[:, None]).long()
    model.eval()
    with torch.no_grad():
        got = model(ids, seg, mask)[0][-1].float().view(B, S, -1)
        model.use_fused = False
        ref = model(ids, seg, mask)[0][-1].float().view(B, S, -1)
        model.use_fused = True
    assert torch.isfinite(got).all()
    for b in range(B):
        rel = ((got[b] - ref[b]).norm() / ref[b].norm()).item()
        assert _cos(got[b], ref[b]) >= 0.9995 and rel <= 1e-2, (b, _cos(got[b], ref[b]), rel)

    eng = model.fused_engine()
    model.train()
    d_out = (torch.randn(B * S, 256, device="cuda") * 0.1).bfloat16()
    for dropout in (False, True):
        arena.zero_grad()
        _, sv = eng.forward(ids, seg, mask, training=True, seed=SEED, dropout=dropout)
        eng.backward(sv, d_out)
        torch.cuda.synchronize()
        bad = [s.name for s in arena.slots if not torch.isfinite(arena.grad(s.name)).all()]
        assert not bad, (dropout, bad)
