"""The one-pass attention backward (S <= 128: attn_bwd_onepass_kernel) against the general multi-block path
(attn_delta_kernel, attn_bwd_kernel, attn_dq_convert_kernel) on the same inputs: dqkv and its fp8 copy are bitwise
equal, padded and packed, with and without dropout, for sequence lengths at every query-block edge, a length-1
sequence, a fully masked row (padded) and an empty sequence (packed).  The QKV bias gradient that ``dbias=`` adds
equals the column sums of dqkv up to fp32 reordering, and in deterministic mode it is the fixed-order column sum
exactly."""
import pytest
import torch

pytestmark = pytest.mark.gpu

HEADS, H = 2, 128
SEED = 0x5EED1234


def _api():
    from bert_pytorch_b200.ops import api
    return api


def _lengths(S):
    """per-sequence lengths: 1, both sides of the 64-query block edge, 127, S, a fully masked row (0) and a few more"""
    return [1, 63, 64, 65, 127, S, 0, 5, S - 1, 40]


def _case(S, form, p_drop, seed=1):
    K = _api()
    g = torch.Generator(device="cuda").manual_seed(1000 * S + seed)
    lens = _lengths(S)
    B = len(lens)
    qkv = (torch.randn(B, S, 3 * H, device="cuda", generator=g) * 0.5).bfloat16()
    dctx = (torch.randn(B, S, H, device="cuda", generator=g) * 0.5).bfloat16()
    kw = dict(p_drop=p_drop, seed=SEED, stream=5)
    if form == "padded":
        seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
        ctx, lse = K.attention_fwd(qkv, seqlens, HEADS, **kw)
        args = (qkv, seqlens, ctx, dctx, lse, HEADS)
    else:
        n = [min(max(x, 0), S) for x in lens]                 # the 0 entry is an empty sequence here
        rows = torch.cat([torch.arange(b * S, b * S + n[b], device="cuda") for b in range(B)])
        pq, pd = qkv.view(B * S, -1)[rows].contiguous(), dctx.view(B * S, -1)[rows].contiguous()
        cu = torch.tensor([0] + torch.tensor(n).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
        ctx, lse = K.attention_fwd(pq, None, HEADS, cu_seqlens=cu, S=S, **kw)
        args = (pq, None, ctx, pd, lse, HEADS)
        kw.update(cu_seqlens=cu, S=S)
    return args, kw


def _fp8(K):
    meta = K.Fp8Meta(["dqkv"], [True], torch.device("cuda"))
    meta.record("dqkv")[:] = torch.tensor([0.0, 1.0, 1.0, 0.0])
    return meta


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.uint8)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("form", ["padded", "varlen"])
@pytest.mark.parametrize("S", [8, 64, 120, 128])
def test_onepass_matches_the_general_path_bitwise(S, form, p_drop, fp8):
    if fp8 and form == "varlen":
        pytest.skip("the varlen form writes no fp8 side output")
    K = _api()
    args, kw = _case(S, form, p_drop)
    if fp8:
        m1, m2 = _fp8(K), _fp8(K)
        one, q1 = K.attention_bwd(*args, fp8=(m1, "dqkv"), **kw)
        gen, q2 = K.attention_bwd(*args, fp8=(m2, "dqkv"), _general=True, **kw)
        torch.cuda.synchronize()
        assert torch.equal(_bits(q1), _bits(q2)), "fp8 copy of dqkv"
        assert torch.equal(m1.record("dqkv")[0], m2.record("dqkv")[0]), "amax of dqkv"
    else:
        one = K.attention_bwd(*args, **kw)
        gen = K.attention_bwd(*args, _general=True, **kw)
        torch.cuda.synchronize()
    diff = (_bits(one) != _bits(gen)).nonzero()
    assert diff.numel() == 0, f"{diff.size(0)} elements differ, first at {diff[0].tolist()}"


@pytest.mark.parametrize("form", ["padded", "varlen"])
@pytest.mark.parametrize("S", [8, 64, 120, 128])
def test_onepass_bias_gradient_is_the_column_sum(S, form):
    K = _api()
    args, kw = _case(S, form, 0.1, seed=2)
    dbias = torch.full((3 * H,), 0.25, dtype=torch.float32, device="cuda")     # accumulates onto what is there
    dqkv = K.attention_bwd(*args, dbias=dbias, **kw)
    torch.cuda.synchronize()
    x = dqkv.reshape(-1, 3 * H).double()
    ref = 0.25 + x.sum(0)
    bound = 1e-6 * x.abs().sum(0) + 1e-7
    err = (dbias.double() - ref).abs()
    assert bool((err <= bound).all()), f"worst error / bound {(err / bound).max().item():.3g}"
    assert torch.equal(dqkv, K.attention_bwd(*args, **kw)), "dbias changed dqkv"


@pytest.mark.parametrize("form", ["padded", "varlen"])
@pytest.mark.parametrize("S", [64, 128])
def test_onepass_bias_gradient_in_deterministic_mode_is_colsum(S, form, monkeypatch):
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    K = _api()
    assert K.deterministic()
    args, kw = _case(S, form, 0.1, seed=3)
    dbias = torch.full((3 * H,), 0.25, dtype=torch.float32, device="cuda")
    dqkv = K.attention_bwd(*args, dbias=dbias, **kw)
    ref = torch.full_like(dbias, 0.25)
    K.colsum_accumulate(dqkv.reshape(-1, 3 * H), ref)
    torch.cuda.synchronize()
    assert torch.equal(dbias, ref)
    assert torch.equal(dqkv, K.attention_bwd(*args, _general=True, **kw))


def test_general_path_takes_the_bias_gradient():
    """S > 128 runs the multi-block path; dbias gets the column sums of its dqkv as well"""
    K = _api()
    g = torch.Generator(device="cuda").manual_seed(7)
    B, S = 3, 256
    qkv = (torch.randn(B, S, 3 * H, device="cuda", generator=g) * 0.5).bfloat16()
    dctx = (torch.randn(B, S, H, device="cuda", generator=g) * 0.5).bfloat16()
    seqlens = torch.tensor([S, 200, 129], dtype=torch.int32, device="cuda")
    ctx, lse = K.attention_fwd(qkv, seqlens, HEADS)
    dbias = torch.zeros(3 * H, dtype=torch.float32, device="cuda")
    dqkv = K.attention_bwd(qkv, seqlens, ctx, dctx, lse, HEADS, dbias=dbias)
    ref = torch.zeros_like(dbias)
    K.colsum_accumulate(dqkv.reshape(-1, 3 * H), ref)
    torch.cuda.synchronize()
    x = dqkv.reshape(-1, 3 * H).double()
    assert bool(((dbias.double() - ref.double()).abs() <= 1e-6 * x.abs().sum(0) + 1e-7).all())
