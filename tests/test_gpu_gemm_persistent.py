"""Persistent wgmma GEMM: several work units per CTA at the BERT-large shapes, both schedules (128 x 256 cooperative,
128 x 128 ping-pong), every epilogue the fused engine uses, ragged tails, and bitwise replay of the dropout epilogue
(twice eagerly and from a captured CUDA graph) -- against fp32 torch references."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

M = 12288          # phase-1 tokens per micro-step: 96 x 128


def _ops():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)


def _check(out, ref, tol=2e-2):
    out, ref = out.float(), ref.float()
    err = (out - ref).abs().max().item()
    denom = ref.abs().max().item() + 1e-6
    assert err / denom < tol, f"max abs err {err} vs ref scale {denom}"


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("N", [1024, 3072, 4096])
def test_forward_epilogues_many_units(bn, N):
    """EPI_BIAS, EPI_BIAS_GELU_DG (+ aux_out) and EPI_BIAS_DROP_RES (+ mask_in) at M = 12288, K = 1024."""
    K_ = _ops()
    Kd = 1024
    a, b, bias, res = _rand(M, Kd, scale=0.05), _rand(N, Kd, scale=0.05), _rand(N), _rand(M, N)
    x = a.float() @ b.float().t() + bias.float()
    _check(K_.gemm(a, b, epi=K_.EPI_BIAS, bias=bias, block_n=bn), x)
    aux = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    out = K_.gemm(a, b, epi=K_.EPI_BIAS_GELU_DG, bias=bias, aux_out=aux, block_n=bn)
    xd = x.double()
    Phi = 0.5 * (1.0 + torch.erf(xd / math.sqrt(2.0)))
    _check(out, (xd * Phi).float())
    _check(aux, (Phi + xd * torch.exp(-0.5 * xd * xd) / math.sqrt(2.0 * math.pi)).float())
    mask = K_.dropout_mask(M, N, 0.1, 7, 3, "cuda")
    keep = ((mask.unsqueeze(-1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).reshape(M, N).bool()
    out = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, mask_in=mask, block_n=bn)
    _check(out, torch.where(keep, x / 0.9, torch.zeros_like(x)) + res.float())


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("N,Kd", [(4096, 1024), (1024, 4096), (1024, 3072), (1024, 1024)])
def test_dgrad_epilogues_many_units(bn, N, Kd):
    """NN dgrad shapes: EPI_MUL + colsum (FFN-2 dgrad), EPI_ADD (FFN-1 and QKV dgrad), plain (attention-out dgrad)."""
    K_ = _ops()
    a, b, res = _rand(M, Kd, scale=0.05), _rand(Kd, N, scale=0.05), _rand(M, N)
    ref = a.float() @ b.float()
    cs = torch.zeros(N, device="cuda")
    out = K_.gemm(a, b, layout=K_.NN, epi=K_.EPI_MUL, res=res, colsum=cs, block_n=bn)
    _check(out, ref * res.float())
    assert torch.allclose(cs, out.float().sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(M))
    _check(K_.gemm(a, b, layout=K_.NN, epi=K_.EPI_ADD, res=res, block_n=bn), ref + res.float())
    _check(K_.gemm(a, b, layout=K_.NN, block_n=bn), ref)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("N,Kd,splits", [(1024, 4096, 1), (4096, 1024, 2), (1024, 1024, 4), (3072, 1024, -1)])
def test_wgrad_accumulate_split_k(bn, N, Kd, splits):
    """EPI_ACCUM_F32 (TN, reduction over the 12288 tokens) with split-K: several K ranges of a tile on different CTAs."""
    K_ = _ops()
    a, b = _rand(M, N, scale=0.1), _rand(M, Kd, scale=0.1)
    base = torch.randn(N, Kd, device="cuda")
    out = base.clone()
    K_.gemm(a, b, layout=K_.TN, epi=K_.EPI_ACCUM_F32, out=out, block_n=bn, k_splits=splits)
    _check(out, base + a.float().t() @ b.float(), tol=1e-2)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("Mr,N,Kd", [(12290, 1032, 264), (1000, 1000, 520), (129, 136, 72), (17 * 128, 8 * 128, 128)])
def test_ragged_tails_and_uneven_units(bn, Mr, N, Kd):
    """Ragged M/N edges, unit counts that are not a multiple of the grid (and 17 x 8 = 136 units: 4 CTAs take two),
    fewer units than SMs."""
    K_ = _ops()
    a, b, res = _rand(Mr, Kd), _rand(N, Kd), _rand(Mr, N)
    _check(K_.gemm(a, b, epi=K_.EPI_ADD, res=res, block_n=bn), a.float() @ b.float().t() + res.float())
    bn_ = _rand(Kd, N)
    _check(K_.gemm(a, bn_, layout=K_.NN, block_n=bn), a.float() @ bn_.float())


@pytest.mark.parametrize("bn", [128, 256])
def test_dropout_bits_replay_and_graph(bn):
    """Generated dropout (mask_out) is bitwise identical between two calls and when replayed from a CUDA graph."""
    K_ = _ops()
    N, Kd = 1024, 1024
    a, b, bias, res = _rand(M, Kd, scale=0.05), _rand(N, Kd, scale=0.05), _rand(N), _rand(M, N)
    kw = dict(epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, seed=1234, stream=9, block_n=bn)
    m1 = torch.empty(M, N // 8, dtype=torch.uint8, device="cuda")
    m2 = torch.empty_like(m1)
    o1 = K_.gemm(a, b, mask_out=m1, **kw)
    o2 = K_.gemm(a, b, mask_out=m2, **kw)
    assert torch.equal(o1, o2) and torch.equal(m1, m2)
    assert torch.equal(m1, K_.dropout_mask(M, N, 0.1, 1234, 9, "cuda"))
    og = torch.empty_like(o1)
    mg = torch.zeros_like(m1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        K_.gemm(a, b, out=og, mask_out=mg, **kw)          # warm-up (tensor-map cache) outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        K_.gemm(a, b, out=og, mask_out=mg, **kw)
    og.zero_()
    mg.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, o1) and torch.equal(mg, m1)


@pytest.mark.parametrize("bn", [128, 256])
def test_fp8_nt_model_shape(bn):
    """fp8 operands (K-major NT) through the persistent kernel at the FFN-1 forward shape."""
    K_ = _ops()
    N, Kd = 4096, 1024
    a, b, bias = _rand(M, Kd), _rand(N, Kd, scale=0.05), _rand(N)
    meta = K_.Fp8Meta(["a", "b"], [False, False], "cuda")
    qa, qb = meta.quantize(a, "a", calibrate=True), meta.quantize(b, "b", calibrate=True)
    out = K_.gemm(qa, qb, epi=K_.EPI_BIAS, bias=bias, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"),
                  block_n=bn)
    _check(out, a.float() @ b.float().t() + bias.float(), tol=6e-2)
