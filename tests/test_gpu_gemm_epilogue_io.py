"""GEMM epilogues that read a second [M, N] tensor: residual add, saved-factor product, bias + dropout + residual
with given keep bits.  Checked against fp32 torch references at both tile widths: several units per CTA,
residual and output as column slices of wider tensors, ragged tails, keep bits applied bitwise, bitwise replay
(twice eagerly and from a CUDA graph), and the fp8 path."""
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


def _keep(K_, mask, m, n):
    return ((mask.unsqueeze(-1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).reshape(m, n).bool()


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("N,Kd", [(1024, 1024), (4096, 1024), (1024, 4096)])
def test_input_epilogues_many_units(bn, N, Kd):
    """EPI_ADD and EPI_MUL + colsum (NN), EPI_BIAS_DROP_RES with mask_in (NT) at M = 12288."""
    K_ = _ops()
    a, res = _rand(M, Kd, scale=0.05), _rand(M, N)
    bnn = _rand(Kd, N, scale=0.05)
    ref = a.float() @ bnn.float()
    _check(K_.gemm(a, bnn, layout=K_.NN, epi=K_.EPI_ADD, res=res, block_n=bn), ref + res.float())
    cs = torch.zeros(N, device="cuda")
    out = K_.gemm(a, bnn, layout=K_.NN, epi=K_.EPI_MUL, res=res, colsum=cs, block_n=bn)
    _check(out, ref * res.float())
    assert torch.allclose(cs, out.float().sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(M))
    bnt, bias = _rand(N, Kd, scale=0.05), _rand(N)
    x = a.float() @ bnt.float().t() + bias.float()
    mask = K_.dropout_mask(M, N, 0.1, 5, 2, "cuda")
    out = K_.gemm(a, bnt, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, mask_in=mask, block_n=bn)
    _check(out, torch.where(_keep(K_, mask, M, N), x / 0.9, torch.zeros_like(x)) + res.float())


@pytest.mark.parametrize("bn", [128, 256])
def test_strided_column_slices(bn):
    """res and out are column slices of wider tensors (row pitch != N), at an offset that keeps 16-byte alignment."""
    K_ = _ops()
    N, Kd = 1024, 1024
    a, b = _rand(M, Kd, scale=0.05), _rand(N, Kd, scale=0.05)
    res_full, out_full = _rand(M, N + 256), torch.zeros(M, N + 136, dtype=torch.bfloat16, device="cuda")
    res, out = res_full[:, 128:128 + N], out_full[:, 8:8 + N]
    K_.gemm(a, b, epi=K_.EPI_ADD, res=res, out=out, block_n=bn)
    _check(out, a.float() @ b.float().t() + res.float())
    assert torch.count_nonzero(out_full[:, :8]) == 0 and torch.count_nonzero(out_full[:, 8 + N:]) == 0


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("Mr,N,Kd", [(12290, 1032, 264), (1000, 1000, 520), (129, 136, 72), (300, 384, 64)])
def test_ragged_tails(bn, Mr, N, Kd):
    """Ragged M and N edges: out-of-range rows and columns of the input tile are zero-filled and never stored."""
    K_ = _ops()
    a, b, res = _rand(Mr, Kd), _rand(Kd, N), _rand(Mr, N)
    out_full = torch.zeros(Mr + 8, N, dtype=torch.bfloat16, device="cuda")
    out = out_full[:Mr]
    K_.gemm(a, b, layout=K_.NN, epi=K_.EPI_ADD, res=res, out=out, block_n=bn)
    _check(out, a.float() @ b.float() + res.float())
    assert torch.count_nonzero(out_full[Mr:]) == 0
    _check(K_.gemm(a, b, layout=K_.NN, epi=K_.EPI_MUL, res=res, block_n=bn), (a.float() @ b.float()) * res.float())


@pytest.mark.parametrize("bn", [128, 256])
def test_mask_in_bits_applied_bitwise(bn):
    """With zero operands the dropout epilogue returns res exactly where a keep bit is 0 and bias / 0.9 + res
    (one bf16 rounding) where it is 1: every bit of mask_in lands on its own element."""
    K_ = _ops()
    N, Kd = 1280, 128                                   # N % 256 != 0: a ragged 256-wide tile at the right edge
    a, b = torch.zeros(M, Kd, dtype=torch.bfloat16, device="cuda"), _rand(N, Kd)
    bias, res = _rand(N), _rand(M, N)
    mask = K_.dropout_mask(M, N, 0.3, 11, 4, "cuda")
    out = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.3, mask_in=mask, block_n=bn)
    keep = _keep(K_, mask, M, N)
    one = torch.tensor(65536.0, device="cuda")                  # the kernel's fp32 drop scale
    scale = one / (one - float(int(0.3 * 65536.0 + 0.5)))
    ref = torch.where(keep, bias.float() * scale + res.float(), res.float()).to(torch.bfloat16)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("bn", [128, 256])
def test_two_calls_and_graph_replay_bitwise(bn):
    """Two calls and a CUDA-graph replay of the input-reading epilogues give bitwise equal outputs."""
    K_ = _ops()
    N, Kd = 1024, 1024
    a, b, bias, res = _rand(M, Kd, scale=0.05), _rand(N, Kd, scale=0.05), _rand(N), _rand(M, N)
    mask = K_.dropout_mask(M, N, 0.1, 1234, 9, "cuda")
    cs1, cs2 = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    kw = dict(epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, mask_in=mask, block_n=bn)
    o1, o2 = K_.gemm(a, b, **kw), K_.gemm(a, b, **kw)
    m1 = K_.gemm(a, b, epi=K_.EPI_MUL, res=res, colsum=cs1, block_n=bn)
    m2 = K_.gemm(a, b, epi=K_.EPI_MUL, res=res, colsum=cs2, block_n=bn)
    assert torch.equal(o1, o2) and torch.equal(m1, m2)
    og = torch.empty_like(o1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        K_.gemm(a, b, out=og, **kw)                     # warm-up (tensor-map cache) outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        K_.gemm(a, b, out=og, **kw)
    og.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, o1)


@pytest.mark.parametrize("bn", [128, 256])
def test_fp8_bias_dropout_residual(bn):
    """fp8 operands with the residual-reading dropout epilogue (the fp8 forward of the attention output)."""
    K_ = _ops()
    N, Kd = 1024, 1024
    a, b, bias, res = _rand(M, Kd), _rand(N, Kd, scale=0.05), _rand(N), _rand(M, N)
    meta = K_.Fp8Meta(["a", "b"], [False, False], "cuda")
    qa, qb = meta.quantize(a, "a", calibrate=True), meta.quantize(b, "b", calibrate=True)
    mask = K_.dropout_mask(M, N, 0.1, 3, 1, "cuda")
    out = K_.gemm(qa, qb, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, mask_in=mask,
                  scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"), block_n=bn)
    x = a.float() @ b.float().t() + bias.float()
    _check(out, torch.where(_keep(K_, mask, M, N), x / 0.9, torch.zeros_like(x)) + res.float(), tol=6e-2)
