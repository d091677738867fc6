"""The bf16 GEMM epilogues stage their output through shared memory and store it with TMA, and load their residual or
saved factor with TMA.  Checked at both tile widths: nothing outside the [M, N] window of a wider tensor is written,
the bf16 output equals bit for bit the fp32 recomputation from the same kernel's fp32 accumulator, and an output that
aliases the residual gives the same bits as a separate one."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M = 12288 - 37          # ragged last row block, several units per CTA
SENTINEL = 0x7BAD       # bf16 bit pattern of the bytes around the output window


def _ops():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)


def _framed(rows, cols, left, right):
    """a [rows, cols] column window of a wider bf16 tensor whose every element holds the sentinel"""
    full = torch.full((rows, left + cols + right), SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return full, full[:, left:left + cols]


def _outside_untouched(full, left, cols):
    bits = full.view(torch.int16)
    return bool((bits[:, :left] == SENTINEL).all()) and bool((bits[:, left + cols:] == SENTINEL).all())


def _keep(mask, m, n):
    return ((mask.unsqueeze(-1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1).reshape(m, n).bool()


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", ["none", "bias", "bias_drop_res", "add", "mul", "bias_gelu_dg", "bias_tanh"])
def test_output_window(bn, epi):
    """N = 1000 (not a multiple of 64) as a column slice of a wider tensor: every byte outside [M, N] of out and
    aux_out keeps the sentinel, every byte inside is written, and the plain, bias, add and mul outputs equal the fp32
    recomputation bit for bit, the ragged last 64-column subtile included.  At this N the dropout epilogue draws its keep bits
    in the kernel (mask_in needs N % 128 == 0)."""
    K_ = _ops()
    N, Kd, left, right = 1000, 256, 24, 40
    a, b = _rand(M, Kd, scale=0.1), _rand(N, Kd, scale=0.1)
    full, out = _framed(M, N, left, right)
    kw = {"out": out, "block_n": bn}
    aux_full = None
    if epi == "none":
        kw["epi"] = K_.EPI_NONE
    elif epi == "bias":
        kw.update(epi=K_.EPI_BIAS, bias=_rand(N))
    elif epi == "bias_drop_res":
        kw.update(epi=K_.EPI_BIAS_DROP_RES, bias=_rand(N), res=_rand(M, N), p_drop=0.1, seed=7)
    elif epi == "add":
        kw.update(epi=K_.EPI_ADD, res=_rand(M, N))
    elif epi == "mul":
        kw.update(epi=K_.EPI_MUL, res=_rand(M, N))
    elif epi == "bias_gelu_dg":
        aux_full, aux = _framed(M, N, left, right)
        kw.update(epi=K_.EPI_BIAS_GELU_DG, bias=_rand(N), aux_out=aux)
    else:
        kw.update(epi=K_.EPI_BIAS_TANH, bias=_rand(N))
    K_.gemm(a, b, **kw)
    torch.cuda.synchronize()
    assert _outside_untouched(full, left, N)
    assert not bool((out.view(torch.int16) == SENTINEL).any())
    if epi in ("none", "bias", "add", "mul"):          # values too, the ragged last 64-column subtile included
        acc = K_.gemm(a, b, epi=K_.EPI_F32, out=torch.empty(M, N, device="cuda"), block_n=bn)
        ref = (acc if epi == "none" else acc + kw["bias"].float() if epi == "bias"
               else acc + kw["res"].float() if epi == "add" else acc * kw["res"].float())
        assert torch.equal(out.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))
    if aux_full is not None:
        assert _outside_untouched(aux_full, left, N)
        assert not bool((aux_full[:, left:left + N].view(torch.int16) == SENTINEL).any())


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", ["none", "bias", "add", "mul", "bias_drop_res"])
def test_exact_epilogue_arithmetic(bn, epi):
    """The bf16 output equals, bit for bit, torch's fp32 recomputation from the same kernel's fp32 output (alpha times
    the accumulator): + bias, x keep x scale, + residual (or x saved factor), then round to nearest even."""
    K_ = _ops()
    N, Kd, alpha = 1024, 512, 0.75
    a, b = _rand(M, Kd, scale=0.2), _rand(N, Kd, scale=0.2)
    acc = K_.gemm(a, b, epi=K_.EPI_F32, out=torch.empty(M, N, device="cuda"), alpha=alpha, block_n=bn)
    bias, res = _rand(N), _rand(M, N)
    if epi == "none":
        out, ref = K_.gemm(a, b, alpha=alpha, block_n=bn), acc
    elif epi == "bias":
        out = K_.gemm(a, b, epi=K_.EPI_BIAS, bias=bias, alpha=alpha, block_n=bn)
        ref = acc + bias.float()
    elif epi == "add":
        out = K_.gemm(a, b, epi=K_.EPI_ADD, res=res, alpha=alpha, block_n=bn)
        ref = acc + res.float()
    elif epi == "mul":
        out = K_.gemm(a, b, epi=K_.EPI_MUL, res=res, alpha=alpha, block_n=bn)
        ref = acc * res.float()
    else:
        p = 0.1
        mask = K_.dropout_mask(M, N, p, 21, 3, "cuda")
        out = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=p, mask_in=mask, alpha=alpha,
                      block_n=bn)
        one = torch.tensor(65536.0, device="cuda")                  # the kernel's fp32 drop scale
        scale = one / (one - float(int(p * 65536.0 + 0.5)))
        x = acc + bias.float()
        ref = torch.where(_keep(mask, M, N), x * scale, torch.zeros_like(x)) + res.float()
    assert torch.equal(out.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", ["add", "mul", "bias_drop_res"])
def test_output_aliasing_residual(bn, epi):
    """out may be the residual tensor itself: each subtile is read before it is written and units are disjoint."""
    K_ = _ops()
    N, Kd = 1024, 512
    a, b, bias, res = _rand(M, Kd, scale=0.1), _rand(N, Kd, scale=0.1), _rand(N), _rand(M, N)
    kw = {"block_n": bn}
    if epi == "add":
        kw["epi"] = K_.EPI_ADD
    elif epi == "mul":
        kw["epi"] = K_.EPI_MUL
    else:
        kw.update(epi=K_.EPI_BIAS_DROP_RES, bias=bias, p_drop=0.1, mask_in=K_.dropout_mask(M, N, 0.1, 5, 1, "cuda"))
    separate = K_.gemm(a, b, res=res, **kw)
    inplace = res.clone()
    K_.gemm(a, b, res=inplace, out=inplace, **kw)
    assert torch.equal(inplace, separate)
