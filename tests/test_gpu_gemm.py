"""wgmma GEMM vs a plain fp32 PyTorch reference of the same op (T3 of SURVEY.md 4.2)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 128), (384, 1024, 1024), (1000, 512, 320),
                                   (4096, 3072, 1024), (130, 264, 72)])
@pytest.mark.parametrize("block_n", [128, 256, None])
def test_gemm_nt(M, N, K, block_n):
    K_ = _ops()
    a, b = _rand(M, K), _rand(N, K)
    out = K_.gemm(a, b, layout=K_.NT, block_n=block_n)
    _check(out, a.float() @ b.float().t())


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (512, 1024, 4096), (1000, 320, 512)])
@pytest.mark.parametrize("block_n", [128, 256, None])
def test_gemm_nn(M, N, K, block_n):
    K_ = _ops()
    a, b = _rand(M, K), _rand(K, N)
    out = K_.gemm(a, b, layout=K_.NN, block_n=block_n)
    _check(out, a.float() @ b.float())


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (1024, 1024, 4096), (320, 520, 1000)])
@pytest.mark.parametrize("block_n,splits", [(128, 1), (256, 1), (256, 4), (128, 3), (256, -1)])
def test_gemm_tn_accumulate(M, N, K, block_n, splits):
    K_ = _ops()
    a, b = _rand(K, M), _rand(K, N)
    base = torch.randn(M, N, device="cuda")
    out = base.clone()
    K_.gemm(a, b, layout=K_.TN, epi=K_.EPI_ACCUM_F32, out=out, block_n=block_n, k_splits=splits)
    _check(out, base + a.float().t() @ b.float(), tol=1e-2)


@pytest.mark.parametrize("M,N,K", [(1024, 4096, 12288), (1024, 1024, 4096), (520, 1000, 3000), (3072, 1024, 2048)])
def test_gemm_tn_auto_split(M, N, K):
    """k_splits=-1: the automatic split-K (as many K ranges as fill the SMs, at least 4 k-blocks each), merged by
    red.add; then wgrad_accumulate, which picks its own split."""
    K_ = _ops()
    a, b = _rand(K, M), _rand(K, N)
    base = torch.randn(M, N, device="cuda")
    out = base.clone()
    K_.gemm(a, b, layout=K_.TN, epi=K_.EPI_ACCUM_F32, out=out, block_n=256, k_splits=-1)
    _check(out, base + a.float().t() @ b.float(), tol=1e-2)
    grad = torch.zeros(M, N, device="cuda")
    K_.wgrad_accumulate(a, b, grad)                      # the engine's entry point (split-K heuristics)
    _check(grad, a.float().t() @ b.float(), tol=1e-2)


@pytest.mark.parametrize("M,N,K", [(4096, 1024, 12288), (1024, 1024, 4096), (3072, 1024, 2048), (520, 1000, 3000),
                                   (256, 256, 64)])
def test_gemm_tn_auto_split_narrow_tiles(M, N, K):
    """k_splits=-2: any negative value selects the automatic split-K, here on 128 x 128 tiles (twice the tiles of the
    128 x 256 test above, so fewer splits fill the SMs)."""
    K_ = _ops()
    a, b = _rand(K, M), _rand(K, N)
    base = torch.randn(M, N, device="cuda")
    out = base.clone()
    K_.gemm(a, b, layout=K_.TN, epi=K_.EPI_ACCUM_F32, out=out, block_n=128, k_splits=-2)
    _check(out, base + a.float().t() @ b.float(), tol=1e-2)


@pytest.mark.parametrize("M,N,K,splits", [(4096, 1024, 12288, -2), (1024, 4096, 4096, 1), (512, 512, 1024, -2), (768, 1536, 2048, 3),
                                          (304, 1000, 520, 1)])
def test_gemm_tn_256_wide_tiles(M, N, K, splits):
    """The 128 x 256 tiles (4-stage ring of 48 KB) for the fp32 weight-gradient epilogue, alone, with split-K and with
    the automatic split (k_splits < 0); accumulates into ``out``."""
    K_ = _ops()
    a, b = _rand(K, M), _rand(K, N)
    out = torch.randn(M, N, device="cuda")
    ref = out.clone() + a.float().t() @ b.float()
    K_.gemm(a, b, layout=K_.TN, epi=K_.EPI_ACCUM_F32, out=out, block_n=256, k_splits=splits)
    assert (out - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_epilogues_both_tile_widths(bn):
    """Bias, bias + dropout + residual, add, bias + tanh and fp32 store on the 128 x 128 (ping-pong) and 128 x 256
    (cooperative) kernels."""
    import functools
    K_ = _ops()
    real_gemm = K_.gemm
    K_ = type("Bn", (), {k: getattr(K_, k) for k in dir(K_) if k.startswith("EPI_") or k in ("NT", "NN", "TN")})
    K_.gemm = staticmethod(functools.partial(real_gemm, block_n=bn))
    M, N, Kd = 512, 1024, 256
    a, b, bias, res = _rand(M, Kd), _rand(N, Kd), _rand(N), _rand(M, N)
    ref = a.float() @ b.float().t()
    _check(K_.gemm(a, b, epi=K_.EPI_BIAS, bias=bias), ref + bias.float())
    _check(K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.0), ref + bias.float() + res.float())
    _check(K_.gemm(a, b, epi=K_.EPI_ADD, res=res), ref + res.float())
    _check(K_.gemm(a, b, epi=K_.EPI_BIAS_TANH, bias=bias), torch.tanh(ref + bias.float()))
    _check(K_.gemm(a, b, epi=K_.EPI_F32), ref, tol=5e-3)


def test_gemm_unbuilt_pair_raises():
    """Only the (operand form, epilogue) pairs that are built run: any other pair is refused before a launch."""
    K_ = _ops()
    M, N, Kd = 256, 256, 128
    a, bias, res = _rand(M, Kd), _rand(N), _rand(M, N)
    with pytest.raises(RuntimeError, match="no kernel"):
        K_.gemm(_rand(Kd, M), _rand(Kd, N), layout=K_.TN, epi=K_.EPI_BIAS, bias=bias)
    with pytest.raises(RuntimeError, match="no kernel"):
        K_.gemm(a, _rand(Kd, N), layout=K_.NN, epi=K_.EPI_BIAS_TANH, bias=bias)
    meta = K_.Fp8Meta(["a", "b"], [False, False], "cuda")
    qa, qb = meta.quantize(a, "a", calibrate=True), meta.quantize(_rand(N, Kd), "b", calibrate=True)
    with pytest.raises(RuntimeError, match="no kernel"):
        K_.gemm(qa, qb, epi=K_.EPI_MUL, res=res, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"))
    with pytest.raises(RuntimeError, match="unknown GEMM epilogue"):
        K_.gemm(a, _rand(N, Kd), epi=2)


def test_gemm_dropout_statistics_and_determinism():
    K_ = _ops()
    M, N, Kd = 1024, 1024, 64
    a, b, bias = _rand(M, Kd), _rand(N, Kd), torch.zeros(N, device="cuda", dtype=torch.bfloat16)
    res = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    full = K_.gemm(a, b, epi=K_.EPI_BIAS, bias=bias).float()
    d1 = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, seed=123, stream=5).float()
    d2 = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, seed=123, stream=5).float()
    d3 = K_.gemm(a, b, epi=K_.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1, seed=124, stream=5).float()
    assert torch.equal(d1, d2)
    assert not torch.equal(d1, d3)
    kept = d1 != 0
    frac = 1.0 - kept.float().mean().item()
    assert abs(frac - 0.1) < 0.01, frac
    assert torch.allclose(d1[kept], full[kept] / 0.9, rtol=2e-2, atol=2e-2)


def test_gemm_nt_wide_tiles_many_tiles_and_tails():
    """128 x 256 tiles: more tiles than SMs (several waves of CTAs, ring wrap) and ragged M/N edges."""
    K_ = _ops()
    for (M, N, Kd) in [(12288, 1024, 1024), (1000, 1000, 520), (257, 264, 64), (4096, 30528, 256)]:
        a, b = _rand(M, Kd), _rand(N, Kd)
        out = K_.gemm(a, b, layout=K_.NT, block_n=256)
        _check(out, a.float() @ b.float().t())


def _gelu_and_grad(x):
    x = x.double()
    Phi = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    return (x * Phi).float(), (Phi + x * phi).float()


def _bf16_ulp_err(out, ref):
    """|out - bf16(ref)| in units of bf16 ulps of the reference (floored at the ulp of 2^-14: below that the
    activation is smaller than anything the next GEMM can resolve against O(1) neighbours)."""
    ref = ref.float()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 7)
    return ((out.float() - ref).abs() / ulp).max().item()


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("M,N,Kd", [(512, 1024, 256), (12288, 4096, 128), (300, 520, 64)])
def test_gemm_bias_gelu_with_derivative(bn, M, N, Kd):
    """EPI_BIAS_GELU_DG: out = gelu(x), aux = gelu'(x) with x = a b^T + bias (K16: both leave the FFN-1 epilogue)."""
    K_ = _ops()
    a, b, bias = _rand(M, Kd, scale=0.3), _rand(N, Kd, scale=0.3), _rand(N)
    x = a.float() @ b.float().t() + bias.float()
    g_ref, d_ref = _gelu_and_grad(x)
    aux = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    out = K_.gemm(a, b, epi=K_.EPI_BIAS_GELU_DG, bias=bias, aux_out=aux, block_n=bn)
    # 1 ulp + accumulation-order flips at bf16 ties + the 1.5e-7 ABSOLUTE error of the erfc polynomial, which is up to
    # ~0.35 bf16 ulp of gelu(x) in the far negative tail (x ~ -4: |gelu| ~ 1e-4) -- seen as 1.34 over 50 M elements
    assert _bf16_ulp_err(out, g_ref) <= 1.5, _bf16_ulp_err(out, g_ref)
    assert _bf16_ulp_err(aux, d_ref) <= 1.5, _bf16_ulp_err(aux, d_ref)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("layout", ["NT", "NN"])
def test_gemm_mul_and_colsum(bn, layout):
    """EPI_MUL (+ fused column sums): the FFN-2 dgrad epilogue d_y1 = (d_y2 W2) * gelu'(x), bias gradient = colsum."""
    K_ = _ops()
    for (M, N, Kd) in [(512, 1024, 256), (12288, 4096, 64), (768, 520, 128)]:
        a = _rand(M, Kd, scale=0.5)
        b = _rand(N, Kd, scale=0.5) if layout == "NT" else _rand(Kd, N, scale=0.5)
        res = _rand(M, N)
        ref = (a.float() @ (b.float().t() if layout == "NT" else b.float())) * res.float()
        cs = torch.randn(N, device="cuda")
        cs0 = cs.clone()
        out = K_.gemm(a, b, layout=getattr(K_, layout), epi=K_.EPI_MUL, res=res, colsum=cs, block_n=bn)
        _check(out, ref)
        want = cs0 + out.float().sum(0)
        assert torch.allclose(cs, want, rtol=2e-3, atol=2e-2 * math.sqrt(M)), (cs - want).abs().max().item()
        cs2 = torch.zeros(N, device="cuda")
        out2 = K_.gemm(a, b, layout=getattr(K_, layout), epi=K_.EPI_ADD, res=res, colsum=cs2, block_n=bn)
        assert torch.allclose(cs2, out2.float().sum(0), rtol=2e-3, atol=2e-2 * math.sqrt(M))
