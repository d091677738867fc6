"""fp8 (e4m3 / e5m2, per-tensor delayed scaling) operands on the wgmma GEMM vs fp32 references."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from bert_pytorch_b200 import ops
    return ops


def _deq(q, meta, site):
    dt = torch.float8_e5m2 if meta.is_e5m2(site) else torch.float8_e4m3fn
    return q.view(dt).float() * meta.inv_scale(site)


@pytest.mark.parametrize("layout", ["NT", "NN", "TN"])
@pytest.mark.parametrize("shape", [(512, 768, 1024), (256, 256, 128), (1000, 520, 384)])
def test_fp8_gemm_matches_dequantised_reference(layout, shape):
    ops = _ops()
    api = ops.api
    M, N, K = shape
    if layout == "TN":
        M, N = (M + 15) // 16 * 16, (N + 15) // 16 * 16
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(5)
    if layout == "NT":
        a = torch.randn(M, K, device=dev, generator=g).bfloat16()
        b = (torch.randn(N, K, device=dev, generator=g) * 0.05).bfloat16()
    elif layout == "NN":
        a = (torch.randn(M, K, device=dev, generator=g) * 1e-3).bfloat16()
        b = (torch.randn(K, N - N % 16, device=dev, generator=g) * 0.05).bfloat16()
    else:
        a = (torch.randn(K, M, device=dev, generator=g) * 1e-3).bfloat16()
        b = torch.randn(K, N, device=dev, generator=g).bfloat16()
    a_e5 = layout != "NT"                       # gradients travel as e5m2, activations / weights as e4m3
    meta = api.Fp8Meta(["a", "b"], [a_e5, False], dev)
    qa = meta.quantize(a, "a", calibrate=True)
    qb = meta.quantize(b, "b", calibrate=True)
    lay = {"NT": api.NT, "NN": api.NN, "TN": api.TN}[layout]
    epi = api.EPI_F32 if layout == "TN" else api.EPI_NONE
    out = api.gemm(qa, qb, layout=lay, epi=epi, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"),
                   a_e5m2=a_e5, b_e5m2=False)
    torch.cuda.synchronize()
    da, db = _deq(qa, meta, "a"), _deq(qb, meta, "b")
    ref = {"NT": lambda: da @ db.t(), "NN": lambda: da @ db, "TN": lambda: da.t() @ db}[layout]()
    err = (out.float() - ref).abs().max().item()
    tol = 1e-2 * ref.abs().max().item() + 1e-6       # bf16 output rounding (fp32 for TN)
    assert err <= tol, (layout, shape, err, tol)
    # and the quantisation itself is sane: relative error vs the unquantised product within fp8 expectations
    full = {"NT": lambda: a.float() @ b.float().t(), "NN": lambda: a.float() @ b.float(),
            "TN": lambda: a.float().t() @ b.float()}[layout]()
    rel = (out.float() - full).norm() / full.norm()
    assert rel < (0.2 if a_e5 else 0.08), rel


def test_fp8_quantize_roundtrip_and_delayed_update():
    ops = _ops()
    api = ops.api
    dev = torch.device("cuda")
    x = (torch.randn(4096, 1024, device=dev) * 3).bfloat16()
    meta = api.Fp8Meta(["x", "g"], [False, True], dev)
    q = meta.quantize(x, "x", calibrate=True)
    rec = meta.record("x").tolist()
    amax = x.float().abs().max().item()
    assert rec[0] == pytest.approx(amax)                  # amax re-recorded by the quantise pass
    assert amax * rec[1] <= 448.0 and amax * rec[1] * 2 > 448.0
    deq = _deq(q, meta, "x")
    assert ((deq - x.float()).abs() <= x.float().abs() * 0.0625 + 2e-3 / rec[1]).all()
    meta.update()                                          # delayed scaling: same scale again, amax cleared
    rec2 = meta.record("x").tolist()
    assert rec2[0] == 0.0 and rec2[1] == rec[1]
    assert meta.record("g").tolist()[1] == 1.0             # untouched site keeps its scale


def test_fp8_gemm_bias_epilogue():
    ops = _ops()
    api = ops.api
    dev = torch.device("cuda")
    a = torch.randn(768, 1024, device=dev).bfloat16()
    w = (torch.randn(1024, 1024, device=dev) * 0.03).bfloat16()
    bias = torch.randn(1024, device=dev).bfloat16()
    meta = api.Fp8Meta(["a", "w"], [False, False], dev)
    qa, qw = meta.quantize(a, "a", calibrate=True), meta.quantize(w, "w", calibrate=True)
    out = api.gemm(qa, qw, epi=api.EPI_BIAS, bias=bias, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("w"))
    ref = _deq(qa, meta, "a") @ _deq(qw, meta, "w").t() + bias.float()
    assert (out.float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()


def test_fp8_engine_tracks_bf16_engine():
    """The fused kernel program with fp8 GEMM operands vs the same program in bf16: same loss within fp8 noise,
    weight gradients within the expected quantisation error; second micro-step runs on delayed scales."""
    import copy
    from test_gpu_kernels import _tiny_model, _batch
    from bert_pytorch_b200.models.arena import ParamArena
    model = _tiny_model(hidden=256, layers=2, heads=4, inter=1024).cuda()
    model8 = copy.deepcopy(model)
    a16, a8 = ParamArena(model), ParamArena(model8)
    ids, seg, mask, labels, nsl = _batch()
    e16, e8 = model.pretrain_engine(), model8.pretrain_engine()
    e8.engine.enable_fp8()
    for step in range(2):
        a16.zero_grad(); a8.zero_grad()
        l16 = e16.forward_backward(ids, seg, mask, labels, nsl)
        l8 = e8.forward_backward(ids, seg, mask, labels, nsl)
        assert abs(l16.item() - l8.item()) < 0.05 * abs(l16.item()), (step, l16.item(), l8.item())
        worst = 0.0
        gmax = max(p.grad.float().abs().max().item() for p in model.parameters())
        for (n, p), q in zip(model.named_parameters(), model8.parameters()):
            if p.grad.float().abs().max().item() < 1e-3 * gmax:     # e.g. key.bias: exactly-zero true gradient
                continue
            rel = ((p.grad - q.grad).float().norm() / p.grad.float().norm()).item()
            worst = max(worst, rel)
            assert rel < 0.25, (step, n, rel)
        assert worst > 0.0                 # the fp8 path really ran (not bitwise the bf16 program)
    rec = e8.engine.meta.table
    assert torch.isfinite(rec).all() and (rec[:, 1] > 0).all()


def test_producer_kernels_emit_fp8_copies():
    """LayerNorm fwd/bwd, GELU and dGELU write the fp8 copy of their output in the same pass (delayed scaling):
    the copy must dequantise to the bf16 output and the amax record must see the tensor."""
    ops = _ops()
    api = ops.api
    dev = torch.device("cuda")
    M, H = 512, 1024
    x = torch.randn(M, H, device=dev).bfloat16()
    g, b = torch.rand(H, device=dev) + 0.5, torch.randn(H, device=dev) * 0.1
    meta = api.Fp8Meta(["ln", "gelu", "dxd", "dgelu"], [False, False, True, True], dev)
    # scales as the previous step would have left them
    for site, t in (("ln", 16.0), ("gelu", 8.0), ("dxd", 0.25), ("dgelu", 0.25)):      # generous: nothing saturates
        rec = meta.record(site)
        rec[0] = t
    meta.update()

    def close(q, ref, site, rel):
        deq = _deq(q, meta, site)
        err = (deq - ref.float()).abs()
        assert (err <= rel * ref.float().abs() + 2.0 / meta.record(site)[1].item() * (2e-3 if not meta.is_e5m2(site) else 2e-5)).all(), site
        assert meta.record(site)[0].item() == pytest.approx(ref.float().abs().max().item(), rel=2e-2)
        assert ref.float().abs().max().item() * meta.record(site)[1].item() < (57344.0 if meta.is_e5m2(site) else 448.0)

    y, mean, rstd, q = api.layer_norm_fwd(x, g, b, fp8=(meta, "ln"))
    close(q, y, "ln", 0.07)
    act, q = api.gelu_fwd(x, fp8=(meta, "gelu"))
    close(q, act, "gelu", 0.07)
    dy = (torch.randn(M, H, device=dev) * 0.01).bfloat16()
    dg, db, dbias = (torch.zeros(H, device=dev) for _ in range(3))
    dx, dxd, q = api.layer_norm_bwd(dy, x, mean, rstd, g, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True, p_drop=0.1,
                                    seed=11, drop_stream=3, fp8=(meta, "dxd"))
    close(q, dxd, "dxd", 0.14)
    dbi = torch.zeros(H, device=dev)
    d1, q = api.dgelu_bwd(dy, x, dbi, fp8=(meta, "dgelu"))
    close(q, d1, "dgelu", 0.14)


def test_attention_kernels_emit_fp8_copies():
    """Attention forward / backward write the fp8 copy of ctx / dqkv in the same kernels (S = 128 single-block and
    S = 256 streaming variants)."""
    ops = _ops()
    api = ops.api
    dev = torch.device("cuda")
    for S in (128, 256):
        B, heads = 2, 2
        H = heads * 64
        qkv = (torch.randn(B, S, 3 * H, device=dev) * 0.5).bfloat16()
        lens = torch.tensor([S, S - 40], device=dev, dtype=torch.int32)
        meta = api.Fp8Meta(["ctx", "dqkv"], [False, True], dev)
        meta.record("ctx")[0] = 8.0
        meta.record("dqkv")[0] = 16.0
        meta.update()
        ctx, lse, q = api.attention_fwd(qkv, lens, heads, fp8=(meta, "ctx"))
        deq = _deq(q, meta, "ctx")
        assert ((deq - ctx.float()).abs() <= ctx.float().abs() * 0.07 + 2e-3 / meta.record("ctx")[1].item()).all()
        assert meta.record("ctx")[0].item() == pytest.approx(ctx.float().abs().max().item(), rel=2e-2)
        dctx = torch.randn(B, S, H, device=dev).bfloat16()
        dqkv, q2 = api.attention_bwd(qkv, lens, ctx, dctx, lse, heads, fp8=(meta, "dqkv"))
        deq2 = _deq(q2, meta, "dqkv")
        assert ((deq2 - dqkv.float()).abs() <= dqkv.float().abs() * 0.14 + 2e-5 / meta.record("dqkv")[1].item() + 1e-6).all()
        assert meta.record("dqkv")[0].item() == pytest.approx(dqkv.float().abs().max().item(), rel=2e-2)
