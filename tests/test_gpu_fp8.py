"""fp8 (e4m3 / e5m2, per-tensor delayed scaling) operands on the wgmma GEMM vs fp32 references (the exact references of
every fp8 kernel are in test_gpu_fp8_reference.py)."""
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
