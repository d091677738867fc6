"""wgmma fused attention (forward + backward): run-to-run agreement under dropout, which exposes races.  The accuracy
tests against an fp64 reference are in test_gpu_attention_reference.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


@pytest.mark.parametrize("B,S,heads,lens,p_drop", [
    (3, 128, 4, [128, 77, 1], 0.1), (2, 128, 2, [128, 64], 0.0), (2, 64, 2, [64, 50], 0.1),
    (3, 512, 4, [512, 300, 129], 0.1), (2, 256, 2, [256, 130], 0.1), (2, 384, 2, [384, 1], 0.0), (40, 128, 16, None, 0.1),
])
def test_row_kernels_match_round1_kernels(B, S, heads, lens, p_drop):
    """(The name dates from two kernel generations that were compared here; there is one kernel per direction now.)
    Forward and backward twice on the same inputs and the same dropout stream: same Philox bits, so context,
    log-sum-exp and all three gradients must agree to bf16 rounding (dQ is reduced over key blocks with fp32
    reductions whose order is free); a race shows up as a run-to-run difference.  The big case has far more CTAs
    than the machine holds at once."""
    K = _api()
    torch.manual_seed(2)
    H = heads * 64
    qkv = (torch.randn(B, S, 3 * H, device="cuda") * 0.7).to(torch.bfloat16)
    seqlens = torch.tensor(lens if lens is not None else [S - (i % 5) * 7 for i in range(B)], device="cuda", dtype=torch.int32)
    dctx = (torch.randn(B, S, H, device="cuda") * 0.5).to(torch.bfloat16)
    kw = dict(p_drop=p_drop, seed=99, stream=6)
    ctx0, lse0 = K.attention_fwd(qkv, seqlens, heads, **kw)
    g0 = K.attention_bwd(qkv, seqlens, ctx0, dctx, lse0, heads, **kw).float()
    for _ in range(2):
        ctx1, lse1 = K.attention_fwd(qkv, seqlens, heads, **kw)
        g1 = K.attention_bwd(qkv, seqlens, ctx0, dctx, lse0, heads, **kw).float()
        torch.cuda.synchronize()
        valid = (torch.arange(S, device="cuda")[None, :] < seqlens[:, None])            # padded query rows: don't care
        assert ((ctx1.float() - ctx0.float()).abs() * valid[:, :, None]).max().item() < 2e-2
        assert ((lse1 - lse0).abs() * valid[:, None, :]).max().item() < 1e-3
        scale = g0.abs().max().item()
        assert torch.isfinite(g1).all()
        assert (g1 - g0).abs().max().item() <= 1.5e-2 * max(scale, 1.0), ((g1 - g0).abs().max().item(), scale)
