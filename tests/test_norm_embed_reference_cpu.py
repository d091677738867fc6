"""The fp64 references of tests/test_gpu_norm_embed_reference.py against torch.autograd in float64 on the CPU, on
random small shapes: they must be right before the H100 suite trusts them."""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_norm_embed_reference as ref


@pytest.mark.parametrize("M,H", [(1, 8), (7, 64), (33, 264), (5, 1032)])
def test_layer_norm_references_match_autograd(M, H):
    g = torch.Generator().manual_seed(M * 100 + H)
    x = (torch.randn(M, H, generator=g, dtype=torch.float64) * 2 + 0.5).requires_grad_(True)
    gamma = (torch.randn(H, generator=g, dtype=torch.float64) * 0.5 + 1).requires_grad_(True)
    beta = torch.randn(H, generator=g, dtype=torch.float64).requires_grad_(True)
    dy = torch.randn(M, H, generator=g, dtype=torch.float64)
    y = F.layer_norm(x, (H,), gamma, beta, eps=ref.EPS)
    y.backward(dy)
    yr, mu, rstd = ref.ln_fwd_ref(x.detach(), gamma.detach(), beta.detach())
    torch.testing.assert_close(yr, y.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mu, x.detach().mean(-1), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(rstd, 1 / torch.sqrt(x.detach().var(-1, unbiased=False) + ref.EPS), rtol=1e-12, atol=0)
    dx, dgamma, dbeta, xhat = ref.ln_bwd_ref(dy, x.detach(), mu, rstd, gamma.detach())
    torch.testing.assert_close(dx, x.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dgamma, gamma.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dbeta, beta.grad, rtol=1e-12, atol=1e-12)


def test_layer_norm_reference_of_equal_rows_is_beta():
    x = torch.full((3, 776), 1.75, dtype=torch.float64)        # its sum and mean are exact
    gamma, beta = torch.rand(776, dtype=torch.float64), torch.randn(776, dtype=torch.float64)
    y, mu, rstd = ref.ln_fwd_ref(x, gamma, beta)
    assert torch.equal(y, beta.expand_as(y)) and torch.allclose(rstd, torch.full_like(rstd, 1e6))


@pytest.mark.parametrize("with_type", [True, False])
def test_embedding_references_match_autograd(with_type):
    g = torch.Generator().manual_seed(3)
    V, P, H, M = 50, 16, 24, 70
    word = torch.randn(V, H, generator=g, dtype=torch.float64).requires_grad_(True)
    pos = torch.randn(P, H, generator=g, dtype=torch.float64).requires_grad_(True)
    typ = torch.randn(2, H, generator=g, dtype=torch.float64).requires_grad_(True)
    ids = torch.randint(0, V, (M,), generator=g)
    prow = torch.randint(0, P, (M,), generator=g)
    seg = torch.randint(0, 2, (M,), generator=g)
    e = F.embedding(ids, word) + F.embedding(prow, pos) + (F.embedding(seg, typ) if with_type else 0)
    de = torch.randn(M, H, generator=g, dtype=torch.float64)
    e.backward(de)
    er = ref.embed_sum_ref(word.detach(), pos.detach(), typ.detach() if with_type else None, ids, prow, seg)
    assert er.dtype == torch.bfloat16
    # one bf16 rounding (half an ulp: at most 2^-8 relative) of a sum whose fp32 rounding is far below it
    torch.testing.assert_close(er.double(), e.detach(), rtol=2.0 ** -8 + 2.0 ** -22, atol=1e-30)
    for table, key in ((word, ids), (pos, prow)) + (((typ, seg),) if with_type else ()):
        start = torch.randn(table.shape, generator=g, dtype=torch.float64)
        torch.testing.assert_close(ref.scatter_ref(start, key, de), start + table.grad, rtol=1e-12, atol=1e-12)
