"""Bandwidth-bound kernels, optimizer kernels and the fused engine vs PyTorch fp32 references."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


@pytest.mark.parametrize("M,H", [(64, 64), (1000, 1024), (300, 768), (130, 256), (257, 128), (300, 320), (200, 2048)])
def test_layer_norm_fwd_bwd(M, H):
    K = _api()
    x = (torch.randn(M, H, device="cuda") * 2 + 0.5).to(torch.bfloat16)
    g = torch.randn(H, device="cuda") * 0.5 + 1.0
    b = torch.randn(H, device="cuda") * 0.1
    dy = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    y, mean, rstd = K.layer_norm_fwd(x, g, b)
    xr = x.float().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = F.layer_norm(xr, (H,), gr, br, eps=1e-12)
    assert ((y.float() - yr).abs() / (yr.abs() + 1.0)).max() < 1.6e-2     # bf16 output rounding
    yr.backward(dy.float())
    dg, db, dbias = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    dx, dxd = K.layer_norm_bwd(dy, x, mean, rstd, g, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True, p_drop=0.0)
    assert (dx.float() - xr.grad).abs().max() < 3e-2 * max(1.0, xr.grad.abs().max().item())
    assert torch.equal(dx, dxd)
    assert torch.allclose(dg, gr.grad, rtol=2e-2, atol=2e-1)
    assert torch.allclose(db, br.grad, rtol=2e-2, atol=2e-1)
    assert torch.allclose(dbias, dx.float().sum(0), rtol=2e-2, atol=2e-1)


@pytest.mark.parametrize("M,H", [(512, 1024), (200, 320)])
def test_layer_norm_bwd_input_dropout(M, H):
    """``in_stream`` (the embedding LN, whose output was dropped out): dy is first multiplied by the keep decisions of
    that stream, element index row * H + col, and by the kept-element scale -- against an fp32 reference fed the same
    mask from the host twin of the generator."""
    K = _api()
    from bert_pytorch_b200.utils import philox
    p, seed, stream = 0.1, 1234, 1023 * 8
    x = (torch.randn(M, H, device="cuda") * 2 + 0.5).to(torch.bfloat16)
    g = torch.randn(H, device="cuda") * 0.5 + 1.0
    b = torch.randn(H, device="cuda") * 0.1
    dy = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    y, mean, rstd = K.layer_norm_fwd(x, g, b)
    keep = torch.from_numpy(philox.keep_mask(seed, stream, M * H, p)).view(M, H).cuda()
    xr = x.float().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    F.layer_norm(xr, (H,), gr, br, eps=1e-12).backward(dy.float() * keep * philox.keep_scale(p))
    dg, db = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    dx, dxd = K.layer_norm_bwd(dy, x, mean, rstd, g, dgamma=dg, dbeta=db, p_drop=p, seed=seed, in_stream=stream)
    assert dxd is None
    assert (dx.float() - xr.grad).abs().max() < 3e-2 * max(1.0, xr.grad.abs().max().item())
    assert torch.allclose(dg, gr.grad, rtol=2e-2, atol=2e-1)
    assert torch.allclose(db, br.grad, rtol=2e-2, atol=2e-1)


def test_layer_norm_dropout_mask_consistency():
    """The LN-backward dropped gradient must use the same mask as the GEMM epilogue of the forward."""
    K = _api()
    M, H = 512, 1024
    a = torch.randn(M, 64, device="cuda").to(torch.bfloat16)
    w = torch.randn(H, 64, device="cuda").to(torch.bfloat16)
    zeros_b = torch.zeros(H, device="cuda", dtype=torch.bfloat16)
    res = torch.zeros(M, H, device="cuda", dtype=torch.bfloat16)
    fwd = K.gemm(a, w, epi=K.EPI_BIAS_DROP_RES, bias=zeros_b, res=res, p_drop=0.1, seed=77, stream=19)
    x = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    g = torch.ones(H, device="cuda")
    y, mean, rstd = K.layer_norm_fwd(x, g, torch.zeros(H, device="cuda"))
    dy = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    dx, dxd = K.layer_norm_bwd(dy, x, mean, rstd, g, dgamma=None, dbeta=None, dbias=None, want_dropped=True,
                               p_drop=0.1, seed=77, drop_stream=19)
    kept_fwd = fwd != 0
    kept_bwd = dxd != 0
    # identical masks wherever neither value is an exact zero by accident
    assert (kept_fwd ^ kept_bwd).float().mean().item() < 1e-3


def test_dropout_keep_bits_leave_the_wide_gemm_and_feed_layer_norm_backward():
    """The hidden-dropout decisions are written by the 128 x 256 GEMM epilogue (1 bit per element, GemmCall::mask_out)
    and read back by the LayerNorm backward instead of re-running Philox: the bits must describe the forward output,
    and the backward with the mask must be BITWISE the backward that regenerates it."""
    K = _api()
    M, H = 1024, 1024
    a = torch.randn(M, 64, device="cuda").to(torch.bfloat16)
    w = torch.randn(H, 64, device="cuda").to(torch.bfloat16)
    zeros_b = torch.zeros(H, device="cuda", dtype=torch.bfloat16)
    res = torch.zeros(M, H, device="cuda", dtype=torch.bfloat16)
    mask = torch.zeros(M, H // 8, dtype=torch.uint8, device="cuda")
    fwd = K.gemm(a, w, epi=K.EPI_BIAS_DROP_RES, bias=zeros_b, res=res, p_drop=0.1, seed=77, stream=19, block_n=256,
                 mask_out=mask)
    ref = K.gemm(a, w, epi=K.EPI_BIAS_DROP_RES, bias=zeros_b, res=res, p_drop=0.1, seed=77, stream=19, block_n=256)
    assert torch.equal(fwd, ref)                                          # writing the bits does not change the output
    # the same bits from the stand-alone generator (K.dropout_mask), and the epilogue applying them instead of Philox
    gen = K.dropout_mask(M, H, 0.1, 77, 19, "cuda")
    assert torch.equal(gen, mask)
    from bert_pytorch_b200.utils import philox                   # ... and the host twin of the generator
    assert torch.equal(gen.cpu(), torch.from_numpy(philox.keep_bits(77, 19, M, H, 0.1)))
    via = K.gemm(a, w, epi=K.EPI_BIAS_DROP_RES, bias=zeros_b, res=res, p_drop=0.1, seed=77, stream=19, block_n=256, mask_in=gen)
    assert torch.equal(via, ref)
    bits = ((mask.view(M, H // 8, 1) >> torch.arange(8, device="cuda", dtype=torch.uint8).view(1, 1, 8)) & 1).view(M, H).bool()
    assert abs(1.0 - bits.float().mean().item() - 0.1) < 0.01
    assert ((fwd != 0) ^ bits).float().mean().item() < 1e-3               # exact zeros of the product are the only mismatches
    assert not (fwd[~bits] != 0).any()
    x = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    g = torch.rand(H, device="cuda") + 0.5
    y, mean, rstd = K.layer_norm_fwd(x, g, torch.zeros(H, device="cuda"))
    dy = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    outs = []
    for km in (None, mask):
        dg, db, dbias = (torch.zeros(H, device="cuda") for _ in range(3))
        dx, dxd = K.layer_norm_bwd(dy, x, mean, rstd, g, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True, p_drop=0.1,
                                   seed=77, drop_stream=19, keep_mask=km)
        outs.append((dx, dxd, dg, db, dbias))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])      # dx, dx_dropped: bitwise
    for u, v in zip(outs[0][2:], outs[1][2:]):                # column sums finish with atomics: order-dependent rounding
        assert torch.allclose(u, v, rtol=1e-4, atol=1e-3)


def test_embedding_fwd_bwd():
    K = _api()
    B, S, H, V = 4, 32, 256, 1000
    word = torch.randn(V, H, device="cuda").to(torch.bfloat16)
    pos = torch.randn(64, H, device="cuda").to(torch.bfloat16)
    typ = torch.randn(2, H, device="cuda").to(torch.bfloat16)
    g, b = torch.rand(H, device="cuda") + 0.5, torch.randn(H, device="cuda") * 0.1
    ids = torch.randint(0, V, (B * S,), device="cuda", dtype=torch.int32)
    seg = torch.randint(0, 2, (B * S,), device="cuda", dtype=torch.int32)
    y, e, mean, rstd = K.embedding_fwd(ids, seg, word, pos, typ, g, b, S)
    posi = torch.arange(S, device="cuda").repeat(B)
    er = word.float()[ids.long()] + pos.float()[posi] + typ.float()[seg.long()]
    assert (e.float() - er).abs().max() < 5e-2
    yr = F.layer_norm(e.float(), (H,), g, b, eps=1e-12)
    assert (y.float() - yr).abs().max() < 3e-2
    de = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
    gw, gp, gt = torch.zeros(V, H, device="cuda"), torch.zeros(64, H, device="cuda"), torch.zeros(2, H, device="cuda")
    K.embedding_bwd_scatter(de, ids, seg, gw, gp, gt, S)
    rw = torch.zeros_like(gw).index_add_(0, ids.long(), de.float())
    rp = torch.zeros_like(gp).index_add_(0, posi, de.float())
    rt = torch.zeros_like(gt).index_add_(0, seg.long(), de.float())
    assert torch.allclose(gw, rw, atol=1e-3) and torch.allclose(gp, rp, atol=1e-3) and torch.allclose(gt, rt, atol=1e-2)


def test_mlm_compact_gather_scatter_ce():
    K = _api()
    B, S, H, V, MP = 6, 64, 128, 2048, 16
    labels = torch.full((B, S), -1, device="cuda", dtype=torch.int32)
    for b in range(B):
        n = 3 + b * 2
        p = torch.randperm(S, device="cuda")[:n]
        labels[b, p] = torch.randint(0, V, (n,), device="cuda", dtype=torch.int32)
    idx, tgt, count = K.mlm_compact(labels, MP)
    assert int(count) == int((labels >= 0).sum())
    flat = labels.view(-1)
    valid = idx >= 0
    assert torch.equal(flat[idx[valid].long()], tgt[valid])
    assert (tgt[~valid] == -1).all()
    seq = torch.randn(B * S, H, device="cuda").to(torch.bfloat16)
    rows = K.gather_rows(seq, idx)
    assert torch.equal(rows[valid], seq[idx[valid].long()])
    assert (rows[~valid] == 0).all()
    back = torch.zeros_like(seq)
    K.scatter_rows(rows, idx, back)
    assert torch.equal(back[idx[valid].long()], rows[valid])
    # CE
    logits = (torch.randn(B * MP, V, device="cuda") * 3).to(torch.bfloat16)
    ref_in = logits.float().requires_grad_(True)
    ref = F.cross_entropy(ref_in, tgt.long(), ignore_index=-1)
    (ref * 4.0).backward()
    loss = torch.zeros(1, device="cuda")
    K.softmax_ce_(logits, tgt, count, 4.0, loss)
    assert abs(loss.item() - ref.item()) < 2e-2 * max(1.0, abs(ref.item()))
    assert (logits.float() - ref_in.grad).abs().max() < 2e-3


def test_colsum():
    K = _api()
    x = torch.randn(5000, 1000 + 24, device="cuda").to(torch.bfloat16)
    out = torch.ones(x.size(1), device="cuda")
    K.colsum_accumulate(x, out)
    assert torch.allclose(out, 1 + x.float().sum(0), rtol=1e-3, atol=1e-2)


def test_multi_tensor_l2norm_scale():
    K = _api()
    ts = [torch.randn(n, device="cuda") for n in (7, 70000, 1024, 333333)] + \
         [torch.randn(5000, device="cuda").to(torch.bfloat16)]
    total, per = K.multi_tensor_l2norm(ts, per_tensor=True)
    ref = torch.stack([t.float().norm() for t in ts])
    assert torch.allclose(per, ref, rtol=1e-3)
    assert abs(total.item() - ref.norm().item()) < 1e-2
    outs = [torch.empty_like(t) for t in ts]
    flag = K.multi_tensor_scale(ts, outs, 0.5)
    assert int(flag) == 0
    for t, o in zip(ts, outs):
        assert torch.allclose(o.float(), t.float() * 0.5, rtol=1e-2, atol=1e-3)
    ts[1][5] = float("inf")
    assert int(K.multi_tensor_scale(ts, outs, 0.5)) == 1


def _tiny_model(hidden=128, layers=2, heads=2, inter=256, vocab=1024, drop=0.0, nsp=True):
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    cfg = BertConfig(vocab_size_or_config_json_file=vocab, hidden_size=hidden, num_hidden_layers=layers,
                     num_attention_heads=heads, intermediate_size=inter, max_position_embeddings=128,
                     hidden_dropout_prob=drop, attention_probs_dropout_prob=drop, next_sentence=nsp)
    cfg.max_predictions_per_seq = 16
    torch.manual_seed(0)
    return BertForPreTraining(cfg)


def _batch(B=4, S=64, V=1024, MP=10):
    torch.manual_seed(1)
    ids = torch.randint(5, V, (B, S), device="cuda")
    seg = torch.zeros_like(ids)
    seg[:, S // 2:] = 1
    lens = torch.tensor([S, S - 7, S // 2, S - 1], device="cuda")[:B]
    mask = (torch.arange(S, device="cuda")[None] < lens[:, None]).long()
    labels = torch.full((B, S), -1, device="cuda")
    for b in range(B):
        p = torch.randperm(int(lens[b]), device="cuda")[:MP]
        labels[b, p] = ids[b, p]
    nsl = torch.randint(0, 2, (B,), device="cuda")
    return ids, seg, mask, labels, nsl


def test_fused_pretrainer_matches_oracle():
    """Loss and every parameter gradient of the fused kernel program vs fp32 autograd on the same weights
    (dropout off)."""
    _check_fused_pretrainer_against_oracle(vocab=1024)


def test_fused_pretrainer_matches_oracle_at_bert_vocab():
    """The same at BERT's padded vocabulary of 30528: the decoder GEMM with N = 30528, the MLM cross-entropy over
    30528 columns, and the tied word-embedding gradient at its real size."""
    _check_fused_pretrainer_against_oracle(vocab=30528)


def _check_fused_pretrainer_against_oracle(vocab):
    from bert_pytorch_b200.models import BertPretrainingCriterion
    from bert_pytorch_b200.models.arena import ParamArena
    model = _tiny_model(vocab=vocab).cuda()
    arena = ParamArena(model)
    batch = _batch(V=vocab)
    ids, seg, mask, labels, nsl = batch
    # oracle: fp32 autograd through the nn.Module forward, on bf16-rounded weights
    oracle = copy.deepcopy(model)
    for p in oracle.parameters():
        p.data = p.data.to(torch.bfloat16).float()
    oracle.bert.use_fused = False
    crit = BertPretrainingCriterion(model.config.vocab_size)
    scores, nsp = oracle(ids, seg, mask)
    ref_loss = crit(scores, labels, nsp, nsl)
    ref_loss.backward()
    eng = model.pretrain_engine()
    assert eng is not None
    arena.zero_grad()
    loss = eng.forward_backward(ids, seg, mask, labels, nsl, grad_scale=1.0)
    assert abs(loss.item() - ref_loss.item()) < 3e-2 * abs(ref_loss.item()), (loss.item(), ref_loss.item())
    bad = []
    gmax = max(po.grad.abs().max().item() for po in oracle.parameters())
    for (n, p), po in zip(model.named_parameters(), oracle.parameters()):
        g, go = p.grad.float(), po.grad.float()
        # key.bias has an exactly-zero true gradient (softmax shift invariance): floor the scale
        denom = max(go.abs().max().item(), 1e-3 * gmax)
        rel = (g - go).abs().max().item() / denom
        if rel > 8e-2:
            bad.append((n, rel, denom))
    assert not bad, bad[:10]


def test_encoder_autograd_bridge_matches_oracle():
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForQuestionAnswering
    cfg = BertConfig(vocab_size_or_config_json_file=1024, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                     intermediate_size=256, max_position_embeddings=128, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    torch.manual_seed(0)
    model = BertForQuestionAnswering(cfg).cuda()
    oracle = copy.deepcopy(model)
    for p in oracle.parameters():
        p.data = p.data.to(torch.bfloat16).float()
    oracle.bert.use_fused = False
    ids, seg, mask, _, _ = _batch()
    s, e = model(ids, seg, mask)
    so, eo = oracle(ids, seg, mask)
    assert (s - so).abs().max() < 5e-2 and (e - eo).abs().max() < 5e-2
    (s.sum() + e.sum()).backward()
    (so.sum() + eo.sum()).backward()
    w, wo = model.bert.encoder.layer[0].output.dense.weight, oracle.bert.encoder.layer[0].output.dense.weight
    rel = (w.grad - wo.grad).abs().max() / (wo.grad.abs().max() + 1e-6)
    assert rel < 8e-2, rel


def test_gelu_kernels():
    K = _api()
    x = (torch.randn(3000, 1024, device="cuda") * 2).to(torch.bfloat16)
    dy = torch.randn(3000, 1024, device="cuda").to(torch.bfloat16)
    y = K.gelu_fwd(x)
    xf = x.float().requires_grad_(True)
    ref = F.gelu(xf)
    assert ((y.float() - ref).abs() / (ref.abs() + 1.0)).max() < 1e-2
    ref.backward(dy.float())
    db = torch.zeros(1024, device="cuda")
    dx = K.dgelu_bwd(dy, x, db)
    assert (dx.float() - xf.grad).abs().max() < 3e-2
    assert torch.allclose(db, xf.grad.sum(0), rtol=2e-2, atol=0.5)     # db sums the unrounded fp32 products


def test_checkpoint_activations_replays_dropout_exactly():
    """--checkpoint_activations on the fused engine: segments are recomputed in the backward with the same
    Philox streams, so loss and gradients equal the store-everything program (dropout ON)."""
    from bert_pytorch_b200.models.arena import ParamArena
    m1 = _tiny_model(layers=5, drop=0.1).cuda()
    m2 = copy.deepcopy(m1)
    a1, a2 = ParamArena(m1), ParamArena(m2)
    m1.train(); m2.train()
    m2.checkpoint_activations(True)
    batch = _batch()
    e1, e2 = m1.pretrain_engine(), m2.pretrain_engine()
    e1.engine._seed_base = e2.engine._seed_base = 1234
    a1.zero_grad(); a2.zero_grad()
    l1 = e1.forward_backward(*batch)
    l2 = e2.forward_backward(*batch)
    assert abs(l1.item() - l2.item()) <= 1e-5 * abs(l1.item())      # the loss sum itself is reduced with atomics
    for (n, p), q in zip(m1.named_parameters(), m2.parameters()):
        scale = p.grad.abs().max().item() + 1e-12
        assert (p.grad - q.grad).abs().max().item() <= 1e-4 * scale, n      # split-K atomics reorder fp32 adds


def test_cuda_graph_replay_matches_eager_program():
    """forward_backward switches to a captured CUDA graph after two eager calls per input signature: the
    replays must produce the eager program's loss and gradients on fresh inputs (dropout off), and advance
    the dropout stream on every replay (dropout on)."""
    from bert_pytorch_b200.models.arena import ParamArena
    m_g = _tiny_model().cuda()
    m_e = copy.deepcopy(m_g)
    a_g, a_e = ParamArena(m_g), ParamArena(m_e)
    e_g, e_e = m_g.pretrain_engine(), m_e.pretrain_engine()
    e_e.use_graphs = False
    assert e_g.use_graphs
    base = _batch()
    for it in range(5):
        ids = torch.roll(base[0], it, dims=1)
        labels = torch.roll(base[3], it, dims=1)
        batch = (ids, base[1], base[2], labels, base[4])
        a_g.zero_grad(); a_e.zero_grad()
        lg = e_g.forward_backward(*batch).clone()
        le = e_e.forward_backward(*batch)
        assert abs(lg.item() - le.item()) <= 1e-5 * abs(le.item()), (it, lg.item(), le.item())
        for (n, p), q in zip(m_g.named_parameters(), m_e.parameters()):
            scale = q.grad.abs().max().item() + 1e-12
            assert (p.grad - q.grad).abs().max().item() <= 1e-4 * scale, (it, n)
    assert any("graph" in ent for ent in e_g._graphs.values())
    # dropout: two replays on identical inputs must draw different masks
    m_d = _tiny_model(drop=0.1).cuda()
    a_d = ParamArena(m_d)
    e_d = m_d.pretrain_engine()
    losses = []
    for it in range(6):
        a_d.zero_grad()
        losses.append(e_d.forward_backward(*base).item())
    assert any("graph" in ent for ent in e_d._graphs.values())
    assert len({round(x, 6) for x in losses[3:]}) == 3, losses


def test_wgrad_side_stream_matches_single_stream():
    """Weight-gradient GEMMs forked onto a second stream (eager calls, then the captured graph with the fork/join
    inside) give the single-stream program's loss and gradients."""
    from bert_pytorch_b200.models.arena import ParamArena
    m_s = _tiny_model().cuda()
    m_e = copy.deepcopy(m_s)
    a_s, a_e = ParamArena(m_s), ParamArena(m_e)
    e_s, e_e = m_s.pretrain_engine(), m_e.pretrain_engine()
    e_s.engine.wgrad_side = True
    e_e.engine.wgrad_side = False
    e_e.use_graphs = False
    base = _batch()
    for it in range(5):
        ids = torch.roll(base[0], it, dims=1)
        labels = torch.roll(base[3], it, dims=1)
        batch = (ids, base[1], base[2], labels, base[4])
        a_s.zero_grad(); a_e.zero_grad()
        ls = e_s.forward_backward(*batch).clone()
        le = e_e.forward_backward(*batch)
        torch.cuda.synchronize()
        assert abs(ls.item() - le.item()) <= 1e-5 * abs(le.item()), (it, ls.item(), le.item())
        for (n, p), q in zip(m_s.named_parameters(), m_e.parameters()):
            scale = q.grad.abs().max().item() + 1e-12
            assert (p.grad - q.grad).abs().max().item() <= 1e-4 * scale, (it, n)
    assert e_s.engine._wstream is not None and not e_s.engine._wkeep
    assert any("graph" in ent for ent in e_s._graphs.values())


def test_kfac_taps_of_the_fused_engine_match_module_hooks():
    """K-FAC statistics collected from the engine's saved activations (no module hooks fire on the fused path)
    equal the ones the hooks collect on the autograd path; the preconditioned step keeps gradients finite."""
    from bert_pytorch_b200 import kfac
    from bert_pytorch_b200.models import BertPretrainingCriterion
    from bert_pytorch_b200.models.arena import ParamArena
    m_f = _tiny_model().cuda()
    m_t = copy.deepcopy(m_f)
    for p in m_t.parameters():
        p.data = p.data.to(torch.bfloat16).float()
    m_t.bert.use_fused = False
    a_f = ParamArena(m_f)
    skip = ["BertLMPredictionHead", "embedding"]
    k_f = kfac.KFAC(m_f, factor_update_freq=1, inv_update_freq=1, skip_layers=skip, damping=0.003)
    k_t = kfac.KFAC(m_t, factor_update_freq=1, inv_update_freq=1, skip_layers=skip, damping=0.003)
    m_f.train(); m_t.train()
    ids, seg, mask, labels, nsl = _batch()
    a_f.zero_grad()
    eng = m_f.pretrain_engine()
    eng.forward_backward(ids, seg, mask, labels, nsl)
    crit = BertPretrainingCriterion(m_t.config.vocab_size)
    scores, nsp = m_t(ids, seg, mask)
    crit(scores, labels, nsp, nsl).backward()
    name = "bert.encoder.layer.1.output.dense"
    lf, lt = k_f.layer(name), k_t.layer(name)
    assert lf is not None and lf.A_new is not None and lt.A_new is not None
    for key in ("A_new", "G_new"):
        a, b = getattr(lf, key).float(), getattr(lt, key).float()
        rel = (a - b).norm() / b.norm()
        assert rel < 5e-2, (key, rel.item())
    k_f.step()
    assert all(torch.isfinite(p.grad).all() for p in m_f.parameters() if p.grad is not None)
    assert not any("graph" in e for e in eng._graphs.values())      # Python-side taps: no graph capture with K-FAC


@pytest.mark.parametrize("n,dtype", [(2, torch.bfloat16), (9, torch.bfloat16), (1, torch.float16), (5, torch.float32)])
def test_small_n_head_linear_on_the_tcgen05_gemm(n, dtype):
    """K28 / K29: the QA (N = 2) and classifier (N = num_labels) heads through _HeadLinearFn (N padded to 8, NT fp32-store
    forward, NN dgrad, TN fp32 wgrad) against nn.Linear in fp32: outputs and all three gradients."""
    from bert_pytorch_b200.models.fused import head_linear
    torch.manual_seed(0)
    M, H = 4 * 384, 256
    lin = torch.nn.Linear(H, n).cuda()
    x = (torch.randn(4, 384, H, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    y = head_linear(lin, x)
    assert y.shape == (4, 384, n)
    gy = torch.randn_like(y.float())
    y.float().backward(gy)
    xr = x.detach().float().requires_grad_(True)
    wr = lin.weight.detach().to(torch.bfloat16).float().requires_grad_(True)       # the kernel multiplies bf16 operands
    br = lin.bias.detach().clone().requires_grad_(True)
    yr = xr.to(torch.bfloat16).float() @ wr.t() + br
    yr.backward(gy)
    assert (y.float() - yr).abs().max().item() < 2e-2 * max(1.0, yr.abs().max().item())
    for got, want in ((x.grad.float(), xr.grad), (lin.weight.grad.float(), wr.grad), (lin.bias.grad.float(), br.grad)):
        assert (got - want).abs().max().item() <= 2e-2 * max(want.abs().max().item(), 1e-3), (got - want).abs().max().item()
