"""The LayerNorm and embedding kernels (ops/csrc/norm_embed.cu) against fp64 references on the device, computed from
the same bf16 inputs the kernels read, at every kernel instantiation, around every grid-stride boundary and under every
dropout source; and the refusals of their bindings.

Every bound is derived from the fp32 arithmetic of the kernel it checks (u = 2^-24, the unit roundoff of fp32; a sum
whose longest chain of dependent additions is n is off by at most n u times the sum of the magnitudes of its terms;
terms of O(u^2) are dropped, and HIGHER_ORDER covers them).  Each check prints its worst error over its bound.

Grid caps, from the launchers: the LayerNorm forward sweeps sms * 4 blocks x 8 rows; the backward sms * 3 blocks x
groups(H) rows; the embedding forward sms * 8 blocks x 4 rows."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                   # fp32 unit roundoff
EPS = 1e-12
RSQRT_ERR = 4 * U                # rsqrtf: at most 2 ulp (CUDA C programming guide), an fp32 ulp is <= 2^-23 relative
HIGHER_ORDER = 1.0 + 2.0 ** -10  # the O(u^2) products of the first-order error terms below
EMB_STREAM = 1023 * 8            # the embedding dropout stream of the engine

LN_H = [256, 512, 768, 1024,     # non-TAIL (H = CHUNKS * 256 / WPR * 256)
        8, 64, 264, 504,         # TAIL, forward CHUNKS 2 (backward WPR 1 or 2)
        520, 776, 1016,          # TAIL, forward CHUNKS 4 (backward WPR 4)
        1032, 1536, 2048]        # TAIL, forward CHUNKS 8 (backward WPR 8)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references (device-agnostic: tests/test_norm_embed_reference_cpu.py checks them against torch.autograd)
# ---------------------------------------------------------------------------------------------------------------------
def ln_stats_ref(x, eps=EPS):
    """fp64 mean, biased variance and rstd = 1 / sqrt(var + eps) of every row of ``x``"""
    xd = x.double()
    mu = xd.mean(-1)
    var = ((xd - mu[:, None]) ** 2).mean(-1)
    return mu, var, (var + eps).rsqrt()


def ln_fwd_ref(x, gamma, beta, eps=EPS):
    """fp64 (x - mu) * rsqrt(var + eps) * gamma + beta, and (mu, rstd)"""
    mu, _, rstd = ln_stats_ref(x, eps)
    xhat = (x.double() - mu[:, None]) * rstd[:, None]
    return xhat * gamma.double() + beta.double(), mu, rstd


def ln_bwd_ref(dy, x, mean, rstd, gamma):
    """fp64 LayerNorm backward at the given statistics: dx = rstd (g - mean(g) - xhat mean(g xhat)) with g = gamma dy;
    dgamma = sum_rows dy xhat, dbeta = sum_rows dy.  Returns (dx, dgamma, dbeta, xhat)."""
    xhat = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    g = dy.double() * gamma.double()
    dx = rstd.double()[:, None] * (g - g.mean(-1, keepdim=True) - xhat * (g * xhat).mean(-1, keepdim=True))
    return dx, (dy.double() * xhat).sum(0), dy.double().sum(0), xhat


def embed_sum_ref(word, pos, type_emb, ids, pos_rows, seg):
    """bf16((word[id] + pos[p]) + type[seg]), summed in fp32 in the kernel's order"""
    e = word.float()[ids.long()] + pos.float()[pos_rows.long()]
    if type_emb is not None:
        e = e + type_emb.float()[seg.long()]
    return e.bfloat16()


def scatter_ref(table, key, de):
    """fp64 table + index_add of the rows of ``de`` at ``key``"""
    return table.double().index_add(0, key.long(), de.double())


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _groups(H):                  # rows per block of the LayerNorm backward (norm_embed.cu: ln_bwd_groups)
    return 8 if H <= 256 else 4 if H <= 512 else 2 if H <= 1024 else 1


def _fwd_sweep():
    return _sms() * 4 * 8


def _bwd_sweep(H):
    return _sms() * 3 * _groups(H)


def _emb_sweep():
    return _sms() * 8 * 4


def _rows(spec, sweep, groups=1):
    """a row count named relative to the grid: 'sweep+1', 'g-1', or a number"""
    env = {"sweep": sweep, "g": groups}
    return int(eval(spec, {}, env))


def _ulp(ref):
    """bf16 ulp of the reference, floored at the ulp of 2^-14 (as tests/test_gpu_fp8_reference.py::_bf16_ulp_err)"""
    return torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 7)


def _report(tag, err, bound):
    """assert err <= bound elementwise; prints and returns the worst err / bound"""
    err, bound = err.double(), bound.double()
    ratio = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    print(f"[norm/embed] {tag}: worst err / bound = {ratio:.3e}")
    assert torch.isfinite(err).all() and (err <= bound).all(), (tag, ratio)
    return ratio


def _keep(seed, stream, M, H, p, dev="cuda"):
    from bert_pytorch_b200.utils import philox
    return torch.from_numpy(philox.keep_mask(seed, stream, M * H, p)).view(M, H).to(dev)


def _keep_bits(seed, stream, M, H, p):
    from bert_pytorch_b200.utils import philox
    return torch.from_numpy(philox.keep_bits(seed, stream, M, H, p)).cuda()


def _stat_bounds(x, n_chain):
    """Derived bounds of the fp32 row statistics of the bf16 rows ``x`` (the LayerNorm forward and the embedding).
    mean = fl(sum / H), the sum over a chain of n_chain additions (a lane's 8 columns per 256-column chunk, then five
    shuffle levels): |mean - mu| <= dmu = (n_chain + 1) u sum|x| / H.  The two-pass variance sums the squares of
    d = fl(x - mean) (2u each) over the same chain (n_chain u), scales by 1/H (2u) and adds eps (u), around mean
    instead of mu (+ (mean - mu)^2): |V_kernel - V| <= dV = (n_chain + 5) u (var + dmu^2) + dmu^2 with V = var + eps.
    rstd = rsqrtf(V_kernel): relative error <= r / 2 + r^2 + RSQRT_ERR with r = dV / V (r <= 0.1)."""
    H = x.size(-1)
    mu, var, rs = ln_stats_ref(x)
    dmu = (n_chain + 1) * U * x.double().abs().sum(-1) / H
    V = var + EPS
    r = ((n_chain + 5) * U * (var + dmu ** 2) + dmu ** 2 + U * V) / V
    return mu, var, rs, dmu, r, (0.5 * r + r * r + RSQRT_ERR) * HIGHER_ORDER


def _fwd_chain(H):
    return 8 * ((H + 255) // 256) + 5


def _check_ln_output(tag, y, mean, rstd, x, gamma, beta, *, roundings, keep=None, scale=1.0, const_rows=None):
    """y = bf16(dropout(LN(x))) and the saved statistics against fp64.  ``roundings``: fp32 roundings of
    (x - mean) * rstd * gamma before the final add (2 for the LayerNorm forward: the subtraction and the product with
    rstd, then one fma; 3 for the embedding, whose product with gamma is rounded on its own).
    Rows of equal values (``const_rows``, a bool mask) have sum and mean exact and a variance of exactly 0: there y must
    be bf16(beta) bit for bit, mean the value itself and rstd rsqrtf(eps)."""
    H = x.size(-1)
    mu, var, rs, dmu, r, rel_rs = _stat_bounds(x, _fwd_chain(H))
    const = const_rows if const_rows is not None else torch.zeros(x.size(0), dtype=torch.bool, device=x.device)
    live = ~const
    assert (r[live] <= 0.1).all()
    if mean is not None:
        _report(f"{tag} mean", (mean.double() - mu).abs()[live], dmu[live])
        _report(f"{tag} rstd", (rstd.double() / rs - 1).abs()[live], rel_rs[live])
    xhat = (x.double() - mu[:, None]) * rs[:, None]
    g, b = gamma.double(), beta.double()
    ref = xhat * g + b
    # |t - xhat| for t = fl(fl(x - mean) * rstd): the mean's error scaled by rstd, plus the relative errors of rstd and of
    # the roundings; then gamma times that, and the final add (u of its operands)
    shift = (dmu * rs)[:, None]
    e = g.abs() * (shift + (shift + xhat.abs()) * (rel_rs[:, None] + roundings * U)) + U * ((xhat * g).abs() + b.abs())
    if keep is not None:          # o = fl(y32 * scale) where kept, else 0 (2u: the product and the fp32 scale itself)
        ref = ref * keep * scale
        e = keep * (scale * e + 2 * U * scale * ((xhat * g).abs() + b.abs()))
    bound = (0.5 * _ulp(ref) + e) * HIGHER_ORDER
    _report(f"{tag} y", (y.double() - ref)[live], bound[live])
    if const.any():
        yb = (b.expand_as(ref) * (keep * scale if keep is not None else 1.0)).float().bfloat16()
        assert torch.equal(y[const], yb[const]), f"{tag}: a row of equal values must give beta"
        if mean is not None:
            assert torch.equal(mean[const].double(), mu[const]), f"{tag}: mean of a row of equal values"
            want = 1.0 / math.sqrt(float(np.float32(EPS)))
            _report(f"{tag} rstd (equal rows)", (rstd[const].double() / want - 1).abs(),
                    torch.full_like(rstd[const].double(), RSQRT_ERR))


def _ln_input(M, H, gen):
    """rows of N(0.5, 2), every fifth row (from row 1) all one value, every fifth (from row 3) N(48, 1): |mu| >> sigma"""
    x = torch.randn(M, H, device="cuda", generator=gen) * 2 + 0.5
    r = torch.arange(M, device="cuda")
    const = r % 5 == 1
    x[const] = torch.randn(int(const.sum()), 1, device="cuda", generator=gen) * 3
    off = r % 5 == 3
    x[off] = 48 + torch.randn(int(off.sum()), H, device="cuda", generator=gen)
    return x.bfloat16(), const


def _gamma_beta(H, gen):
    return (torch.randn(H, device="cuda", generator=gen) * 0.5 + 1.0,
            torch.randn(H, device="cuda", generator=gen) * 0.5)


# ---------------------------------------------------------------------------------------------------------------------
# 1. LayerNorm forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", ["1", "7", "8", "9", "sweep-1", "sweep", "sweep+1", "12288"])
@pytest.mark.parametrize("H", LN_H)
def test_layer_norm_fwd_matches_fp64(H, rows):
    K = _api()
    M = _rows(rows, _fwd_sweep())
    gen = torch.Generator(device="cuda").manual_seed(H * 7919 + M)
    x, const = _ln_input(M, H, gen)
    gamma, beta = _gamma_beta(H, gen)
    y, mean, rstd = K.layer_norm_fwd(x, gamma, beta)
    _check_ln_output(f"LN fwd H={H} M={M}", y, mean, rstd, x, gamma, beta, roundings=2, const_rows=const)
    y2, m2, r2 = K.layer_norm_fwd(x, gamma, beta, save_stats=False)     # null statistic pointers
    assert m2 is None and r2 is None and torch.equal(y2, y)


# ---------------------------------------------------------------------------------------------------------------------
# 2. LayerNorm backward
# ---------------------------------------------------------------------------------------------------------------------
def _bwd_chains(M, H, Z):
    """(n_row, L): the longest addition chain of a row sum (4 per f32x2 component, 1 to combine them, 5 shuffle levels,
    WPR across the warps of a row) and of a column sum: the rows a thread walks (ceil(M / stride)), the GROUPS - 1 row
    groups of a block, a finalize warp's ceil(ceil(grid / Z) / 8) partials, the 8 warps, then Z slices added to the
    starting value."""
    groups, wpr = _groups(H), 8 // _groups(H)
    if H % 256 == 0 and H <= 1024:
        wpr = H // 256
    grid = min((M + groups - 1) // groups, _sms() * 3)
    stride = grid * groups
    per = (grid + Z - 1) // Z
    return 10 + wpr, (M + stride - 1) // stride + groups - 1 + (per + 7) // 8 + 8 + Z


def _ln_bwd_bounds(dy_eff, dy_round, x, mean, rstd, gamma, n_row):
    """Reference dx (fp64 on the kernel's own statistics) and the bound of the kernel's fp32 dx before its bf16 rounding.
    xh = fma(x, rstd, fl(-mean rstd)) is off by dx_h = u (|mean rstd| + |xhat|); dg = fl(d gamma) by u |g| (plus the
    2u of d = fl(dy * scale) under input dropout, dy_round = 2: the product and the fp32 scale); the row sums s1 = sum dg, s2 = sum dg xh by
    n_row u sum|.| plus their terms' errors; c = -rstd s / H three more roundings; o = fma(xh, c2, fma(dg, rstd, c1))
    two (u of their operands)."""
    H = x.size(-1)
    dx, dgam, dbet, xhat = ln_bwd_ref(dy_eff, x, mean, rstd, gamma)
    r = rstd.double()[:, None]
    g = dy_eff.double() * gamma.double()
    ag = g.abs()
    dxh = U * ((mean.double()[:, None] * r).abs() + xhat.abs())
    dg = (1 + dy_round) * U * ag
    s1, s2 = g.sum(-1, keepdim=True), (g * xhat).sum(-1, keepdim=True)
    e_s1 = n_row * U * ag.sum(-1, keepdim=True) + dg.sum(-1, keepdim=True)
    e_s2 = n_row * U * (ag * xhat.abs()).sum(-1, keepdim=True) + (dg * xhat.abs() + ag * dxh).sum(-1, keepdim=True)
    e_c1 = r / H * (e_s1 + 3 * U * s1.abs())
    e_c2 = r / H * (e_s2 + 3 * U * s2.abs())
    c1, c2 = -r * s1 / H, -r * s2 / H
    e = (r * dg + e_c1 + xhat.abs() * e_c2 + dxh * c2.abs() + U * ((g * r).abs() + c1.abs())
         + U * (dx.abs() + (xhat * c2).abs()))
    return dx, dgam, dbet, xhat, e * HIGHER_ORDER, dxh


def _run_ln_bwd(K, dy, x, mean, rstd, gamma, starts, **kw):
    acc = [s.clone() if s is not None else None for s in starts]
    dx, dxd = K.layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma=acc[0], dbeta=acc[1], dbias=acc[2], **kw)
    return dx, dxd, acc


def _check_ln_bwd(tag, M, H, Z, dy, x, mean, rstd, gamma, dx, dxd, acc, starts, *, keep_out=None, keep_in=None, p=0.0):
    from bert_pytorch_b200.utils import philox
    scale = philox.keep_scale(p)
    dy_eff = dy.double() * (keep_in * scale if keep_in is not None else 1.0)
    n_row, L = _bwd_chains(M, H, Z)
    ref, dgam, dbet, xhat, e, dxh = _ln_bwd_bounds(dy_eff, 2.0 if keep_in is not None else 0.0, x, mean, rstd, gamma, n_row)
    _report(f"{tag} dx", (dx.double() - ref).abs(), 0.5 * _ulp(ref) + e)
    o_ref, e_o = ref, e
    if dxd is not None:
        if keep_out is not None:
            o_ref = ref * keep_out * scale
            e_o = keep_out * (scale * e + 2 * U * scale * ref.abs()) * HIGHER_ORDER
        _report(f"{tag} dx_dropped", (dxd.double() - o_ref).abs(), 0.5 * _ulp(o_ref) + e_o)
    # column sums: L u (|start| + sum |terms|) plus the terms' own errors (dgamma: d * dx_h, and the rounding of d
    # under input dropout; dbias: the fp32 dropped gradient's bound)
    d_round = 2 * U * dy_eff.abs() if keep_in is not None else torch.zeros_like(dy_eff)
    names = ("dgamma", "dbeta", "dbias")
    terms = (dy_eff * xhat, dy_eff, o_ref)
    own = ((dy_eff.abs() * dxh + d_round * xhat.abs()).sum(0), d_round.sum(0), e_o.sum(0))
    for k in range(3):
        if acc[k] is None:
            continue
        if k == 2 and dxd is None:
            assert torch.equal(acc[k], starts[k]), f"{tag}: dbias changed without the dropped gradient"
            continue
        want = starts[k].double() + terms[k].sum(0)
        bound = (L * U * (starts[k].double().abs() + terms[k].abs().sum(0)) + own[k]) * HIGHER_ORDER
        _report(f"{tag} {names[k]}", (acc[k].double() - want).abs(), bound)


def _bwd_inputs(M, H, seed):
    K = _api()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x, _ = _ln_input(M, H, gen)
    gamma, beta = _gamma_beta(H, gen)
    _, mean, rstd = K.layer_norm_fwd(x, gamma, beta)
    dy = torch.randn(M, H, device="cuda", generator=gen).bfloat16()
    starts = [torch.randn(H, device="cuda", generator=gen) for _ in range(3)]
    return K, x, gamma, mean, rstd, dy, starts


@pytest.mark.parametrize("rows", ["1", "g", "g+1", "sweep-1", "sweep+1", "2*sweep+3"])
@pytest.mark.parametrize("H", LN_H)
def test_layer_norm_bwd_matches_fp64(H, rows, monkeypatch):
    """Dropped gradient of the regenerated drop_stream, then of keep_mask (host twin of the generator: the same bits as
    K.dropout_mask), in the default (8 atomic slices) and the deterministic (one slice) finalize."""
    M = _rows(rows, _bwd_sweep(H), _groups(H))
    K, x, gamma, mean, rstd, dy, starts = _bwd_inputs(M, H, H * 31 + M)
    p, seed, stream = 0.1, 4242, 19
    keep = _keep(seed, stream, M, H, p)
    bits = _keep_bits(seed, stream, M, H, p)
    if (M * H // 8) % 4 == 0:                      # the generator kernel writes whole 32-bit words
        assert torch.equal(K.dropout_mask(M, H, p, seed, stream, "cuda"), bits)
    base = None
    for det in (False, True):
        monkeypatch.setenv("B200_DETERMINISTIC", "1" if det else "0")
        for km in (None, bits):
            dx, dxd, acc = _run_ln_bwd(K, dy, x, mean, rstd, gamma, starts, want_dropped=True, p_drop=p, seed=seed,
                                       drop_stream=stream, keep_mask=km)
            if base is None:
                base = (dx, dxd)
            else:                                  # the keep bits read from memory are the regenerated ones
                assert torch.equal(dx, base[0]) and torch.equal(dxd, base[1])
            tag = f"LN bwd H={H} M={M} {'det' if det else 'default'} {'keep_mask' if km is not None else 'philox'}"
            _check_ln_bwd(tag, M, H, 1 if det else 8, dy, x, mean, rstd, gamma, dx, dxd, acc, starts, keep_out=keep, p=p)


@pytest.mark.parametrize("H", [256, 320, 768, 1032])
def test_layer_norm_bwd_optional_outputs_and_p0(H, monkeypatch):
    """Each column sum as None in turn; want_dropped=False leaves dbias untouched; p = 0 gives dx_dropped == dx."""
    M = _bwd_sweep(H) + 1
    K, x, gamma, mean, rstd, dy, starts = _bwd_inputs(M, H, H + 5)
    for det in (False, True):
        monkeypatch.setenv("B200_DETERMINISTIC", "1" if det else "0")
        Z = 1 if det else 8
        for none in range(3):
            st = [None if k == none else starts[k] for k in range(3)]
            dx, dxd, acc = _run_ln_bwd(K, dy, x, mean, rstd, gamma, st, want_dropped=True, p_drop=0.1, seed=3,
                                       drop_stream=7)
            _check_ln_bwd(f"LN bwd H={H} no {('dgamma', 'dbeta', 'dbias')[none]} det={det}", M, H, Z, dy, x, mean, rstd,
                          gamma, dx, dxd, acc, st, keep_out=_keep(3, 7, M, H, 0.1), p=0.1)
        dx, dxd, acc = _run_ln_bwd(K, dy, x, mean, rstd, gamma, starts, want_dropped=False, p_drop=0.1, seed=3,
                                   drop_stream=7)
        assert dxd is None
        _check_ln_bwd(f"LN bwd H={H} no dropped det={det}", M, H, Z, dy, x, mean, rstd, gamma, dx, None, acc, starts)
        dx0, dxd0, acc = _run_ln_bwd(K, dy, x, mean, rstd, gamma, starts, want_dropped=True, p_drop=0.0)
        assert torch.equal(dx0, dxd0) and torch.equal(dx0, dx)
        _check_ln_bwd(f"LN bwd H={H} p=0 det={det}", M, H, Z, dy, x, mean, rstd, gamma, dx0, dxd0, acc, starts)


@pytest.mark.parametrize("H", [256, 768, 1024, 320])
@pytest.mark.parametrize("rows", ["g+1", "sweep+1"])
def test_layer_norm_bwd_input_dropout_matches_fp64(H, rows):
    """in_stream (the embedding LayerNorm, whose output was dropped out): dy times the stream's keep bits and scale.
    This always runs the TAIL kernel, H = 256 / 768 / 1024 included."""
    M = _rows(rows, _bwd_sweep(H), _groups(H))
    K, x, gamma, mean, rstd, dy, starts = _bwd_inputs(M, H, H * 3 + M)
    p, seed = 0.1, 99
    dx, dxd, acc = _run_ln_bwd(K, dy, x, mean, rstd, gamma, starts, p_drop=p, seed=seed, in_stream=EMB_STREAM)
    assert dxd is None
    _check_ln_bwd(f"LN bwd in_stream H={H} M={M}", M, H, 8, dy, x, mean, rstd, gamma, dx, None, acc, starts,
                  keep_in=_keep(seed, EMB_STREAM, M, H, p), p=p)


# ---------------------------------------------------------------------------------------------------------------------
# 3. embedding forward
# ---------------------------------------------------------------------------------------------------------------------
def _tables(V, P, H, gen):
    word = torch.randn(V, H, device="cuda", generator=gen).bfloat16()
    pos = (torch.randn(P, H, device="cuda", generator=gen) * 0.5).bfloat16()
    typ = (torch.randn(2, H, device="cuda", generator=gen) * 0.5).bfloat16()
    return word, pos, typ


@pytest.mark.parametrize("form", ["padded", "packed", "no-type"])
@pytest.mark.parametrize("H", [64, 256, 320, 768, 1024, 1032, 2048])
def test_embedding_fwd_matches_fp64(H, form):
    """CHUNKS 1 / 2 / 3 / 4 / 8 and the col < H tails.  padded: position row % S, M not a multiple of 4 and above the
    grid cap; packed: pos_ids in arbitrary order; no-type: type=None.  Ids include the last vocabulary row."""
    K = _api()
    V, S, p, seed = 1000, 128, 0.1, 555
    M = {"padded": _emb_sweep() + 7, "packed": 1001, "no-type": 130}[form]
    gen = torch.Generator(device="cuda").manual_seed(H * 13 + M)
    word, pos, typ = _tables(V, S, H, gen)
    gamma, beta = _gamma_beta(H, gen)
    ids = torch.randint(0, V, (M,), device="cuda", generator=gen, dtype=torch.int32)
    ids[::17] = V - 1
    seg = torch.randint(0, 2, (M,), device="cuda", generator=gen, dtype=torch.int32)
    pos_ids = torch.randint(0, S, (M,), device="cuda", generator=gen, dtype=torch.int32) if form == "packed" else None
    t = None if form == "no-type" else typ
    y, e, mean, rstd = K.embedding_fwd(ids, seg, word, pos, t, gamma, beta, S, p_drop=p, seed=seed, stream=EMB_STREAM,
                                       pos_ids=pos_ids)
    prow = pos_ids if pos_ids is not None else torch.arange(M, device="cuda", dtype=torch.int32) % S
    assert torch.equal(e, embed_sum_ref(word, pos, t, ids, prow, seg)), "e must be bf16((word + pos) + type)"
    from bert_pytorch_b200.utils import philox
    _check_ln_output(f"embedding H={H} {form}", y, mean, rstd, e, gamma, beta, roundings=3,
                     keep=_keep(seed, EMB_STREAM, M, H, p), scale=philox.keep_scale(p))


# ---------------------------------------------------------------------------------------------------------------------
# 4. embedding backward
# ---------------------------------------------------------------------------------------------------------------------
def _check_table(tag, got, start, key, de, chain=None, absum=None):
    """|got - (start + index_add)| <= chain u (|start| + sum |terms|) per entry; chain = the entry's term count + 1 (any
    summation order) unless given"""
    ref = scatter_ref(start, key, de)
    if absum is None:
        absum = torch.zeros_like(ref).index_add(0, key.long(), de.double().abs())
    if chain is None:
        chain = (torch.bincount(key.long(), minlength=start.size(0)).double() + 1)[:, None]
    bound = chain * U * (start.double().abs() + absum) * HIGHER_ORDER
    _report(tag, (got.double() - ref).abs(), bound)


def _bwd_case(M, H, V, S, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    de = torch.randn(M, H, device="cuda", generator=gen).bfloat16()
    ids = torch.randint(0, V, (M,), device="cuda", generator=gen, dtype=torch.int32)
    seg = torch.randint(0, 2, (M,), device="cuda", generator=gen, dtype=torch.int32)
    starts = [torch.randn(n, H, device="cuda", generator=gen) for n in (V, S, 2)]
    return gen, de, ids, seg, starts


@pytest.mark.parametrize("form", ["packed", "packed-no-seg", "ragged", "no-type"])
@pytest.mark.parametrize("H", [64, 320, 1032])
def test_embedding_bwd_atomic_scatter_matches_fp64(H, form, monkeypatch):
    """Every table row by atomics: packed rows (pos_ids), a ragged batch (M % S != 0), gtype=None; without segment ids
    every row is token type 0."""
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    K = _api()
    V, S = 300, 128
    M = 3 * S + 5 if form == "ragged" else 1001
    gen, de, ids, seg, starts = _bwd_case(M, H, V, S, H + M)
    pos_ids = torch.randint(0, S, (M,), device="cuda", generator=gen, dtype=torch.int32) if "packed" in form else None
    if form == "packed-no-seg":
        seg = None
    gw, gp, gt = (s.clone() for s in starts)
    K.embedding_bwd_scatter(de, ids, seg, gw, gp, None if form == "no-type" else gt, S, pos_ids=pos_ids)
    prow = pos_ids if pos_ids is not None else torch.arange(M, device="cuda", dtype=torch.int32) % S
    tkey = seg if seg is not None else torch.zeros(M, dtype=torch.int32, device="cuda")
    _check_table(f"emb bwd {form} H={H} word", gw, starts[0], ids, de)
    _check_table(f"emb bwd {form} H={H} pos", gp, starts[1], prow, de)
    if form == "no-type":
        assert torch.equal(gt, starts[2])
    else:
        _check_table(f"emb bwd {form} H={H} type", gt, starts[2], tkey, de)


@pytest.mark.parametrize("S", [100, 128, 512])
@pytest.mark.parametrize("H", [64, 320, 1032])
def test_embedding_bwd_position_type_reduction_matches_fp64(H, S, monkeypatch):
    """Padded batch: position rows summed over the batch by their one owner, the two token-type rows as
    type 1 = sum m f and type 0 = sum f - type 1 over the batch, 8 positions of a block, then one atomic per block.
    Bound of a type entry: its value comes from sums over every row (both types) at a chain of B (batch) + 1 (the
    difference) + 8 (positions of a block) + ceil(S / 8) (block atomics) + 1 (the starting value)."""
    monkeypatch.setenv("B200_DETERMINISTIC", "0")
    K = _api()
    V, B = 300, 3
    M = B * S
    gen, de, ids, seg, starts = _bwd_case(M, H, V, S, H * 5 + S)
    for with_type in (True, False):
        gw, gp, gt = (s.clone() for s in starts)
        K.embedding_bwd_scatter(de, ids, seg, gw, gp, gt if with_type else None, S)
        prow = torch.arange(M, device="cuda", dtype=torch.int32) % S
        _check_table(f"emb bwd postype H={H} S={S} word", gw, starts[0], ids, de)
        _check_table(f"emb bwd postype H={H} S={S} pos", gp, starts[1], prow, de)
        if with_type:
            _check_table(f"emb bwd postype H={H} S={S} type", gt, starts[2], seg, de,
                         chain=B + 10 + (S + 7) // 8, absum=de.double().abs().sum(0)[None, :].expand(2, H))
        else:
            assert torch.equal(gt, starts[2])


@pytest.mark.parametrize("M", [1, 63, 64, 65, 4097])
@pytest.mark.parametrize("H", [64, 1032, 2048])
def test_embedding_bwd_sorted_scatter_matches_fp64(H, M, monkeypatch):
    """Deterministic mode: rows sorted by table row, tiles of 64 sorted rows, the (H + 1023) / 1024 column split; a run
    of one id crossing several tiles; gtype=None.  Its chains (piece sums, then one add per tile) are at most the
    entry's term count + 1."""
    monkeypatch.setenv("B200_DETERMINISTIC", "1")
    K = _api()
    V, S = 300, 128
    gen, de, ids, seg, starts = _bwd_case(M, H, V, S, H * 11 + M)
    if M > 300:
        ids[40:300] = 7                            # one id over rows 40 .. 299: five 64-row tiles
    for with_type in (True, False):
        gw, gp, gt = (s.clone() for s in starts)
        K.embedding_bwd_scatter(de, ids, seg, gw, gp, gt if with_type else None, S)
        prow = torch.arange(M, device="cuda", dtype=torch.int32) % S
        _check_table(f"emb bwd sorted H={H} M={M} word", gw, starts[0], ids, de)
        _check_table(f"emb bwd sorted H={H} M={M} pos", gp, starts[1], prow, de)
        if with_type:
            _check_table(f"emb bwd sorted H={H} M={M} type", gt, starts[2], seg, de)
        else:
            assert torch.equal(gt, starts[2])


# ---------------------------------------------------------------------------------------------------------------------
# 5. refusals of the bindings, and empty batches
# ---------------------------------------------------------------------------------------------------------------------
def _ext():
    from bert_pytorch_b200 import ops
    return ops.extension()


def test_bindings_refuse_shapes_the_kernels_cannot_take():
    K, C = _api(), _ext()
    dev = "cuda"
    f32 = lambda *s: torch.zeros(*s, device=dev)
    bf = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bfloat16)
    i32 = lambda n: torch.zeros(n, device=dev, dtype=torch.int32)
    M, H = 64, 256
    x, y = bf(M, H), bf(M, H)
    # LayerNorm: lengths of gamma / beta / mean / rstd and of the column sums
    for g, b, m, r in [(f32(H - 8), f32(H), f32(M), f32(M)), (f32(H), f32(H + 8), f32(M), f32(M)),
                       (f32(H), f32(H), f32(M - 1), f32(M)), (f32(H), f32(H), f32(M), f32(M + 1))]:
        with pytest.raises(RuntimeError):
            C.layer_norm_fwd(x, g, b, y, m, r, EPS, None, None, False)
    ws = f32(C.ln_bwd_workspace(M, H))
    ok = dict(mean=f32(M), rstd=f32(M), gamma=f32(H))
    for bad in [dict(mean=f32(M - 1)), dict(rstd=f32(2 * M)), dict(gamma=f32(H - 8))]:
        a = {**ok, **bad}
        with pytest.raises(RuntimeError):
            C.layer_norm_bwd(x, x, a["mean"], a["rstd"], a["gamma"], bf(M, H), None, None, None, None, ws, 0.0, 0, 0,
                             K.NO_STREAM, None, None, False, None, False)
    for k in range(3):
        acc = [f32(H), f32(H), f32(H)]
        acc[k] = f32(H - 8)
        with pytest.raises(RuntimeError):
            C.layer_norm_bwd(x, x, f32(M), f32(M), f32(H), bf(M, H), bf(M, H), acc[0], acc[1], acc[2], ws, 0.0, 0, 0,
                             K.NO_STREAM, None, None, False, None, False)
    # embedding: H beyond the LayerNorm kernels, H % 8 != 0 (misaligned 16-byte rows), in both backward modes
    for Hb in (2056, 100):
        ids = i32(M)
        with pytest.raises(RuntimeError):
            K.embedding_fwd(ids, ids, bf(10, Hb), bf(10, Hb), bf(2, Hb), f32(Hb), f32(Hb), 8)
        for det in (False, True):
            with pytest.raises(RuntimeError):
                C.embedding_bwd_scatter(bf(M, Hb), ids, ids, f32(10, Hb), f32(8, Hb), f32(2, Hb), 8, None, det)
    # colsum: N % 8, unit column stride, 16-byte aligned rows -- in both modes
    wide = bf(M, 1020)
    for bad in (bf(M, 1020), wide[:, :1016], bf(1024, M).t()):
        for det in (False, True):
            with pytest.raises(RuntimeError):
                C.colsum(bad, f32(bad.size(1)), det)
    torch.cuda.synchronize()


def test_empty_batches_launch_nothing_and_leave_accumulators_alone(monkeypatch):
    K = _api()
    H, V, S = 320, 50, 16
    gen = torch.Generator(device="cuda").manual_seed(0)
    gamma, beta = _gamma_beta(H, gen)
    x = torch.zeros(0, H, device="cuda", dtype=torch.bfloat16)
    y, mean, rstd = K.layer_norm_fwd(x, gamma, beta)
    assert y.shape == (0, H) and mean.numel() == 0 and rstd.numel() == 0
    starts = [torch.randn(H, device="cuda", generator=gen) for _ in range(3)]
    word, pos, typ = _tables(V, S, H, gen)
    ids = torch.zeros(0, device="cuda", dtype=torch.int32)
    tables = [torch.randn(n, H, device="cuda", generator=gen) for n in (V, S, 2)]
    for det in ("0", "1"):
        monkeypatch.setenv("B200_DETERMINISTIC", det)
        acc = [s.clone() for s in starts]
        dx, dxd = K.layer_norm_bwd(x, x, mean, rstd, gamma, dgamma=acc[0], dbeta=acc[1], dbias=acc[2],
                                   want_dropped=True, p_drop=0.1, seed=1, drop_stream=2)
        assert dx.shape == (0, H) and dxd.shape == (0, H)
        ye, e, me, re = K.embedding_fwd(ids, ids, word, pos, typ, gamma, beta, S, p_drop=0.1, seed=1, stream=EMB_STREAM)
        assert ye.shape == (0, H) and e.shape == (0, H) and me.numel() == 0
        g = [t.clone() for t in tables]
        K.embedding_bwd_scatter(x, ids, ids, g[0], g[1], g[2], S)
        cs = starts[0].clone()
        K.colsum_accumulate(x, cs)
        torch.cuda.synchronize()
        for a, s in zip(acc + g + [cs], starts + tables + [starts[0]]):
            assert torch.equal(a, s)
