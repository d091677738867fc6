"""The bf16 wgmma GEMM (ops/csrc/gemm_sm90.cu) against exact and fp64 references: every (operand form, epilogue)
kernel that is built, at both tile widths, at the BERT-large engine shapes, the head shapes and ragged shapes.

1. Exact.  Operands are small integers ([-3, 3]), which bf16 holds exactly, so every partial sum is an integer below
   2^24 and the fp32 accumulator is exact in any order, split-K atomics included.  The expected output is then known
   bit for bit: the kernel's fp32 epilogue sequence (alpha * acc rounded to fp32, + bias, x keep x scale, + residual or
   x saved factor) applied in torch fp32 to the exact accumulator and rounded once to bf16.  A misplaced element, a
   dropped or doubled K slice, a wrong bias / residual / keep bit or a wrong alpha fails outright.  A, B, the bias and
   the residual are windows of larger NaN-filled tensors (pitch > K, > M or > N), so a tensor map that reads past the
   logical dims poisons the result; out and aux_out are windows of sentinel-filled tensors whose bytes outside [M, N]
   must stay untouched.
2. Rounding.  bf16 N(0, 1) operands against fp64: |out - ref| <= C_BOUND (|A| @ |B| + the epilogue terms) + r |ref|
   elementwise, r = 2^-8 for bf16 outputs (their own rounding) and 0 for fp32 outputs.  Every case also asserts that the
   same bound rejects the reference with its last 16-wide K slice dropped and, where there is a bias, with the bias
   left off the last 8-column group.  GELU / GELU' and tanh are held to 1.5 bf16 ulps of the fp64 function of the
   kernel's own pre-activation.
3. Each epilogue feature on its own (alpha, mask_in, regenerated keep bits, mask_out, p_drop = 0, out aliasing res,
   column sums, every split-K factor), the argument refusals of the binding, and a guard that the table below lists
   every kernel that is built."""
import math
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# Every bf16 (operand form, epilogue) pair gemm_sm90.cu builds; each runs at both tile widths (26 kernels)
KERNELS = [("NT", "none"), ("NT", "bias"), ("NT", "bias_drop_res"), ("NT", "add"), ("NT", "mul"),
           ("NT", "bias_gelu_dg"), ("NT", "bias_tanh"), ("NT", "f32"),
           ("NN", "none"), ("NN", "add"), ("NN", "mul"),
           ("TN", "accum_f32"), ("TN", "f32")]
KERNEL_IDS = [f"{l}-{e}" for l, e in KERNELS]
TILES = [128, 256]
EPI_NAMES = ["none", "bias", "bias_drop_res", "add", "accum_f32", "bias_tanh", "f32", "bias_gelu_dg", "mul"]

# Measured on H100 SXM (80 GB HBM3, 700 W) over every case of test_rounding_against_fp64: worst c = 1.1e-6 (TN
# EPI_ACCUM_F32 with the automatic split-K, K = 12288), 6.7e-7 at K = 30528 (MLM dgrad), <= 1e-7 at K = 1024 with a
# bf16 output; GELU / GELU' and tanh at most 0.73 bf16 ulp.  C_BOUND leaves a margin of 3.6 over the worst case.
C_BOUND = 4e-6
R_BF16 = 2.0 ** -8
ULP_BOUND = 1.5

DEV = "cuda"
SENT16 = 0x7BAD                 # bf16 bit pattern around the output windows
SENT32 = 0x7FBADBAD             # fp32 bit pattern (a NaN) around the fp32 output windows
P_DROP, SEED, STREAM = 0.1, 0x5EED0042, 7

# M = 12288 tokens (phase 1: 96 x 128), H = 1024, I = 4096; the MLM head sees 1920 masked rows (96 x 20)
T, H, I, V, ROWS = 12288, 1024, 4096, 30528, 1920
# ragged M (one 64-row fragment of a 128-row tile: M < 64 and 64 < M < 128), N (a single partial staged subtile: N <
# 64) and K (tails of the 64-wide k-block); fewer units than SMs, and several units per CTA (12290 x 1000)
RAGGED = [(1, 264, 72), (63, 56, 1040), (65, 136, 8), (127, 8, 520), (129, 248, 16), (12290, 1000, 56),
          (63, 72, 16), (129, 1000, 520)]
ENGINE = {
    ("NT", "none"): [(4096, H, H)],
    ("NT", "bias"): [(T, 3 * H, H), (ROWS, H, H), (ROWS, V, H)],    # QKV, MLM transform, MLM logits
    ("NT", "bias_drop_res"): [(T, H, H), (T, H, I)],                 # attention output, FFN-2 (+ mask_in)
    ("NT", "add"): [(4096, H, H)],
    ("NT", "mul"): [(4096, H, H)],
    ("NT", "bias_gelu_dg"): [(T, I, H)],                             # FFN-1
    ("NT", "bias_tanh"): [(8, H, H), (96, H, H)],                    # pooler at batch 8 and 96
    ("NT", "f32"): [(4096, 8, H)],                                   # head_linear forward, N = 8
    ("NN", "none"): [(T, H, H), (ROWS, H, V), (8, H, H), (96, H, H), (4096, H, 8)],   # attn-out, MLM, pooler, head
    ("NN", "add"): [(T, H, 3 * H), (T, H, I)],                       # QKV and FFN-1 dgrad
    ("NN", "mul"): [(T, I, H)],                                      # FFN-2 dgrad (x gelu')
    ("TN", "accum_f32"): [(3 * H, H, T), (I, H, T), (H, I, T), (H, H, 96), (V, H, ROWS)],   # wgrads
    ("TN", "f32"): [(8, H, 4096), (H, H, 4096)],                     # head_linear wgrad (M = 8), K-FAC x^T x
}


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _epi(name):
    api = _api()
    return {"none": api.EPI_NONE, "bias": api.EPI_BIAS, "bias_drop_res": api.EPI_BIAS_DROP_RES, "add": api.EPI_ADD,
            "accum_f32": api.EPI_ACCUM_F32, "bias_tanh": api.EPI_BIAS_TANH, "f32": api.EPI_F32,
            "bias_gelu_dg": api.EPI_BIAS_GELU_DG, "mul": api.EPI_MUL}[name]


def _layout(name):
    api = _api()
    return {"NT": api.NT, "NN": api.NN, "TN": api.TN}[name]


HAS_BIAS = ("bias", "bias_drop_res", "bias_tanh", "bias_gelu_dg")
HAS_RES = ("bias_drop_res", "add", "mul")
F32_OUT = ("f32", "accum_f32")


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\n[bf16 gemm reference] file wall time {time.perf_counter() - t0:.1f} s")


def _shapes(kern):
    return RAGGED + ENGINE[kern]


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def _values(shape, exact, g, scale=1.0):
    if exact:
        return torch.randint(-3, 4, shape, device=DEV, generator=g).to(torch.bfloat16)
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


def _poisoned(v):
    """``v`` as a window of a larger tensor whose every other element is NaN: a NaN row above and three below, eight
    NaN columns to the left and a row pitch of at least 16 more columns (a multiple of 8)."""
    if v.dim() == 1:
        buf = torch.full((v.numel() + 16,), float("nan"), dtype=v.dtype, device=DEV)
        w = buf[8:8 + v.numel()]
    else:
        r, c = v.shape
        buf = torch.full((r + 4, (c + 7) // 8 * 8 + 24), float("nan"), dtype=v.dtype, device=DEV)
        w = buf[1:1 + r, 8:8 + c]
    w.copy_(v)
    return w


def _framed(rows, cols, dtype):
    """(frame, window): a [rows, cols] window of a larger tensor whose every element holds the sentinel"""
    if dtype == torch.float32:
        full = torch.full((rows + 2, cols + 24), SENT32, dtype=torch.int32, device=DEV).view(torch.float32)
    else:
        full = torch.full((rows + 2, cols + 24), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return full, full[1:1 + rows, 8:8 + cols]


def _outside_untouched(full, rows, cols):
    bits = full.view(torch.int32 if full.dtype == torch.float32 else torch.int16).clone()
    sent = SENT32 if full.dtype == torch.float32 else SENT16
    bits[1:1 + rows, 8:8 + cols] = sent
    return bool((bits == sent).all())


class Case:
    """Operands of one call in their stored form (a, b) and as the logical A [M, K] and B [K, N]."""

    def __init__(self, layout, epi, M, N, K, exact, g, poison, a_scale=1.0):
        self.layout, self.epi, self.M, self.N, self.K = layout, epi, M, N, K
        shape_a = {"NT": (M, K), "NN": (M, K), "TN": (K, M)}[layout]
        shape_b = {"NT": (N, K), "NN": (K, N), "TN": (K, N)}[layout]
        a, b = _values(shape_a, exact, g, a_scale), _values(shape_b, exact, g)
        self.bias = self.res = self.base = None
        if epi in HAS_BIAS:
            self.bias = _values((N,), exact, g, 2.0)
        if epi in HAS_RES:
            self.res = _values((M, N), exact, g)
        if epi == "accum_f32":                       # the gradient accumulated into: integer-valued when exact
            self.base = (torch.randint(-50, 51, (M, N), device=DEV, generator=g).float() if exact
                         else torch.randn(M, N, device=DEV, generator=g))
        if poison:
            a, b = _poisoned(a), _poisoned(b)
            self.bias = _poisoned(self.bias) if self.bias is not None else None
            self.res = _poisoned(self.res) if self.res is not None else None
        self.a, self.b = a, b
        self.A = a.t() if layout == "TN" else a
        self.B = b.t() if layout == "NT" else b

    def prod(self, rows=None, k_from=0):
        """fp64 A[rows, k_from:] @ B[k_from:] and |A| @ |B| over the same range"""
        A = self.A if rows is None else self.A[rows]
        A, B = A[:, k_from:].double(), self.B[k_from:].double()
        return A @ B, A.abs() @ B.abs()


def _keep_from_bits(mask, M, N):
    return ((mask.unsqueeze(-1) >> torch.arange(8, device=DEV, dtype=torch.uint8)) & 1).reshape(M, N).bool()


def _philox_keep(M, N, p=P_DROP, seed=SEED, stream=STREAM):
    from bert_pytorch_b200.utils import philox
    return torch.from_numpy(philox.keep_mask(seed, stream, M * N, p)).view(M, N).to(DEV)


def _drop_scale32(p=P_DROP):
    one = torch.tensor(65536.0, device=DEV)          # launch(): 65536.f / (65536.f - thresh16), in fp32
    return one / (one - float(int(p * 65536.0 + 0.5)))


def _run(case, bn, alpha, out=None, aux=None, mask_in=None, p=P_DROP, **kw):
    """the kernel of (case.layout, case.epi) on the case's operands; returns out"""
    api = _api()
    e = case.epi
    args = dict(layout=_layout(case.layout), epi=_epi(e), block_n=bn, alpha=alpha)
    if case.bias is not None:
        args["bias"] = case.bias
    if case.res is not None:
        args["res"] = case.res
    if e == "bias_drop_res":
        args.update(p_drop=p, seed=SEED, stream=STREAM)
        if mask_in is not None:
            args["mask_in"] = mask_in
    if e == "bias_gelu_dg":
        args["aux_out"] = aux
    if e == "accum_f32":
        out.copy_(case.base)
    args.update(kw)
    return api.gemm(case.a, case.b, out=out, **args)


def _gelu64(x):
    Phi = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))
    phi = torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    return x * Phi, Phi + x * phi


def _bf16_ulp_err(out, ref):
    """max |out - ref| in bf16 ulps of the fp64 reference (the ulp floored at that of 2^-14: below it the activation is
    smaller than anything the next GEMM resolves against O(1) neighbours)"""
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 7)
    return ((out.double() - ref).abs() / ulp).max().item()


def _act_refs(epi, x):
    """fp64 reference outputs of the activation epilogues from their fp32 pre-activation x: [out] or [out, aux]"""
    if epi == "bias_tanh":
        return [torch.tanh(x.double())]
    return list(_gelu64(x.double()))


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact
# ---------------------------------------------------------------------------------------------------------------------
def _exact_expected(case, alpha, acc, keep):
    """the kernel's fp32 epilogue on the exact fp32 accumulator: bf16 output (rounded once), fp32 output, or the fp32
    pre-activation of tanh / GELU"""
    e = case.epi
    f = acc * alpha                                  # __fmul_rn(acc, alpha)
    if e == "accum_f32":
        return case.base + f
    if e == "f32":
        return f
    if case.bias is not None:
        f = f + case.bias.float()
    if e in ("bias_tanh", "bias_gelu_dg"):
        return f
    if e == "bias_drop_res":
        f = torch.where(keep, f * _drop_scale32(), torch.zeros_like(f)) + case.res.float()
    elif e == "add":
        f = f + case.res.float()
    elif e == "mul":
        f = f * case.res.float()
    return f.to(torch.bfloat16)


def _exact_case(layout, epi, M, N, K, bn, alpha, g, use_mask_in=False, wgrad=False):
    """One exact call on poisoned operands into sentinel-framed outputs; returns a list of failure strings."""
    api = _api()
    tag = f"{layout}-{epi} bn{bn} {M}x{N}x{K} alpha={alpha}"
    case = Case(layout, epi, M, N, K, True, g, poison=True)
    dtype = torch.float32 if epi in F32_OUT else torch.bfloat16
    full, out = _framed(M, N, dtype)
    aux_full, aux = _framed(M, N, torch.bfloat16) if epi == "bias_gelu_dg" else (None, None)
    mask_in, keep = None, None
    if epi == "bias_drop_res":
        if use_mask_in:
            mask_in = api.dropout_mask(M, N, P_DROP, SEED, STREAM, DEV)
            keep = _keep_from_bits(mask_in, M, N)
        else:
            keep = _philox_keep(M, N)
    if wgrad:                                        # the engine's entry point: its own tile width and split-K
        out.copy_(case.base)
        api.wgrad_accumulate(case.a, case.b, out, alpha=alpha)
    else:
        _run(case, bn, alpha, out=out, aux=aux, mask_in=mask_in)
    torch.cuda.synchronize()
    fails = []
    if not _outside_untouched(full, M, N):
        fails.append(f"{tag}: out written outside [M, N]")
    if aux_full is not None and not _outside_untouched(aux_full, M, N):
        fails.append(f"{tag}: aux_out written outside [M, N]")
    prod, _ = case.prod()
    acc = prod.float()
    assert torch.equal(acc.double(), prod), tag      # the exact accumulator is an fp32 value
    want = _exact_expected(case, alpha, acc, keep)
    if epi == "accum_f32":
        assert torch.equal(want.double(), case.base.double() + alpha * prod), tag   # no rounding in the expectation
    if not bool(torch.isfinite(out).all()):
        fails.append(f"{tag}: non-finite output (a NaN outside a window was read)")
    elif epi in ("bias_tanh", "bias_gelu_dg"):
        refs = _act_refs(epi, want)
        for name, got, ref in zip(("out", "aux"), (out, aux), refs):
            err = _bf16_ulp_err(got, ref)
            if not err <= ULP_BOUND:
                fails.append(f"{tag}: {name} {err:.2f} bf16 ulps from fp64")
    elif dtype == torch.float32:
        if not torch.equal(out, want):
            fails.append(f"{tag}: {int((out != want).sum())} fp32 elements differ")
    elif not torch.equal(out.float(), want.float()):        # by value: an all-(-0) product may sum to either zero
        bad = (out.float() != want.float()).nonzero()[:4].tolist()
        fails.append(f"{tag}: {int((out.float() != want.float()).sum())} bf16 elements differ, first at {bad}")
    return fails


@pytest.mark.parametrize("bn", TILES)
@pytest.mark.parametrize("kern", KERNELS, ids=KERNEL_IDS)
def test_exact_integer_operands(kern, bn):
    """Bit-exact outputs on NaN-padded operand windows, nothing written outside the [M, N] window, at the ragged, engine
    and head shapes; alpha alternates between 0.75 and 1."""
    layout, epi = kern
    g = torch.Generator(device=DEV).manual_seed(1000 + KERNELS.index(kern) * 2 + bn)
    fails = []
    for i, (M, N, K) in enumerate(_shapes(kern)):
        engine = (M, N, K) in ENGINE[kern]
        fails += _exact_case(layout, epi, M, N, K, bn, 0.75 if i % 2 == 0 else 1.0, g,
                             use_mask_in=engine and epi == "bias_drop_res",
                             wgrad=engine and epi == "accum_f32" and bn == 256)
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# 2. rounding against fp64
# ---------------------------------------------------------------------------------------------------------------------
def _ref64(case, alpha, prod, absprod, rows, keep, bias=None):
    """fp64 reference and its error scale |A| @ |B| + the epilogue terms, for the rows ``rows``"""
    e = case.epi
    bias = case.bias if bias is None else bias
    ref, absref = alpha * prod, abs(alpha) * absprod
    if e == "accum_f32":
        base = case.base[rows].double()
        return base + ref, absref + base.abs()
    if bias is not None:
        b = bias.double()
        ref, absref = ref + b, absref + b.abs()
    res = case.res[rows].double() if case.res is not None else None
    if e == "bias_drop_res":
        s = _drop_scale32().double()
        k = keep[rows]
        ref = torch.where(k, ref * s, torch.zeros_like(ref)) + res
        absref = torch.where(k, absref * s, torch.zeros_like(absref)) + res.abs()
    elif e == "add":
        ref, absref = ref + res, absref + res.abs()
    elif e == "mul":
        ref, absref = ref * res, absref * res.abs()
    return ref, absref


def _c_of(out, ref, absref, r):
    """smallest c with |out - ref| <= c absref + r |ref| everywhere (inf where absref == 0 and the error is not
    covered by r |ref|)"""
    slack = (out.double() - ref).abs() - r * ref.abs()
    pos = absref > 0
    if bool((slack[~pos] > 0).any()):
        return math.inf
    return max(0.0, (slack[pos] / absref[pos]).max().item()) if bool(pos.any()) else 0.0


def _rows_checked(M, N):
    """all rows, or the first and last 512 where the fp64 reference of the whole output would be large"""
    if M * N <= 8 * 2 ** 20:
        return torch.arange(M, device=DEV)
    return torch.cat([torch.arange(512, device=DEV), torch.arange(M - 512, M, device=DEV)])


def _rounding_case(layout, epi, M, N, K, bn, alpha, g):
    """returns (observed c or ulp error, failures)"""
    api = _api()
    tag = f"{layout}-{epi} bn{bn} {M}x{N}x{K}"
    act = epi in ("bias_tanh", "bias_gelu_dg")
    case = Case(layout, epi, M, N, K, False, g, poison=True, a_scale=1.0 / math.sqrt(K) if act else 1.0)
    keep = _philox_keep(M, N) if epi == "bias_drop_res" else None
    out = torch.empty(M, N, device=DEV, dtype=torch.float32 if epi in F32_OUT else torch.bfloat16)
    aux = torch.empty(M, N, device=DEV, dtype=torch.bfloat16) if epi == "bias_gelu_dg" else None
    _run(case, bn, alpha, out=out, aux=aux, **({"k_splits": -1} if epi == "accum_f32" else {}))
    rows = _rows_checked(M, N)
    prod, absprod = case.prod(rows)
    k0 = (K - 1) // 16 * 16                           # the last 16-wide K slice (ragged when K % 16 != 0)
    dropped, _ = case.prod(rows, k_from=k0)
    fails = []
    if act:
        # the pre-activation is the kernel's own: alpha * acc from the fp32 kernel of the same tile width, + bias; that
        # accumulator is held to the fp64 bound, the activation to 1.5 bf16 ulps of its fp64 value
        acc = api.gemm(case.a, case.b, epi=api.EPI_F32, alpha=alpha, block_n=bn)[rows]
        c = _c_of(acc, alpha * prod, alpha * absprod, 0.0)
        if not c <= C_BOUND:
            fails.append(f"{tag}: fp32 accumulator c = {c:.3e} > {C_BOUND:.1e}")
        x = acc + case.bias.float()
        refs = _act_refs(epi, x)
        worst = 0.0
        for name, got, ref in zip(("out", "aux"), (out, aux), refs):
            err = _bf16_ulp_err(got[rows], ref)
            worst = max(worst, err)
            if not err <= ULP_BOUND:
                fails.append(f"{tag}: {name} {err:.2f} bf16 ulps from fp64")
        # sensitivity: the ulp criterion rejects a dropped K slice and the bias left off the last 8-column group
        xb = x.double() - alpha * dropped
        bad = _act_refs(epi, xb)[0].to(torch.bfloat16)
        if not _bf16_ulp_err(bad, refs[0]) > ULP_BOUND:
            fails.append(f"{tag}: 1.5 ulps would not reject a dropped 16-wide K slice")
        xb = x.double().clone()
        xb[:, N - 8:] -= case.bias[N - 8:].double()
        if not _bf16_ulp_err(_act_refs(epi, xb)[0].to(torch.bfloat16), refs[0]) > ULP_BOUND:
            fails.append(f"{tag}: 1.5 ulps would not reject a bias missing from one 8-column group")
        print(f"[bf16 gemm] {tag}: accumulator c = {c:.3e}, activation {worst:.2f} ulp (C_BOUND = {C_BOUND:.1e})")
        return c, fails
    r = 0.0 if epi in F32_OUT else R_BF16
    ref, absref = _ref64(case, alpha, prod, absprod, rows, keep)
    c = _c_of(out[rows], ref, absref, r)
    print(f"[bf16 gemm] {tag}: c = {c:.3e} (C_BOUND = {C_BOUND:.1e})")
    if not c <= C_BOUND:
        fails.append(f"{tag}: c = {c:.3e} > {C_BOUND:.1e}")

    def rejects(bad):
        return bool((((bad - ref).abs() - r * ref.abs()) > C_BOUND * absref).any())

    if not rejects(_ref64(case, alpha, prod - dropped, absprod, rows, keep)[0]):
        fails.append(f"{tag}: the bound would not reject a dropped 16-wide K slice")
    if case.bias is not None:
        nob = case.bias.clone()
        nob[N - 8:] = 0
        if not rejects(_ref64(case, alpha, prod, absprod, rows, keep, bias=nob)[0]):
            fails.append(f"{tag}: the bound would not reject a bias missing from one 8-column group")
    return c, fails


@pytest.mark.parametrize("bn", TILES)
@pytest.mark.parametrize("kern", KERNELS, ids=KERNEL_IDS)
def test_rounding_against_fp64(kern, bn):
    """bf16 N(0, 1) operands: elementwise fp64 bound at every shape, with the bound's own sensitivity asserted."""
    layout, epi = kern
    g = torch.Generator(device=DEV).manual_seed(2000 + KERNELS.index(kern) * 2 + bn)
    fails = []
    for i, (M, N, K) in enumerate(_shapes(kern)):
        fails += _rounding_case(layout, epi, M, N, K, bn, 0.75 if i % 2 else 1.0, g)[1]
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# 3. epilogue features
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", TILES)
@pytest.mark.parametrize("kern", [k for k in KERNELS if k[1] in ("add", "mul", "bias_drop_res")],
                         ids=[f"{l}-{e}" for l, e in KERNELS if e in ("add", "mul", "bias_drop_res")])
def test_out_aliasing_res(kern, bn):
    """out may be the residual / saved factor itself: the result is the exact one computed from the original values."""
    layout, epi = kern
    g = torch.Generator(device=DEV).manual_seed(3000 + bn)
    fails = []
    for (M, N, K) in [(12290, 1000, 56), (65, 136, 72), (T, H, H)]:
        case = Case(layout, epi, M, N, K, True, g, poison=True)
        keep = _philox_keep(M, N) if epi == "bias_drop_res" else None
        want = _exact_expected(case, 0.75, case.prod()[0].float(), keep)
        _run(case, bn, 0.75, out=case.res)
        if not torch.equal(case.res.float(), want.float()):
            fails.append(f"{layout}-{epi} bn{bn} {M}x{N}x{K}")
    assert not fails, fails


@pytest.mark.parametrize("bn", TILES)
@pytest.mark.parametrize("layout", ["NT", "NN"])
@pytest.mark.parametrize("epi", ["none", "add", "mul"])
def test_colsum_exact(epi, layout, bn):
    """colsum (fragment epilogue for EPI_NONE, staged for EPI_ADD / EPI_MUL) equals the fp64 column sum of the bf16
    output exactly: operands in {-1, 0, 1} and K <= 256 keep |out| <= 257 on a quarter-integer grid, so every fp32
    partial sum is exact in any order."""
    g = torch.Generator(device=DEV).manual_seed(4000 + bn)
    fails = []
    for (M, N, K) in [(12290, 1000, 56), (63, 56, 16), (129, 264, 256), (65, 136, 8), (T, H, 256)]:
        case = Case(layout, epi, M, N, K, True, g, poison=True)
        case.a.clamp_(-1, 1)
        case.b.clamp_(-1, 1)
        if case.res is not None:
            case.res.clamp_(-1, 1)
        base = torch.randint(-100, 101, (N,), device=DEV, generator=g).float()
        cs = base.clone()
        out = _run(case, bn, 0.75, colsum=cs)
        want = _exact_expected(case, 0.75, case.prod()[0].float(), None)
        if not torch.equal(out, want):
            fails.append(f"{M}x{N}x{K}: output")
        if not torch.equal(cs.double(), base.double() + out.double().sum(0)):
            fails.append(f"{M}x{N}x{K}: colsum off by {(cs.double() - base.double() - out.double().sum(0)).abs().max()}")
    assert not fails, fails


@pytest.mark.parametrize("bn", TILES)
def test_accum_f32_every_split(bn):
    """EPI_ACCUM_F32 at every k_splits in 1..k_blocks, above k_blocks (clamped), at values that do not divide
    k_blocks, and at -1 (automatic) with one tile and with k_blocks < 4: exact on integer operands."""
    g = torch.Generator(device=DEV).manual_seed(5000 + bn)
    fails = []
    runs = [((136, 264, 520), s) for s in list(range(1, 10)) + [10, 64, -1]]       # 9 k-blocks: 2, 4, 5 ... uneven
    runs += [((127, 248, 1040), -1), ((127, 120, 4000), -1), ((12290, 1000, 192), -1), ((300, 264, 192), 3),
             ((65, 56, 72), 2), ((T, H, 512), 7)]
    for (M, N, K), s in runs:
        case = Case("TN", "accum_f32", M, N, K, True, g, poison=True)
        full, out = _framed(M, N, torch.float32)
        _run(case, bn, 0.75, out=out, k_splits=s)
        want = case.base + case.prod()[0].float() * 0.75
        if not torch.equal(out, want):
            fails.append(f"{M}x{N}x{K} k_splits={s}: {int((out != want).sum())} elements differ")
        if not _outside_untouched(full, M, N):
            fails.append(f"{M}x{N}x{K} k_splits={s}: written outside [M, N]")
    assert not fails, fails


@pytest.mark.parametrize("bn", TILES)
def test_dropout_keep_bits(bn):
    """EPI_BIAS_DROP_RES: the regenerated keep bits are philox.keep_bits (mask_out, written into a slice of a sentinel
    buffer at ragged M, nothing past M * N / 8 touched); mask_in is applied bit for bit and gives the regenerated
    output; p_drop = 0 keeps every element."""
    from bert_pytorch_b200.utils import philox
    g = torch.Generator(device=DEV).manual_seed(6000 + bn)
    for (M, N, K) in [(1999, 1024, 72), (63, 128, 520), (129, 384, 16)]:
        case = Case("NT", "bias_drop_res", M, N, K, True, g, poison=True)
        acc = case.prod()[0].float()
        nbytes = M * N // 8
        buf = torch.full((nbytes + 64,), 0xA5, dtype=torch.uint8, device=DEV)
        mask_out = buf[16:16 + nbytes].view(M, N // 8)
        regen = _run(case, bn, 0.75, mask_out=mask_out)
        torch.cuda.synchronize()
        assert bool((buf[:16] == 0xA5).all()) and bool((buf[16 + nbytes:] == 0xA5).all()), (M, N)
        bits = philox.keep_bits(SEED, STREAM, M, N, P_DROP)
        assert np.array_equal(mask_out.cpu().numpy(), bits), (M, N)
        keep = _philox_keep(M, N)
        assert torch.equal(regen, _exact_expected(case, 0.75, acc, keep)), (M, N)
        # mask_in: arbitrary bits (not the stream's) are applied exactly
        other = torch.randint(0, 256, (M, N // 8), dtype=torch.uint8, device=DEV, generator=g)
        via = _run(case, bn, 0.75, mask_in=other)
        assert torch.equal(via, _exact_expected(case, 0.75, acc, _keep_from_bits(other, M, N))), (M, N)
        assert torch.equal(_run(case, bn, 0.75, mask_in=mask_out), regen), (M, N)
        none = _run(case, bn, 0.75, p=0.0)
        assert torch.equal(none, ((acc * 0.75 + case.bias.float()) + case.res.float()).to(torch.bfloat16)), (M, N)


# ---------------------------------------------------------------------------------------------------------------------
# 4. argument refusals and the kernel table
# ---------------------------------------------------------------------------------------------------------------------
def _small(layout="NT", M=128, N=256, K=64):
    case = Case(layout, "none", M, N, K, False, None, poison=False)
    return case.a, case.b


def test_refuses_aux_out_of_wrong_shape_or_epilogue():
    api = _api()
    a, b = _small()
    bias = torch.zeros(256, dtype=torch.bfloat16, device=DEV)
    short = torch.empty(127, 256, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match=r"aux_out must be \[M, N\]"):
        api.gemm(a, b, epi=api.EPI_BIAS_GELU_DG, bias=bias, aux_out=short)
    with pytest.raises(RuntimeError, match="aux_out is not written"):
        api.gemm(a, b, epi=api.EPI_BIAS, bias=bias, aux_out=torch.empty(128, 256, dtype=torch.bfloat16, device=DEV))


def test_refuses_bias_the_epilogue_does_not_read():
    api = _api()
    a, b = _small()
    bias = torch.zeros(256, dtype=torch.bfloat16, device=DEV)
    for epi in (api.EPI_NONE, api.EPI_ADD, api.EPI_MUL, api.EPI_F32):
        kw = {"res": torch.zeros(128, 256, dtype=torch.bfloat16, device=DEV)} if epi == api.EPI_MUL else {}
        with pytest.raises(RuntimeError, match="bias is not read"):
            api.gemm(a, b, epi=epi, bias=bias, **kw)


def test_refuses_res_the_epilogue_does_not_read():
    api = _api()
    a, b = _small()
    res = torch.zeros(128, 256, dtype=torch.bfloat16, device=DEV)
    bias = torch.zeros(256, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="res is not read"):
        api.gemm(a, b, epi=api.EPI_NONE, res=res)
    with pytest.raises(RuntimeError, match="res is not read"):
        api.gemm(a, b, epi=api.EPI_BIAS, bias=bias, res=res)


def test_refuses_p_drop_without_dropout():
    api = _api()
    a, b = _small()
    res = torch.zeros(128, 256, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="applies no dropout"):
        api.gemm(a, b, epi=api.EPI_ADD, res=res, p_drop=0.1)


def test_refuses_k_splits_without_accumulate():
    api = _api()
    a, b = _small("TN")
    for s in (2, -1, 0):
        with pytest.raises(RuntimeError, match="needs EPI_ACCUM_F32"):
            api.gemm(a, b, layout=api.TN, epi=api.EPI_F32, k_splits=s)


def test_refuses_block_n_other_than_the_tile_widths():
    api = _api()
    a, b = _small()
    for bn in (0, 64, 512, 1024):
        with pytest.raises(RuntimeError, match="block_n must be 128 or 256"):
            api.gemm(a, b, block_n=bn)


def test_refuses_empty_reduction_unless_accumulating():
    """K == 0 would leave a plain output unwritten; accumulating an empty reduction leaves the target unchanged."""
    api = _api()
    a = torch.empty(128, 8, dtype=torch.bfloat16, device=DEV)[:, :0]
    b = torch.empty(256, 8, dtype=torch.bfloat16, device=DEV)[:, :0]
    with pytest.raises(RuntimeError, match="K == 0"):
        api.gemm(a, b)
    with pytest.raises(RuntimeError, match="K == 0"):
        api.gemm(a, b, epi=api.EPI_F32)
    at, bt = torch.empty(0, 128, dtype=torch.bfloat16, device=DEV), torch.empty(0, 256, dtype=torch.bfloat16, device=DEV)
    grad = torch.randn(128, 256, device=DEV)
    before = grad.clone()
    api.gemm(at, bt, layout=api.TN, epi=api.EPI_ACCUM_F32, out=grad)
    torch.cuda.synchronize()
    assert torch.equal(grad, before)


def test_kernel_table_lists_every_built_kernel():
    """Probe every (layout, epilogue) pair with a tiny call: the pairs that run are exactly the suite's table, so a newly
    built kernel without tests fails here."""
    api = _api()
    M, N, K = 64, 256, 64
    built = set()
    for layout in ("NT", "NN", "TN"):
        a, b = _small(layout, M, N, K)
        for e in EPI_NAMES:
            kw = dict(layout=_layout(layout), epi=_epi(e))
            if e in HAS_BIAS:
                kw["bias"] = torch.zeros(N, dtype=torch.bfloat16, device=DEV)
            if e in ("bias_drop_res", "mul"):
                kw["res"] = torch.zeros(M, N, dtype=torch.bfloat16, device=DEV)
            if e == "bias_gelu_dg":
                kw["aux_out"] = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
            if e == "accum_f32":
                kw["out"] = torch.zeros(M, N, device=DEV)
            for bn in TILES:
                try:
                    api.gemm(a, b, block_n=bn, **kw)
                except RuntimeError as err:
                    assert "no kernel" in str(err), (layout, e, str(err))
                    continue
                built.add((layout, e))
    torch.cuda.synchronize()
    assert built == set(KERNELS), (sorted(built - set(KERNELS)), sorted(set(KERNELS) - built))
