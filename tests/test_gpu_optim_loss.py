"""Optimizer kernels (ops/csrc/optim.cu) and loss heads (ops/csrc/loss.cu) against float64 references written here.

Every reference is computed in fp64 from exactly what the kernel reads: the fp32 arena and the fp32-rounded
hyper-parameters for LAMB / Adam, the bf16 logits for the softmax cross-entropy, the bf16 pooled output and
classifier weight (and fp32 bias) for the NSP head.  The tolerances are derived from the kernels' arithmetic (fp32
accumulation, bf16 output rounding); a failure is a kernel defect until shown otherwise.
"""
import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

CHUNK = 65536          # ops/api.py: a chunk of the optimizer's chunk table never exceeds this many elements
SENTINEL = -1.5 * 2 ** 20   # exact in bf16, so the shadow's padding can hold flat_param's padding value bit for bit


def _api():
    from bert_pytorch_b200 import ops
    from bert_pytorch_b200.ops import api
    assert ops.available()
    return api


def _f32(x: float) -> float:
    """The value a kernel receives for a host float hyper-parameter."""
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------------------------
# modules whose arena slots hit the chunking edges
# ------------------------------------------------------------------------------------------------------------------
class _SelfAttention(nn.Module):
    def __init__(self):
        super().__init__()
        # [7, 13] weights (91 elements) and 7-element biases: the q/k/v run is laid out gap-free, so the slots after
        # the first start at offsets 3, 2, 1, 0 and 3 mod 4 past an aligned one
        self.query, self.key, self.value = nn.Linear(13, 7), nn.Linear(13, 7), nn.Linear(13, 7)


class _Attention(nn.Module):
    def __init__(self):
        super().__init__()
        self.add_module("self", _SelfAttention())


class _Layer(nn.Module):
    def __init__(self):
        super().__init__()
        self.attention = _Attention()


class _Edges(nn.Module):
    """Slots of 1, 2, 3 and 5 elements (no float4 at all, or one plus a tail), exactly one chunk, one tensor spanning
    three chunks with a 5-element tail (unless ``span=False``), and an unaligned q/k/v run."""

    def __init__(self, span=True):
        super().__init__()
        r = lambda n: nn.Parameter(torch.randn(n) * 0.5)
        self.one, self.two, self.three, self.five = r(1), r(2), r(3), r(5)
        self.full = r(CHUNK)
        if span:
            self.span = r(2 * CHUNK + 5)
        self.layer = nn.ModuleList([_Layer()])
        with torch.no_grad():
            for p in self.layer.parameters():
                p.normal_(0.0, 0.5)

    def groups(self, wd):
        """One decaying and one non-decaying group (the weights decay; the biases and the three smallest slots
        do not)."""
        named = list(self.named_parameters())
        nd = lambda n: n.endswith("bias") or n in ("one", "two", "three")
        return [{"params": [p for n, p in named if not nd(n)], "weight_decay": wd},
                {"params": [p for n, p in named if nd(n)], "weight_decay": 0.0}]


def _tiny_bert():
    from bert_pytorch_b200 import BertConfig
    from bert_pytorch_b200.models import BertForPreTraining
    cfg = BertConfig(vocab_size_or_config_json_file=1024, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                     intermediate_size=256, max_position_embeddings=128, hidden_dropout_prob=0.0,
                     attention_probs_dropout_prob=0.0)
    model = BertForPreTraining(cfg)

    def groups(wd):
        named = list(model.named_parameters())
        nd = ("bias", "LayerNorm")
        return [{"params": [p for n, p in named if not any(k in n for k in nd)], "weight_decay": wd},
                {"params": [p for n, p in named if any(k in n for k in nd)], "weight_decay": 0.0}]
    model.groups = groups
    return model


def _module(kind):
    torch.manual_seed(0)
    m = {"edges": _Edges, "one_chunk": lambda: _Edges(span=False), "tiny_bert": _tiny_bert}[kind]()
    return m.cuda()


# ------------------------------------------------------------------------------------------------------------------
# fp64 references over the flat arena
# ------------------------------------------------------------------------------------------------------------------
def _slot_mask(arena):
    mask = torch.zeros(arena.numel, dtype=torch.bool, device=arena.device)
    for s in arena.slots:
        mask[s.offset:s.offset + s.numel] = True
    return mask


def _grads(arena, step, base, seed=0):
    """A gradient for every slot, zero in the padding.  Magnitudes are in [0.5, 1.5) x base x a per-step factor, with
    random signs: no exact zeros (m / (sqrt(v) + eps) stays well conditioned) and the moments carry history."""
    factor = (1.0, 0.25, 2.0, 0.5, 1.5, 1.0, 0.75)[step % 7]
    gen = torch.Generator(device="cuda").manual_seed(1000 * seed + step)
    mag = torch.rand(arena.numel, device="cuda", generator=gen, dtype=torch.float64) + 0.5
    sign = torch.randint(0, 2, (arena.numel,), device="cuda", generator=gen).to(torch.float64) * 2 - 1
    g = (mag * sign * base * factor).float()
    return torch.where(_slot_mask(arena), g, torch.zeros_like(g))


class _Ref:
    """fp64 copy of the optimizer state over the arena layout.  ``torch_consts``: the constants of the torch path,
    which forms 1 - beta in fp64 and rounds it to fp32 (the kernels subtract the fp32 beta from 1 in fp32; for
    beta2 = 0.999 the two differ by 1.3e-5 relative)."""

    def __init__(self, arena, torch_consts=False):
        self.slots = arena.slots
        self.torch_consts = torch_consts
        self.p = arena.flat_param.double().clone()
        self.m = torch.zeros_like(self.p)
        self.v = torch.zeros_like(self.p)

    def _one_minus(self, h, i):
        return _f32(1.0 - h["betas"][i]) if self.torch_consts else 1.0 - _f32(h["betas"][i])

    def _bc(self, h, i, step):
        if not h["bias_correction"]:
            return 1.0
        return 1.0 - (h["betas"][i] if self.torch_consts else _f32(h["betas"][i])) ** step

    def lamb(self, g, h, step):
        lr, (b1, b2), eps, wd = _f32(h["lr"]), map(_f32, h["betas"]), _f32(h["eps"]), _f32(h["wd"])
        gnorm = float(g.norm())
        mgn = _f32(h["max_grad_norm"])
        clip = gnorm / mgn if (mgn > 0 and gnorm > mgn) else 1.0
        bc1 = self._bc(h, 0, step)
        bc2 = self._bc(h, 1, step)
        beta3 = self._one_minus(h, 0) if h["grad_averaging"] else 1.0
        for s in self.slots:
            sl = slice(s.offset, s.offset + s.numel)
            d = wd if s.decay else 0.0
            p, gg = self.p[sl], g[sl] / clip
            if not h["adam_w_mode"]:
                gg = gg + d * p
            m = b1 * self.m[sl] + beta3 * gg
            v = b2 * self.v[sl] + self._one_minus(h, 1) * gg * gg
            u = (m / bc1) / ((v / bc2).sqrt() + eps)
            if h["adam_w_mode"]:
                u = u + d * p
            ratio = lr
            if h["use_nvlamb"] or d != 0.0:
                pn, un = float(p.norm()), float(u.norm())
                if pn > 0 and un > 0:
                    ratio = lr * pn / un
            self.p[sl], self.m[sl], self.v[sl] = p - ratio * u, m, v
        return gnorm

    def adam(self, g, h, step):
        lr, (b1, b2), eps, wd = _f32(h["lr"]), map(_f32, h["betas"]), _f32(h["eps"]), _f32(h["wd"])
        bc1 = self._bc(h, 0, step)
        bc2 = self._bc(h, 1, step)
        for s in self.slots:
            sl = slice(s.offset, s.offset + s.numel)
            d = wd if s.decay else 0.0
            p, gg = self.p[sl], g[sl]
            if not h["adam_w_mode"]:
                gg = gg + d * p
            m = b1 * self.m[sl] + self._one_minus(h, 0) * gg
            v = b2 * self.v[sl] + self._one_minus(h, 1) * gg * gg
            u = (m / bc1) / ((v / bc2).sqrt() + eps)
            if h["adam_w_mode"]:
                u = u + d * p
            self.p[sl], self.m[sl], self.v[sl] = p - lr * u, m, v


# Tolerances per slot: |x - ref| <= rtol |ref| + floor max|ref over the slot|.  The moments carry the relative error
# of the fp32 global norm (the clip divisor, reduced with atomics); p moves by lr x trust ratio x u per step, and its
# error is a few fp32 roundings of p plus the update's relative error.
TOL = {"p": (4e-6, 4e-6), "m": (2e-5, 2e-6), "v": (2e-5, 2e-6)}


def _check_state(arena_like, ref, what):
    for key, (rtol, floor) in TOL.items():
        got, want = arena_like[key], getattr(ref, key)
        for s in ref.slots:
            sl = slice(s.offset, s.offset + s.numel)
            a, b = got[sl].double(), want[sl]
            err = (a - b).abs()
            bound = rtol * b.abs() + floor * float(b.abs().max())
            assert bool((err <= bound).all()), (what, key, s.name, float(err.max()), float((err / bound).max()))


def _arena_state(arena):
    return {"p": arena.flat_param, "m": arena.exp_avg, "v": arena.exp_avg_sq}


def _torch_state(model, ref_slots_by_name, opt, numel):
    """The torch path's parameters and moments scattered into an arena-shaped flat tensor."""
    out = {k: torch.zeros(numel, dtype=torch.float32, device="cuda") for k in ("p", "m", "v")}
    for n, p in model.named_parameters():
        s = ref_slots_by_name[n]
        sl = slice(s.offset, s.offset + s.numel)
        out["p"][sl] = p.detach().reshape(-1)
        st = opt.state[p]
        out["m"][sl] = st["exp_avg"].reshape(-1)
        out["v"][sl] = st["exp_avg_sq"].reshape(-1)
    return out


def _set_sentinels(arena):
    pad = ~_slot_mask(arena)
    for buf in (arena.flat_param, arena.exp_avg, arena.exp_avg_sq):
        buf[pad] = SENTINEL
    arena.flat_shadow[pad] = SENTINEL
    return pad


def _make(kind, opt, flags):
    """(module under the arena, its fused optimizer, an arena-free copy, its torch-path optimizer, arena)."""
    from bert_pytorch_b200.models.arena import ParamArena
    from bert_pytorch_b200.optim import Adam, Lamb
    m_fused = _module(kind)
    m_torch = _module(kind)
    if opt == "lamb":
        kw = dict(lr=flags["lr"], betas=flags["betas"], eps=flags["eps"], bias_correction=flags["bias_correction"],
                  adam_w_mode=flags["adam_w_mode"], grad_averaging=flags["grad_averaging"],
                  max_grad_norm=flags["max_grad_norm"], use_nvlamb=flags["use_nvlamb"])
        cls = Lamb
    else:
        kw = dict(lr=flags["lr"], betas=flags["betas"], eps=flags["eps"], bias_correction=flags["bias_correction"],
                  adam_w_mode=flags["adam_w_mode"])
        cls = Adam
    arena = ParamArena(m_fused)
    o_fused = cls(m_fused.groups(flags["wd"]), **kw)
    arena.bind_optimizer(o_fused)
    assert arena.fused_optimizer_ok()
    o_torch = cls(m_torch.groups(flags["wd"]), **kw)
    return m_fused, o_fused, m_torch, o_torch, arena


def _load_grads(arena, model_torch, g):
    arena.flat_grad.copy_(g)
    for n, p in model_torch.named_parameters():
        s = arena.by_name[n]
        p.grad = g[s.offset:s.offset + s.numel].view(s.shape).clone()


# Dyadic betas are exact in fp32 and fp64 alike, so the fused path, the torch path and the reference use the same
# constants; the tiny-BERT rows keep the defaults (0.9, 0.999) of the runners.
DYADIC = (0.875, 1.0 - 2.0 ** -10)
# max_grad_norm: 0 = off, "above" = 1.0 with the global norm above it every step, "below" = 1.0 with it below
MGN = {"off": (0.0, 1.0), "above": (1.0, 1.0), "below": (1.0, 5e-4)}


def _lamb_case(mgn, aw, nv, ga, bc, kind="edges", betas=DYADIC):
    return ("lamb", kind, dict(lr=1e-2, betas=betas, eps=1e-6, wd=0.01, max_grad_norm=MGN[mgn][0], adam_w_mode=aw,
                               use_nvlamb=nv, grad_averaging=ga, bias_correction=bc), MGN[mgn][1], mgn)


def _adam_case(aw, bc, wd, kind="edges", betas=DYADIC, lr=1e-3):
    return ("adam", kind, dict(lr=lr, betas=betas, eps=1e-8, wd=wd, adam_w_mode=aw, bias_correction=bc), 1.0, None)


# A pairwise covering set over LAMB's flags: every pair of values of any two flags appears in some row (and so every
# single value of every flag).
LAMB_CASES = [
    _lamb_case("off", True, True, True, True),
    _lamb_case("off", False, False, False, False),
    _lamb_case("above", True, False, True, False),
    _lamb_case("above", False, True, False, True),
    _lamb_case("below", True, False, False, True),
    _lamb_case("below", False, True, True, False),
    _lamb_case("above", True, False, True, True, kind="tiny_bert", betas=(0.9, 0.999)),   # FusedLAMB's defaults
]
ADAM_CASES = [_adam_case(aw, bc, wd) for aw in (True, False) for bc in (True, False) for wd in (0.0, 0.01)] + [
    _adam_case(True, False, 0.01, kind="tiny_bert", betas=(0.9, 0.999)),        # the fine-tuning runners' setting
]


def _case_id(c):
    opt, kind, h, base, mgn = c
    if opt == "lamb":
        bits = (f"mgn_{mgn}-aw{int(h['adam_w_mode'])}-nv{int(h['use_nvlamb'])}-ga{int(h['grad_averaging'])}"
                f"-bc{int(h['bias_correction'])}")
    else:
        bits = f"aw{int(h['adam_w_mode'])}-bc{int(h['bias_correction'])}-wd{h['wd']}"
    return f"{opt}-{kind}-{bits}"


# the loss-scaler tests: LAMB clipping, Adam with weight decay and bias correction
_SCALER_CASE = {"lamb": _lamb_case("above", True, False, True, True)[2], "adam": _adam_case(True, True, 0.01)[2]}


def test_edges_module_hits_the_chunk_edges():
    from bert_pytorch_b200.models.arena import ParamArena
    arena = ParamArena(_module("edges"))
    numels = {s.numel for s in arena.slots}
    assert {1, 2, 3, 5, CHUNK, 2 * CHUNK + 5} <= numels
    assert any(s.offset % 4 != 0 for s in arena.slots)           # lamb_stage1's scalar (unaligned) branch runs
    assert any(s.offset % 4 == 2 for s in arena.slots)
    assert arena.numel > sum(s.numel for s in arena.slots)       # there is padding to guard


@pytest.mark.parametrize("case", LAMB_CASES + ADAM_CASES, ids=_case_id)
def test_arena_optimizer_matches_fp64(case):
    """Fused arena LAMB / Adam and the torch path, each against the fp64 reference, after every one of 5 steps;
    the shadow is bf16(p) bit for bit, the gradient arena is cleared, the padding is never written."""
    opt, kind, h, base, mgn = case
    m_fused, o_fused, m_torch, o_torch, arena = _make(kind, opt, h)
    pad = _set_sentinels(arena)
    ref, ref_t = _Ref(arena), _Ref(arena, torch_consts=True)
    for step in range(1, 6):
        g = _grads(arena, step, base)
        _load_grads(arena, m_torch, g)
        o_fused.step()
        o_torch.step()
        if opt == "lamb":
            gnorm = ref.lamb(g.double(), h, step)
            ref_t.lamb(g.double(), h, step)
            if mgn == "above":
                assert gnorm > h["max_grad_norm"]
            elif mgn == "below":
                assert gnorm < h["max_grad_norm"]
            assert abs(float(o_fused.last_grad_norm) - gnorm) <= 2e-5 * gnorm
            assert abs(float(o_torch.last_grad_norm) - gnorm) <= 2e-5 * gnorm
        else:
            ref.adam(g.double(), h, step)
            ref_t.adam(g.double(), h, step)
        _check_state(_arena_state(arena), ref, ("fused", step))
        _check_state(_torch_state(m_torch, arena.by_name, o_torch, arena.numel), ref_t, ("torch", step))
        assert torch.equal(arena.flat_shadow, arena.flat_param.to(torch.bfloat16))
        assert not bool(arena.flat_grad.any())
        assert all(gr["step"] == step for gr in o_fused.param_groups)
        assert all(gr["step"] == step for gr in o_torch.param_groups)
        for buf in (arena.flat_param, arena.exp_avg, arena.exp_avg_sq):
            assert bool((buf[pad] == SENTINEL).all())
        assert bool((arena.flat_shadow[pad].float() == SENTINEL).all())


@pytest.mark.parametrize("opt", ["lamb", "adam"])
def test_loss_scaled_step_is_bitwise_the_unscaled_step(opt):
    """Gradients x 2^16 with inv_scale = 2^-16 give bit for bit what the plain gradients give with no inv_scale: the
    scale is a power of two, so no rounding may differ.

    LAMB's global norm, and the norms of a tensor split over several chunks, finish with fp32 atomics whose order
    changes from run to run; so for LAMB this runs without clipping and on tensors of at most one chunk, where every
    value the update reads is reduced in a fixed order (the trust ratio still applies).  The scaled LAMB step with
    clipping and a multi-chunk tensor is checked against the fp64 reference in test_overflow_skips_the_step."""
    h = _SCALER_CASE[opt]
    kind = "edges"
    if opt == "lamb":
        h, kind = dict(h, max_grad_norm=0.0), "one_chunk"
    _, o_a, _, _, a = _make(kind, opt, h)
    _, o_b, _, _, b = _make(kind, opt, h)
    assert all(s.numel <= CHUNK for s in a.slots) or opt == "adam"
    inv = torch.full((), 2.0 ** -16, device="cuda")
    found = torch.zeros((), device="cuda")
    for step in range(1, 4):
        g = _grads(a, step, 1.0)
        a.flat_grad.copy_(g * 2.0 ** 16)
        b.flat_grad.copy_(g)
        o_a.step(inv_scale=inv, found_inf=found)
        o_b.step()
        assert float(found) == 0.0
        for x, y in ((a.flat_param, b.flat_param), (a.exp_avg, b.exp_avg), (a.exp_avg_sq, b.exp_avg_sq),
                     (a.flat_shadow, b.flat_shadow)):
            assert torch.equal(x, y), step
        if opt == "lamb":
            assert torch.allclose(o_a.last_grad_norm, o_b.last_grad_norm, rtol=2e-5, atol=0)
        assert o_a.param_groups[0]["step"] == o_b.param_groups[0]["step"] == step


def _poison(arena, g):
    """inf, nan and -inf in three different slots: a one-element slot, an unaligned q/k/v slot, and the last (tail)
    element of the tensor that spans three chunks."""
    g = g.clone()
    one, kv, span = arena.by_name["one"], arena.by_name["layer.0.attention.self.key.weight"], arena.by_name["span"]
    assert kv.offset % 4 != 0
    g[one.offset] = float("inf")
    g[kv.offset + 50] = float("nan")
    g[span.offset + span.numel - 1] = float("-inf")
    return g


@pytest.mark.parametrize("opt", ["lamb", "adam"])
def test_overflow_skips_the_step(opt):
    """A scaled step whose gradients hold inf / nan / -inf: found_inf is set, p, the moments and the shadow are
    untouched bit for bit, the gradients are cleared, the step counter stays; the next clean step matches a reference
    that never saw the bad one."""
    h = _SCALER_CASE[opt]
    _, o, _, _, arena = _make("edges", opt, h)
    ref = _Ref(arena)
    step_ref = getattr(ref, opt)
    inv = torch.full((), 2.0 ** -16, device="cuda")
    found = torch.zeros((), device="cuda")
    n_applied = 0
    for it in range(5):
        g = _grads(arena, it, 1.0)
        bad = it == 2
        arena.flat_grad.copy_((_poison(arena, g) if bad else g) * 2.0 ** 16)
        before = [t.clone() for t in (arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow)]
        o.step(inv_scale=inv, found_inf=found)
        assert not bool(arena.flat_grad.any())
        if bad:
            assert float(found) == 1.0
            for x, y in zip((arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow), before):
                assert torch.equal(x, y)
            assert all(gr["step"] == n_applied for gr in o.param_groups)
            found.zero_()                                  # what GradScaler.update does
            continue
        assert float(found) == 0.0
        n_applied += 1
        step_ref(g.double(), h, n_applied)
        assert all(gr["step"] == n_applied for gr in o.param_groups)
        _check_state(_arena_state(arena), ref, ("fused", it))
        assert torch.equal(arena.flat_shadow, arena.flat_param.to(torch.bfloat16))


@pytest.mark.parametrize("opt", ["lamb", "adam"])
def test_grad_scaler_backs_off_on_overflow(opt):
    from bert_pytorch_b200.optim import GradScaler
    h = _SCALER_CASE[opt]
    _, o, _, _, arena = _make("edges", opt, h)
    scaler = GradScaler(init_scale=2.0 ** 16, device="cuda")
    g = _grads(arena, 0, 1.0)
    arena.flat_grad.copy_(g * 2.0 ** 16)
    scaler.step(o)
    scaler.update()
    assert scaler.get_scale() == 2.0 ** 16 and o.param_groups[0]["step"] == 1
    before = [t.clone() for t in (arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow)]
    arena.flat_grad.copy_(_poison(arena, _grads(arena, 1, 1.0)) * 2.0 ** 16)
    scaler.step(o)
    scaler.update()
    assert scaler.get_scale() == 2.0 ** 15
    assert o.param_groups[0]["step"] == 1
    for x, y in zip((arena.flat_param, arena.exp_avg, arena.exp_avg_sq, arena.flat_shadow), before):
        assert torch.equal(x, y)
    assert not bool(arena.flat_grad.any())


@pytest.mark.parametrize("opt", ["lamb", "adam"])
def test_mixed_weight_decays_are_refused(opt):
    """The kernels apply one weight decay to every decaying slot: two different non-zero group values must raise,
    not silently apply the larger one to both groups."""
    h = _SCALER_CASE[opt]
    _, o, _, _, arena = _make("edges", opt, h)
    o.param_groups[1]["weight_decay"] = 0.001
    arena.flat_grad.copy_(_grads(arena, 0, 1.0))
    with pytest.raises(NotImplementedError, match="weight_decay"):
        o.step()


# ------------------------------------------------------------------------------------------------------------------
# flat_unscale_ (GradScaler.unscale_ over the arena)
# ------------------------------------------------------------------------------------------------------------------
N_UNSCALE = 3 * 2 ** 20 + 12     # more float4s than one pass of the grid-stride loop covers; a multiple of 4


@pytest.mark.parametrize("inv", [2.0 ** -16, 0.5, 8.0])
def test_flat_unscale_is_exact_for_power_of_two_scales(inv):
    K = _api()
    g = torch.randn(N_UNSCALE, device="cuda") * 100
    want = g * inv
    found = torch.zeros(1, device="cuda")
    K.flat_unscale_(g, torch.full((1,), inv, device="cuda"), found)
    assert torch.equal(g, want)
    assert float(found) == 0.0


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("bad", [float("inf"), float("nan"), float("-inf")])
def test_flat_unscale_flags_non_finite(where, bad):
    K = _api()
    g = torch.randn(N_UNSCALE, device="cuda")
    g[0 if where == "first" else -1] = bad
    found = torch.zeros(1, device="cuda")
    K.flat_unscale_(g, torch.full((1,), 2.0 ** -16, device="cuda"), found)
    assert float(found) == 1.0


def test_flat_unscale_does_not_flag_finite_values_whose_sum_overflows():
    K = _api()
    g = torch.zeros(N_UNSCALE, device="cuda")
    g[:2] = 3e38                   # one float4 (3e38, 3e38, 0, 0): finite, but its sum is not
    g[-4:] = torch.tensor([-3e38, -3e38, 3e38, -3e38])
    want = g.clone()
    found = torch.zeros(1, device="cuda")
    K.flat_unscale_(g, torch.ones(1, device="cuda"), found)
    assert float(found) == 0.0
    assert torch.equal(g, want)


@pytest.mark.parametrize("n", [N_UNSCALE + 1, N_UNSCALE + 2, N_UNSCALE + 3, 7])
def test_flat_unscale_rejects_a_numel_not_a_multiple_of_4(n):
    """The kernel works in float4s: a tail would be neither unscaled nor checked, so the binding refuses it."""
    K = _api()
    g = torch.ones(n, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 4"):
        K.flat_unscale_(g, torch.full((1,), 0.5, device="cuda"), torch.zeros(1, device="cuda"))


# ------------------------------------------------------------------------------------------------------------------
# softmax_ce_ (MLM head)
# ------------------------------------------------------------------------------------------------------------------
def _ce_rows(R, V, gen):
    """Logits and targets whose rows exercise the online max / sum: N(0, 3); the maximum in the last column (found on
    its thread's last iteration); all logits equal; magnitudes around +-60; targets at column 0 and V - 1; ignored
    rows (target -1)."""
    x = torch.randn(R, V, device="cuda", generator=gen) * 3
    tgt = torch.randint(0, V, (R,), device="cuda", generator=gen)
    kinds = 7
    for r in range(R):
        k = r % kinds
        if k == 1:
            x[r, -1] = x[r].max() + 4
        elif k == 2:
            x[r] = 1.5
        elif k == 3:
            sign = torch.randint(0, 2, (V,), device="cuda", generator=gen) * 2 - 1
            x[r] = sign * (60 + torch.rand(V, device="cuda", generator=gen))
        elif k == 4:
            tgt[r] = 0
        elif k == 5:
            tgt[r] = V - 1
        elif k == 6:
            tgt[r] = -1
    return x.to(torch.bfloat16), tgt.to(torch.int32)


def _ce_reference(x, tgt, grad_scale):
    """fp64 loss sum / count and d loss / d logits, from the bf16 logits."""
    x = x.double()
    valid = tgt >= 0
    cnt = int(valid.sum())
    lse = torch.logsumexp(x, dim=1)
    g = torch.softmax(x, dim=1)
    rows = torch.nonzero(valid).squeeze(1)
    g[rows, tgt[rows].long()] -= 1.0
    g *= grad_scale / max(cnt, 1)
    g[~valid] = 0.0
    loss = float((lse[rows] - x[rows, tgt[rows].long()]).sum()) / max(cnt, 1)
    return loss, g, cnt


def _check_ce(got, ref, grad_scale, cnt):
    # bf16 output rounding is at most 2^-9 relative and __expf's error ~1e-5: 2^-8 relative.  The floor is 2^-16 of
    # the row's gradient scale: at the target the kernel forms p - 1, so p's fp32 error becomes an absolute error there
    err = (got.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -16 * grad_scale / max(cnt, 1)
    assert bool((err <= bound).all()), (float(err.max()), float((err / bound).max()))


@pytest.mark.parametrize("grad_scale", [1.0, 65536.0])
@pytest.mark.parametrize("R", [1, 80, 640])
@pytest.mark.parametrize("V", [8, 2048, 30528])
def test_softmax_ce_matches_fp64(V, R, grad_scale):
    K = _api()
    gen = torch.Generator(device="cuda").manual_seed(V * 1000 + R)
    x, tgt = _ce_rows(R, V, gen)
    loss_ref, g_ref, cnt = _ce_reference(x, tgt, grad_scale)
    count = torch.tensor([cnt], dtype=torch.int32, device="cuda")
    pre = 3.25
    loss = torch.full((1,), pre, device="cuda")
    K.softmax_ce_(x, tgt, count, grad_scale, loss)
    _check_ce(x, g_ref, grad_scale, cnt)
    assert abs((float(loss) - pre) - loss_ref) <= 1e-4 * abs(loss_ref) + 2 ** -22 * pre


def test_softmax_ce_row_strided_view():
    """logits = big[:, :V] with a leading dimension past V: the kernel strides by it and never touches the columns
    past V."""
    K = _api()
    R, V, LD = 80, 2048, 2048 + 24
    gen = torch.Generator(device="cuda").manual_seed(5)
    x, tgt = _ce_rows(R, V, gen)
    big = (torch.randn(R, LD, device="cuda", generator=gen) * 7).to(torch.bfloat16)
    big[:, :V] = x
    right = big[:, V:].clone()
    view = big[:, :V]
    assert view.stride(0) == LD
    loss_ref, g_ref, cnt = _ce_reference(x, tgt, 2.0)
    loss = torch.zeros(1, device="cuda")
    K.softmax_ce_(view, tgt, torch.tensor([cnt], dtype=torch.int32, device="cuda"), 2.0, loss)
    _check_ce(view, g_ref, 2.0, cnt)
    assert torch.equal(big[:, V:], right)
    assert abs(float(loss) - loss_ref) <= 1e-4 * abs(loss_ref)


@pytest.mark.parametrize("V", [8, 30528])
def test_softmax_ce_count_zero(V):
    """No valid target (mlm_compact's count is 0): nothing is added to the loss, every gradient is zero."""
    K = _api()
    R = 80
    gen = torch.Generator(device="cuda").manual_seed(9)
    x = (torch.randn(R, V, device="cuda", generator=gen) * 3).to(torch.bfloat16)
    labels = torch.full((2, 40), -1, dtype=torch.int32, device="cuda")
    _, tgt, count = K.mlm_compact(labels, R // 2)
    assert int(count) == 0 and bool((tgt == -1).all())
    loss = torch.full((1,), 1.75, device="cuda")
    K.softmax_ce_(x, tgt, count, 65536.0, loss)
    assert float(loss) == 1.75
    assert not bool(x.any())


# ------------------------------------------------------------------------------------------------------------------
# nsp_head_ (NSP classifier + cross-entropy + backward)
# ------------------------------------------------------------------------------------------------------------------
def _nsp_reference(pooled, w, bias, labels, grad_scale):
    """fp64 from the bf16 pooled / w and fp32 bias.  dz uses tanh' = 1 - pooled^2 of the bf16 pooled value: the
    kernel's contract (pooled is the tanh output the pooler GEMM stored)."""
    x, wd, b = pooled.double(), w.double(), bias.double()
    logits = x @ wd.t() + b
    valid = labels >= 0
    n = int(valid.sum())
    p = torch.softmax(logits, dim=1)
    onehot = torch.zeros_like(p)
    onehot[valid, labels[valid]] = 1.0
    d = torch.where(valid[:, None], (p - onehot) * grad_scale / max(n, 1), torch.zeros_like(p))
    lse = torch.logsumexp(logits, dim=1)
    terms = torch.where(valid, lse - logits.gather(1, labels.clamp(min=0)[:, None]).squeeze(1), torch.zeros_like(lse))
    # the kernel's logits are fp32 dot products over H: bound their error by 2^-18 x sum |x w| (+ |bias|), which
    # covers the depth of its reduction (per-thread sums, warp tree, four warps) for H <= 1024
    dl = 2.0 ** -18 * ((x.abs() @ wd.abs().t()).max(dim=1).values + b.abs().max())
    mag = logits.abs().max(dim=1).values + 1.0       # scale of the fp32 max / log-sum-exp roundings
    return dict(loss=float(terms.sum()) / max(n, 1), terms=terms / max(n, 1), d=d, dz=(d @ wd) * (1 - x * x),
                dw=d.t() @ x, db=d.sum(0), dl=dl, mag=mag, n=n, x=x, w=wd)


@pytest.mark.parametrize("grad_scale", [1.0, 1024.0])
@pytest.mark.parametrize("H", [128, 200, 1024])
@pytest.mark.parametrize("B", [1, 7, 256])
def test_nsp_head_matches_fp64(B, H, grad_scale):
    K = _api()
    gen = torch.Generator(device="cuda").manual_seed(B * 10000 + H)
    pooled = torch.tanh(torch.randn(B, H, device="cuda", generator=gen) * 1.5).to(torch.bfloat16)
    w = (torch.randn(2, H, device="cuda", generator=gen) * 0.05).to(torch.bfloat16)
    bias = torch.randn(2, device="cuda", generator=gen) * 0.1
    labels = torch.randint(0, 2, (B,), device="cuda", generator=gen)
    if B > 1:
        labels[::3] = -1                      # a mix of 0, 1 and ignored
    pre_loss, pre_dw, pre_db = 0.5, torch.randn(2, H, device="cuda", generator=gen), torch.randn(2, device="cuda", generator=gen)
    loss, dw, db = torch.full((1,), pre_loss, device="cuda"), pre_dw.clone(), pre_db.clone()
    dz = K.nsp_head_(pooled, w, bias, labels, grad_scale, loss, dw, db)
    r = _nsp_reference(pooled, w, bias, labels, grad_scale)
    u = 2.0 ** -24
    # |d loss / d logit| error: p0 p1 x the logit-difference error (<= 2 dl) plus a few roundings of exp / log / division
    dd = (0.5 * r["dl"] + 8 * u * r["mag"]) * grad_scale / max(r["n"], 1)                         # per row
    dd = torch.where(labels >= 0, dd, torch.zeros_like(dd))
    # dz: bf16 rounding (2^-9) and d's relative error inside 2^-8; the floor covers the fp32 rounding of the two-term
    # sum d0 w0 + d1 w1, which cancels (d0 = -d1), and d's absolute error
    x, wd, d = r["x"], r["w"], r["d"]
    terms = d[:, :1].abs() * wd[0].abs() + d[:, 1:].abs() * wd[1].abs()
    err = (dz.double() - r["dz"]).abs()
    bound = 2.0 ** -8 * r["dz"].abs() + (3 * u * terms + dd[:, None] * (wd[0].abs() + wd[1].abs())) * (1 - x * x).abs()
    assert bool((err <= bound).all()), ("dz", float(err.max()), float((err / bound).max()))
    # dw / db / loss: fp32 atomics over the B rows, in any order (n u sum|terms|), plus d's own error
    atom = (B + 2) * u
    dw_err = (dw.double() - pre_dw.double() - r["dw"]).abs()
    dw_bound = dd[None, :] @ x.abs() + atom * (pre_dw.double().abs() + d.abs().t() @ x.abs())
    assert bool((dw_err <= dw_bound).all()), ("dw", float(dw_err.max()), float((dw_err / dw_bound).max()))
    db_err = (db.double() - pre_db.double() - r["db"]).abs()
    db_bound = dd.sum() + atom * (pre_db.double().abs() + d.abs().sum(0))
    assert bool((db_err <= db_bound).all()), ("db", db_err, db_bound)
    valid = (labels >= 0).double()
    loss_bound = (float(((2 * r["dl"] + 8 * u * r["mag"]) * valid).sum()) / max(r["n"], 1)
                  + atom * (pre_loss + float(r["terms"].abs().sum())))
    assert abs(float(loss) - pre_loss - r["loss"]) <= loss_bound


@pytest.mark.parametrize("B", [1, 7])
def test_nsp_head_all_ignored(B):
    """Every label -1: the loss is unchanged, dz is zero, dw and db are not written."""
    K = _api()
    H = 200
    gen = torch.Generator(device="cuda").manual_seed(3)
    pooled = torch.tanh(torch.randn(B, H, device="cuda", generator=gen)).to(torch.bfloat16)
    w = (torch.randn(2, H, device="cuda", generator=gen) * 0.05).to(torch.bfloat16)
    bias = torch.randn(2, device="cuda", generator=gen)
    labels = torch.full((B,), -1, dtype=torch.long, device="cuda")
    loss = torch.full((1,), 0.625, device="cuda")
    dw, db = torch.randn(2, H, device="cuda", generator=gen), torch.randn(2, device="cuda", generator=gen)
    dw0, db0 = dw.clone(), db.clone()
    dz = K.nsp_head_(pooled, w, bias, labels, 1024.0, loss, dw, db)
    assert float(loss) == 0.625
    assert not bool(dz.any())
    assert torch.equal(dw, dw0) and torch.equal(db, db0)
