"""K-FAC gradient preconditioner.

Call-compatible with how the reference drives gpauloski/kfac_pytorch (run_pretraining.py:321-355 and :405-409;
SURVEY.md N10, X6-X9): ``KFAC(model, lr=, factor_decay=, damping=, kl_clip=, factor_update_freq=,
inv_update_freq=, skip_layers=, comm_method=CommMethod.HYBRID_OPT, grad_worker_fraction=, inv_dtype=,
accumulate_data=, compute_factor_in_hook=, distribute_layer_factors=, grad_scaler=)``; ``.step()`` between
``scaler.unscale_`` and the optimizer step; ``.param_groups`` (so an LR scheduler can drive its ``lr``),
``.state_dict()`` / ``.load_state_dict()`` for checkpoints.  That package cannot be installed here, so the
maths below is our own statement of K-FAC (Martens & Grosse) for linear layers:

  per registered layer with input a [M, in] (+ ones column when the layer has a bias) and output gradient
  g [M, out] (gradient of the *mean* loss):
      A = a^T a / M                G = M * g^T g               (both fp32, symmetric)
  running averages  F <- decay * F + (1 - decay) * F_new  (first sample initialises F),
  eigendecompositions  A = Q_A diag(d_A) Q_A^T,  G = Q_G diag(d_G) Q_G^T  every ``inv_update_freq`` steps,
  preconditioned gradient  P = Q_G [ (Q_G^T W_g Q_A) / (d_G d_A^T + damping) ] Q_A^T  with W_g = [dW | db],
  KL clipping  nu = min(1, sqrt(kl_clip / (lr^2 * sum_layers <P, W_g>))),  grads <- nu * P.

Work distribution (``comm_method``): factors are averaged over all ranks every factor update; layer l's
eigendecomposition runs on rank ``l % world`` (both factors on the same rank, ``distribute_layer_factors=
False``); with COMM_OPT every rank receives the eigen-pairs and preconditions locally, with MEM_OPT only the
inverse worker preconditions and broadcasts the result, HYBRID_OPT uses ``grad_worker_fraction`` of the ranks
as gradient workers per layer.  Collectives go through the repo's ``Comm`` interface, i.e. the same
gloo / NCCL / peer-memory transport as the gradient reduction.

Where the activations come from: on the plain-PyTorch path forward-pre / backward hooks on the ``nn.Linear``
modules (``compute_factor_in_hook``); on the fused sm_90a path the engine hands the very tensors it already
saved for backward to :meth:`KFAC.tap`, and the factor SYRKs run on the wgmma GEMM (TN layout, fp32 out).
Registered: ``nn.Linear`` layers whose class/name path does not match ``skip_layers`` (Q, K, V, attention
output, FFN output, NSP) -- ``LinearActivation`` layers (FFN-in, pooler, MLM transform) are not, matching what
kfac_pytorch's module-type registry would do with this model.
"""
from __future__ import annotations

import enum
import math
from typing import Dict, Iterable, List, Optional

import torch
from torch import nn

from ..parallel.comm import Comm, SingleComm


class CommMethod(enum.Enum):
    COMM_OPT = 1
    MEM_OPT = 2
    HYBRID_OPT = 3


class _Layer:
    def __init__(self, name: str, module: nn.Linear, index: int):
        self.name, self.module, self.index = name, module, index
        self.has_bias = module.bias is not None
        self.A: Optional[torch.Tensor] = None
        self.G: Optional[torch.Tensor] = None
        self.QA = self.dA = self.QG = self.dG = None
        self._a: Optional[torch.Tensor] = None       # hook path: saved input
        self.A_new: Optional[torch.Tensor] = None    # accumulated since the last factor update
        self.G_new: Optional[torch.Tensor] = None
        self.n_new = 0

    def grad_matrix(self) -> torch.Tensor:
        g = self.module.weight.grad
        if self.has_bias:
            return torch.cat([g, self.module.bias.grad.unsqueeze(1)], dim=1)
        return g


def _factor(x: torch.Tensor) -> torch.Tensor:
    """x^T x in fp32 -- wgmma TN GEMM on CUDA bf16 inputs, torch elsewhere."""
    if x.is_cuda and x.dtype == torch.bfloat16 and x.size(1) % 8 == 0:
        from .. import ops
        if ops.available():
            from ..ops import api as K
            return K.gemm(x, x, layout=K.TN, epi=K.EPI_F32)
    xf = x.float()
    return xf.t() @ xf


class KFAC:
    def __init__(self, model: nn.Module, lr: float = 0.1, factor_decay: float = 0.95, damping: float = 0.001,
                 kl_clip: float = 0.001, factor_update_freq: int = 10, inv_update_freq: int = 100,
                 skip_layers: Optional[Iterable[str]] = None, comm_method: CommMethod = CommMethod.COMM_OPT,
                 grad_worker_fraction: float = 0.25, inv_dtype: torch.dtype = torch.float32,
                 accumulate_data: bool = True, compute_factor_in_hook: bool = False,
                 distribute_layer_factors: Optional[bool] = None, grad_scaler=None, comm: Optional[Comm] = None,
                 use_eigen_decomp: bool = True, verbose: bool = False):
        if not 0.0 < factor_decay <= 1.0:
            raise ValueError("factor_decay must be in (0, 1]")
        if damping <= 0 or kl_clip is not None and kl_clip <= 0:
            raise ValueError("damping and kl_clip must be positive")
        if factor_update_freq < 1 or inv_update_freq < 1:
            raise ValueError("update frequencies must be >= 1")
        self.model = model
        self.comm = comm if comm is not None else SingleComm()
        self.comm_method = comm_method
        self.grad_worker_fraction = grad_worker_fraction
        self.inv_dtype = inv_dtype
        self.grad_scaler = grad_scaler
        self.accumulate_data, self.compute_factor_in_hook = accumulate_data, compute_factor_in_hook
        self.param_groups = [dict(lr=lr, factor_decay=factor_decay, damping=damping, kl_clip=kl_clip,
                                  factor_update_freq=factor_update_freq, inv_update_freq=inv_update_freq)]
        self.skip_layers = [s.lower() for s in (skip_layers or [])]
        self.steps = 0
        self.capture = True          # fused engine: whether the next forward/backward feeds tap() (see wants_data)
        self.layers: List[_Layer] = []
        self._by_module: Dict[int, _Layer] = {}
        self._handles = []
        self._register(model)
        for m in model.modules():                # the fused engine looks for this attribute
            object.__setattr__(m, "_kfac", self)

    # -- registration -----------------------------------------------------------------------------------
    def _skipped(self, path_classes: List[str], name: str) -> bool:
        hay = [c.lower() for c in path_classes] + [name.lower()]
        return any(any(s in h for h in hay) for s in self.skip_layers)

    def _register(self, model: nn.Module) -> None:
        def walk(mod: nn.Module, prefix: str, classes: List[str]):
            for child_name, child in mod.named_children():
                full = f"{prefix}.{child_name}" if prefix else child_name
                cls = classes + [type(child).__name__]
                if isinstance(child, nn.Linear):
                    # the tied MLM decoder lives under BertLMPredictionHead and is skipped by default
                    if not self._skipped(cls, full):
                        layer = _Layer(full, child, len(self.layers))
                        self.layers.append(layer)
                        self._by_module[id(child)] = layer
                        self._handles.append(child.register_forward_pre_hook(self._save_input))
                        self._handles.append(child.register_full_backward_hook(self._save_grad_output))
                else:
                    walk(child, full, cls)
        walk(model, "", [type(model).__name__])

    def layer_names(self) -> List[str]:
        return [l.name for l in self.layers]

    # -- statistics capture ---------------------------------------------------------------------------------
    def _save_input(self, module, inputs):
        if not module.training or not torch.is_grad_enabled():
            return
        self._by_module[id(module)]._a = inputs[0].detach()

    def _save_grad_output(self, module, grad_input, grad_output):
        layer = self._by_module[id(module)]
        if layer._a is None:
            return
        self.tap(layer, layer._a.reshape(-1, layer._a.size(-1)), grad_output[0].detach().reshape(-1, grad_output[0].size(-1)))
        layer._a = None

    def layer(self, module_or_name) -> Optional[_Layer]:
        if isinstance(module_or_name, str):
            for l in self.layers:
                if l.name == module_or_name or l.name.endswith("." + module_or_name):
                    return l
            return None
        return self._by_module.get(id(module_or_name))

    @torch.no_grad()
    def tap(self, layer, a: torch.Tensor, g: torch.Tensor) -> None:
        """Account one micro-batch: ``a`` [M, in] layer input, ``g`` [M, out] gradient of the (scaled) mean
        loss w.r.t. the layer output."""
        if not isinstance(layer, _Layer):
            layer = self.layer(layer)
            if layer is None:
                return
        M = a.size(0)
        scale = self.grad_scaler.get_scale() if (self.grad_scaler is not None and self.grad_scaler.is_enabled()) else 1.0
        A = _factor(a) / M
        if layer.has_bias:
            col = a.float().sum(0, keepdim=True) / M
            A = torch.cat([torch.cat([A, col.t()], dim=1),
                           torch.cat([col, torch.ones(1, 1, device=A.device)], dim=1)], dim=0)
        G = _factor(g) * (M / (scale * scale))
        if layer.A_new is None or not self.accumulate_data:
            # accumulate_data=False (how the reference configures kfac_pytorch, run_pretraining.py:335): the factors of a
            # step come from ONE micro-batch -- the latest tap replaces the previous one
            layer.A_new, layer.G_new, layer.n_new = A, G, 1
        else:
            layer.A_new += A
            layer.G_new += G
            layer.n_new += 1

    def wants_data(self, last_micro_step: bool) -> bool:
        """Whether the next forward/backward has to feed :meth:`tap`.  With ``accumulate_data=False`` only the last
        micro-batch of an optimizer step whose factors are due counts, so every other micro-step runs without taps --
        and therefore inside the captured CUDA graph (the taps are ~2x the FLOPs of the step itself for BERT-large:
        two 4096^2 and eight 1024^2 factor GEMMs per layer)."""
        due = self.steps % self.param_groups[0]["factor_update_freq"] == 0
        if not due:
            return False
        return True if self.accumulate_data else bool(last_micro_step)

    # -- the step ----------------------------------------------------------------------------------------------
    def _workers(self, layer: _Layer):
        world = self.comm.world_size
        inv = layer.index % world
        if self.comm_method == CommMethod.COMM_OPT:
            grad = list(range(world))
        elif self.comm_method == CommMethod.MEM_OPT:
            grad = [inv]
        else:
            n = max(1, min(world, int(round(world * self.grad_worker_fraction))))
            start = (inv // n) * n
            grad = list(range(start, min(start + n, world)))
        return inv, grad

    @torch.no_grad()
    def step(self) -> None:
        g0 = self.param_groups[0]
        decay, damping, lr, kl_clip = g0["factor_decay"], g0["damping"], g0["lr"], g0["kl_clip"]
        comm, rank = self.comm, self.comm.rank
        # ---- factor update: average over micro-batches and ranks, fold into the running average
        if self.steps % g0["factor_update_freq"] == 0:
            fresh = []
            for l in self.layers:
                if l.A_new is None:
                    continue
                l.A_new = l.A_new / max(l.n_new, 1)
                l.G_new = l.G_new / max(l.n_new, 1)
                fresh += [l.A_new, l.G_new]
            # all factors of the step travel together: one packed transfer per staging buffer on the peer-memory
            # backend (ops/csrc/comm.cu: peer_allreduce_kernel), a loop of all-reduces elsewhere (SURVEY.md X5)
            comm.all_reduce_many_(fresh, op="avg")
            for l in self.layers:
                if l.A_new is None:
                    continue
                for key in ("A", "G"):
                    new, cur = getattr(l, key + "_new"), getattr(l, key)
                    setattr(l, key, new.clone() if cur is None else cur.mul_(decay).add_(new, alpha=1.0 - decay))
                l.A_new = l.G_new = None
                l.n_new = 0
        # ---- eigendecompositions on the layer's inverse worker, shipped to its gradient workers
        if self.steps % g0["inv_update_freq"] == 0:
            for l in self.layers:
                if l.A is None:
                    continue
                inv, grad_workers = self._workers(l)
                if rank == inv:
                    dA, QA = torch.linalg.eigh(l.A.float())
                    dG, QG = torch.linalg.eigh(l.G.float())
                    # eigh returns column-major eigenvector matrices: collectives need dense row-major payloads
                    l.QA, l.dA = QA.to(self.inv_dtype).contiguous(), dA.clamp_(min=0.0).to(self.inv_dtype).contiguous()
                    l.QG, l.dG = QG.to(self.inv_dtype).contiguous(), dG.clamp_(min=0.0).to(self.inv_dtype).contiguous()
                elif rank in grad_workers and l.QA is None:
                    n_a, n_g = l.A.size(0), l.G.size(0)
                    dev = l.A.device
                    l.QA = torch.empty(n_a, n_a, dtype=self.inv_dtype, device=dev)
                    l.dA = torch.empty(n_a, dtype=self.inv_dtype, device=dev)
                    l.QG = torch.empty(n_g, n_g, dtype=self.inv_dtype, device=dev)
                    l.dG = torch.empty(n_g, dtype=self.inv_dtype, device=dev)
                if comm.world_size > 1 and len(grad_workers) > 1:
                    # eigen-pairs travel inside the layer's gradient-worker GROUP only (HYBRID_OPT: half the ranks),
                    # in inv_dtype (fp16 in the shipped recipe); ranks outside the group neither allocate nor receive
                    for key in ("QA", "dA", "QG", "dG"):
                        shape = {"QA": (l.A.size(0),) * 2, "dA": (l.A.size(0),), "QG": (l.G.size(0),) * 2,
                                 "dG": (l.G.size(0),)}[key]
                        got = comm.broadcast_group_(getattr(l, key), inv, grad_workers, shape=shape, dtype=self.inv_dtype,
                                                    device=l.A.device)
                        if rank in grad_workers:
                            setattr(l, key, got)
        # ---- precondition
        vg_sum = torch.zeros((), dtype=torch.float32, device=self.layers[0].module.weight.device) if self.layers else None
        updates: Dict[int, torch.Tensor] = {}
        for l in self.layers:
            if l.A is None or l.module.weight.grad is None:
                continue
            inv, grad_workers = self._workers(l)
            Wg = l.grad_matrix().float()
            if rank in grad_workers and l.QA is not None:
                QA, QG = l.QA.float(), l.QG.float()
                v1 = QG.t() @ Wg @ QA
                v2 = v1 / (l.dG.float().unsqueeze(1) * l.dA.float().unsqueeze(0) + damping)
                P = QG @ v2 @ QA.t()
            else:
                P = torch.zeros_like(Wg)
            if comm.world_size > 1 and len(grad_workers) < comm.world_size:
                # preconditioned gradient: from the inverse worker to the ranks OUTSIDE the gradient-worker group only
                receivers = [inv] + [r for r in range(comm.world_size) if r not in grad_workers]
                P = P.contiguous()
                got = comm.broadcast_group_(P if rank in receivers else None, inv, receivers, shape=tuple(P.shape),
                                            dtype=P.dtype, device=P.device)
                if rank in receivers:
                    P = got
            updates[l.index] = P
            vg_sum += (P * Wg).sum() * (lr ** 2)
        if not updates:
            self.steps += 1
            return
        nu = 1.0
        if kl_clip is not None:
            # KL clip on the device: nu = min(1, sqrt(kl_clip / vg)) (1 where vg <= 0) -- no host read-back in the step
            safe = vg_sum.clamp_min(1e-30)
            nu = torch.where(vg_sum > 0, torch.sqrt(kl_clip / safe).clamp_(max=1.0), torch.ones_like(vg_sum))
        for l in self.layers:
            if l.index not in updates:
                continue
            P = updates[l.index] * nu
            if l.has_bias:
                l.module.weight.grad.copy_(P[:, :-1].to(l.module.weight.grad.dtype))
                l.module.bias.grad.copy_(P[:, -1].to(l.module.bias.grad.dtype))
            else:
                l.module.weight.grad.copy_(P.to(l.module.weight.grad.dtype))
        self.steps += 1

    # -- (de)serialisation ------------------------------------------------------------------------------------
    def state_dict(self) -> dict:
        return {"steps": self.steps, "param_groups": [dict(g) for g in self.param_groups],
                "layers": {l.name: {"A": l.A, "G": l.G} for l in self.layers if l.A is not None}}

    def load_state_dict(self, state: dict) -> None:
        self.steps = int(state.get("steps", 0))
        for g, s in zip(self.param_groups, state.get("param_groups", [])):
            g.update({k: v for k, v in s.items() if k != "lr"})
        for l in self.layers:
            f = state.get("layers", {}).get(l.name)
            if f is not None:
                dev = l.module.weight.device
                l.A, l.G = f["A"].to(dev), f["G"].to(dev)
                l.QA = l.dA = l.QG = l.dG = None      # recomputed at the next inverse update

    def __repr__(self) -> str:
        g = self.param_groups[0]
        return (f"KFAC(layers={len(self.layers)}, comm_method={self.comm_method.name}, "
                f"grad_worker_fraction={self.grad_worker_fraction}, inv_dtype={self.inv_dtype}, " +
                ", ".join(f"{k}={v}" for k, v in g.items()) + ")\n  " + "\n  ".join(self.layer_names()))
