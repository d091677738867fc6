"""BERT model zoo.

The modules below carry the parameters under exactly the state-dict names of the
reference (SURVEY.md 2.5.3; src/modeling.py:338-617, 802-1327) so checkpoints
move freely between the two code bases.  Each module has a plain-PyTorch
``forward`` that is the numerics oracle and the CPU / gloo execution path.  On an
H100 the encoder + pre-training heads do not run these forwards: ``BertModel``
hands the whole encoder to :mod:`bert_pytorch_b200.models.fused`, which executes
hand written sm_90a kernels straight out of the flat parameter arena.

Numerics contract (SURVEY.md appendix B): LayerNorm eps 1e-12 inside the sqrt with
fp32 statistics, erf-GELU, attention scale applied after QK^T, additive -10000
key-padding mask, dropout on attention probabilities / sub-layer outputs /
embeddings, post-LN residual blocks.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from ..config import BertConfig

# ---------------------------------------------------------------------------
# activations (src/modeling.py:118-139)
# ---------------------------------------------------------------------------


def gelu(x: torch.Tensor) -> torch.Tensor:
    return F.gelu(x)  # exact erf form


def swish(x: torch.Tensor) -> torch.Tensor:
    return x * torch.sigmoid(x)


def bias_gelu(bias: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return F.gelu(y + bias)


def bias_tanh(bias: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return torch.tanh(y + bias)


def bias_relu(bias: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return F.relu(y + bias)


def bias_swish(bias: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return swish(y + bias)


#: name -> callable.  ``bias_*`` entries take (bias, y).  Runners may overwrite
#: ``ACT2FN["bias_gelu"]`` like the reference does (run_pretraining.py:240); here the
#: training and inference versions are the same function.
ACT2FN = {
    "gelu": gelu, "relu": F.relu, "swish": swish, "tanh": torch.tanh,
    "bias_gelu": bias_gelu, "bias_tanh": bias_tanh, "bias_relu": bias_relu,
    "bias_swish": bias_swish,
}
bias_gelu_training = bias_gelu


class LinearActivation(nn.Module):
    """``act(x W^T + b)`` kept as one module so the fused engine can run it as one
    GEMM with a bias+activation epilogue (K16/K19/K21).  Parameters: ``weight``
    [out,in], ``bias`` [out].  Initialisation follows the reference quirk Q14: these
    weights keep the kaiming-uniform init (src/modeling.py:169-174) because
    ``init_bert_weights`` only touches nn.Linear / nn.Embedding / LayerNorm."""

    def __init__(self, in_features: int, out_features: int, act: str = "gelu", bias: bool = True):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.act_name = act
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1.0 / math.sqrt(self.in_features)
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.bias is not None:
            return ACT2FN["bias_" + self.act_name](self.bias, F.linear(x, self.weight, None))
        return ACT2FN[self.act_name](F.linear(x, self.weight, None))

    def extra_repr(self) -> str:
        return f"in={self.in_features}, out={self.out_features}, act={self.act_name}"


class BertLayerNorm(nn.Module):
    """LayerNorm over the last dim, eps inside the sqrt, statistics in fp32
    (src/modeling.py:282-336)."""

    def __init__(self, hidden_size: int, eps: float = 1e-12):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.bias = nn.Parameter(torch.zeros(hidden_size))
        self.eps = eps

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xf = x.float()
        mu = xf.mean(-1, keepdim=True)
        var = (xf - mu).pow(2).mean(-1, keepdim=True)
        y = (xf - mu) * torch.rsqrt(var + self.eps)
        return (y * self.weight.float() + self.bias.float()).to(x.dtype)


class BertNonFusedLayerNorm(BertLayerNorm):
    """Name kept for users of the reference's eager LayerNorm (src/modeling.py:282-297).  There is a single
    LayerNorm module here: the kernels live in the fused engine, this module is the parameter holder and the
    eager oracle, so the "non fused" variant is the same class (``variance_epsilon`` is the reference's name
    for ``eps``)."""

    @property
    def variance_epsilon(self) -> float:
        return self.eps


# ---------------------------------------------------------------------------
# encoder
# ---------------------------------------------------------------------------


class BertEmbeddings(nn.Module):
    """word + position (+ token type iff ``config.next_sentence``) -> LN -> dropout
    (src/modeling.py:338-373)."""

    def __init__(self, config: BertConfig):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.has_token_type = bool(getattr(config, "next_sentence", True))
        if self.has_token_type:
            self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, input_ids: torch.Tensor, token_type_ids: Optional[torch.Tensor]) -> torch.Tensor:
        S = input_ids.size(1)
        pos = torch.arange(S, device=input_ids.device).unsqueeze(0).expand_as(input_ids)
        e = self.word_embeddings(input_ids) + self.position_embeddings(pos)
        if self.has_token_type:
            if token_type_ids is None:
                token_type_ids = torch.zeros_like(input_ids)
            e = e + self.token_type_embeddings(token_type_ids)
        return self.dropout(self.LayerNorm(e))


class BertSelfAttention(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.h = config.num_attention_heads
        self.d = config.hidden_size // self.h
        self.query = nn.Linear(config.hidden_size, config.hidden_size)
        self.key = nn.Linear(config.hidden_size, config.hidden_size)
        self.value = nn.Linear(config.hidden_size, config.hidden_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)

    def forward(self, x: torch.Tensor, additive_mask: torch.Tensor) -> torch.Tensor:
        B, S, H = x.shape
        def heads(t):
            return t.view(B, S, self.h, self.d).transpose(1, 2)  # [B,h,S,d]
        q, k, v = heads(self.query(x)), heads(self.key(x)), heads(self.value(x))
        scores = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(self.d)
        scores = scores + additive_mask
        probs = F.softmax(scores.float(), dim=-1).to(x.dtype)
        probs = self.dropout(probs)
        ctx = torch.matmul(probs, v)
        return ctx.transpose(1, 2).reshape(B, S, H)


class BertSelfOutput(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, h: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        return self.LayerNorm(self.dropout(self.dense(h)) + residual)


class BertAttention(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def forward(self, x: torch.Tensor, additive_mask: torch.Tensor) -> torch.Tensor:
        return self.output(self.self(x, additive_mask), x)


class BertIntermediate(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.intermediate_size,
                                          act=config.hidden_act)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.dense_act(x)


class BertOutput(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = BertLayerNorm(config.hidden_size)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, h: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        return self.LayerNorm(self.dropout(self.dense(h)) + residual)


class BertLayer(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)

    def forward(self, x: torch.Tensor, additive_mask: torch.Tensor) -> torch.Tensor:
        a = self.attention(x, additive_mask)
        return self.output(self.intermediate(a), a)


class BertEncoder(nn.Module):
    """L post-LN layers.  With activation checkpointing the layers are grouped in
    ceil(sqrt(L)) sized segments (src/modeling.py:503-520)."""

    def __init__(self, config: BertConfig):
        super().__init__()
        self.layer = nn.ModuleList(BertLayer(config) for _ in range(config.num_hidden_layers))
        self.output_all_encoded_layers = bool(getattr(config, "output_all_encoded_layers", False))
        self._checkpoint_activations = False

    def _segment(self, lo: int, hi: int):
        def run(x, mask):
            for layer in self.layer[lo:hi]:
                x = layer(x, mask)
            return x
        return run

    def forward(self, x: torch.Tensor, additive_mask: torch.Tensor) -> List[torch.Tensor]:
        outs: List[torch.Tensor] = []
        if self._checkpoint_activations and self.training:
            from torch.utils.checkpoint import checkpoint
            L = len(self.layer)
            seg = int(math.ceil(math.sqrt(L)))
            lo = 0
            while lo < L:
                hi = min(L, lo + seg)
                x = checkpoint(self._segment(lo, hi), x, additive_mask * 1, use_reentrant=False)
                lo = hi
            outs.append(x)
            return outs
        for layer in self.layer:
            x = layer(x, additive_mask)
            if self.output_all_encoded_layers:
                outs.append(x)
        if not self.output_all_encoded_layers:
            outs.append(x)
        return outs


class BertPooler(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act="tanh")

    def forward(self, hidden: torch.Tensor) -> torch.Tensor:
        return self.dense_act(hidden[:, 0])


# ---------------------------------------------------------------------------
# heads
# ---------------------------------------------------------------------------


class BertPredictionHeadTransform(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act=config.hidden_act)
        self.LayerNorm = BertLayerNorm(config.hidden_size)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.LayerNorm(self.dense_act(x))


class BertLMPredictionHead(nn.Module):
    """transform -> decoder tied to the word embedding matrix + free bias
    (src/modeling.py:564-579)."""

    def __init__(self, config: BertConfig, embedding_weight: torch.nn.Parameter):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(embedding_weight.size(1), embedding_weight.size(0), bias=False)
        self.decoder.weight = embedding_weight  # tied
        self.bias = nn.Parameter(torch.zeros(embedding_weight.size(0)))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.decoder(self.transform(x)) + self.bias


class BertOnlyMLMHead(nn.Module):
    def __init__(self, config: BertConfig, embedding_weight):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, embedding_weight)

    def forward(self, seq: torch.Tensor) -> torch.Tensor:
        return self.predictions(seq)


class BertOnlyNSPHead(nn.Module):
    def __init__(self, config: BertConfig):
        super().__init__()
        self.seq_relationship = nn.Linear(config.hidden_size, 2)

    def forward(self, pooled: torch.Tensor) -> torch.Tensor:
        return self.seq_relationship(pooled)


class BertPreTrainingHeads(nn.Module):
    def __init__(self, config: BertConfig, embedding_weight):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, embedding_weight)
        self.has_nsp = bool(getattr(config, "next_sentence", True))
        if self.has_nsp:
            self.seq_relationship = nn.Linear(config.hidden_size, 2)

    def forward(self, seq: torch.Tensor, pooled: Optional[torch.Tensor]):
        scores = self.predictions(seq)
        nsp = self.seq_relationship(pooled) if (self.has_nsp and pooled is not None) else None
        return scores, nsp


# ---------------------------------------------------------------------------
# base class: init, flags, (de)serialisation
# ---------------------------------------------------------------------------

CONFIG_NAME = "bert_config.json"
WEIGHTS_NAME = "pytorch_model.bin"
TF_WEIGHTS_NAME = "model.ckpt"

PRETRAINED_MODEL_ARCHIVE_MAP = {
    name: f"https://s3.amazonaws.com/models.huggingface.co/bert/{name}.tar.gz"
    for name in ("bert-base-uncased", "bert-large-uncased", "bert-base-cased", "bert-large-cased",
                 "bert-base-multilingual-uncased", "bert-base-multilingual-cased", "bert-base-chinese")
}


class BertPreTrainedModel(nn.Module):
    """Weight init + checkpoint helpers shared by every model
    (src/modeling.py:620-799)."""

    def __init__(self, config: BertConfig):
        super().__init__()
        if not isinstance(config, BertConfig):
            raise ValueError("config must be a BertConfig (build one with BertConfig.from_json_file)")
        self.config = config

    def init_bert_weights(self, module: nn.Module) -> None:
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, BertLayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    def checkpoint_activations(self, val: bool) -> None:
        for m in self.modules():
            if isinstance(m, BertEncoder):
                m._checkpoint_activations = bool(val)

    def enable_apex(self, val: bool) -> None:
        """Kept for CLI compatibility (src/modeling.py:653-657); selects the fused
        sm_90a LayerNorm/engine path instead of apex."""
        for m in self.modules():
            if isinstance(m, BertModel):
                m.use_fused = bool(val)

    # -- loading ------------------------------------------------------------
    @staticmethod
    def _normalise_keys(state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        out = {}
        for k, v in state.items():
            nk = k
            if nk.endswith("gamma"):
                nk = nk[:-5] + "weight"
            elif nk.endswith("beta"):
                nk = nk[:-4] + "bias"
            if nk.startswith("module."):
                nk = nk[len("module."):]
            out[nk] = v
        return out

    def load_compatible_state_dict(self, state: Dict[str, torch.Tensor], strict: bool = False):
        """Load a state dict that may use TF-era names (gamma/beta), a DDP
        ``module.`` prefix, or lack/have the ``bert.`` prefix."""
        state = self._normalise_keys(state)
        own = set(self.state_dict().keys())
        has_prefix = any(k.startswith("bert.") for k in state)
        wants_prefix = any(k.startswith("bert.") for k in own)
        if wants_prefix and not has_prefix:
            state = {("bert." + k if ("bert." + k) in own else k): v for k, v in state.items()}
        elif has_prefix and not wants_prefix:
            state = {(k[5:] if k.startswith("bert.") else k): v for k, v in state.items()}
        return self.load_state_dict(state, strict=strict)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, state_dict=None, cache_dir=None,
                        from_tf: bool = False, *inputs, **kwargs):
        """Instantiate from a directory / archive / known model name holding
        ``bert_config.json`` + ``pytorch_model.bin`` (or a TF checkpoint)."""
        import tarfile
        import tempfile
        from ..utils.file_utils import cached_path

        src = PRETRAINED_MODEL_ARCHIVE_MAP.get(pretrained_model_name_or_path, pretrained_model_name_or_path)
        resolved = cached_path(src, cache_dir=cache_dir)
        tmp = None
        if os.path.isdir(resolved) or from_tf:
            serialization_dir = resolved
        else:
            tmp = tempfile.mkdtemp()
            with tarfile.open(resolved, "r:*") as tar:
                base = os.path.realpath(tmp)
                for m in tar.getmembers():  # refuse path traversal
                    tgt = os.path.realpath(os.path.join(tmp, m.name))
                    if not tgt.startswith(base + os.sep) and tgt != base:
                        raise RuntimeError(f"unsafe path in archive: {m.name}")
                tar.extractall(tmp)
            serialization_dir = tmp
        config = BertConfig.from_json_file(os.path.join(serialization_dir, CONFIG_NAME))
        model = cls(config, *inputs, **kwargs)
        if from_tf:
            load_tf_weights_in_bert(model, os.path.join(serialization_dir, TF_WEIGHTS_NAME))
        else:
            if state_dict is None:
                state_dict = torch.load(os.path.join(serialization_dir, WEIGHTS_NAME), map_location="cpu")
                if "model" in state_dict and isinstance(state_dict["model"], dict):
                    state_dict = state_dict["model"]
            model.load_compatible_state_dict(state_dict, strict=False)
        if tmp is not None:
            import shutil
            shutil.rmtree(tmp, ignore_errors=True)
        return model


def load_tf_weights_in_bert(model: nn.Module, tf_checkpoint_path: str) -> nn.Module:
    """Import a Google TF checkpoint (src/modeling.py:58-116).  Needs tensorflow; the
    variable walk maps ``kernel``->transposed ``weight``, ``gamma/beta``->LN
    weight/bias, ``output_bias``->bias and skips optimiser slots."""
    try:
        import numpy as np
        import tensorflow as tf  # type: ignore
    except ImportError as e:  # pragma: no cover - tensorflow is optional
        raise ImportError("loading a TF checkpoint requires tensorflow") from e
    for name, _shape in tf.train.list_variables(tf_checkpoint_path):  # pragma: no cover
        if any(s in name for s in ("adam_v", "adam_m", "global_step", "AdamWeightDecayOptimizer")):
            continue
        arr = tf.train.load_variable(tf_checkpoint_path, name)
        ptr = model
        for part in name.split("/"):
            key, idx = (part.rsplit("_", 1) + [None])[:2] if part.rsplit("_", 1)[-1].isdigit() else (part, None)
            if key in ("kernel", "gamma"):
                ptr = getattr(ptr, "weight")
            elif key in ("output_bias", "beta"):
                ptr = getattr(ptr, "bias")
            elif key == "output_weights":
                ptr = getattr(ptr, "weight")
            else:
                ptr = getattr(ptr, key)
            if idx is not None:
                ptr = ptr[int(idx)]
        if name.endswith("_embeddings"):
            ptr = getattr(ptr, "weight")
        elif name.endswith("kernel"):
            arr = np.transpose(arr)
        ptr.data.copy_(torch.from_numpy(arr))
    return model


# ---------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------


class BertModel(BertPreTrainedModel):
    """Embeddings + encoder (+ pooler iff ``next_sentence``) -- src/modeling.py:802-883.

    ``use_fused`` (default True): run the encoder through the sm_90a engine whenever it can.
    ``unpad`` (default False): when the fused engine runs, compute only the tokens whose ``attention_mask`` is 1,
    packed back to back, with variable-length attention over each sequence's tokens (any 0/1 mask, holes included).
    The sequence output is then zero at positions where ``attention_mask == 0``; the padded engine computes those
    positions as attention over the valid keys.  This is exact for every head that never reads masked positions --
    token classification with its masked loss, sequence classification, multiple choice and QA prediction -- but not
    for QA training, whose start / end cross-entropy normalises over all positions, masked ones included.
    fp8 operands have no unpadded path: they run padded (with a warning)."""

    def __init__(self, config: BertConfig):
        super().__init__(config)
        self.embeddings = BertEmbeddings(config)
        self.encoder = BertEncoder(config)
        self.pooler = BertPooler(config) if getattr(config, "next_sentence", True) else None
        self.output_all_encoded_layers = bool(getattr(config, "output_all_encoded_layers", False))
        self.use_fused = True   # the sm_90a engine is used whenever it can be
        self.unpad = False      # fused engine on the unmasked tokens only (see the class docstring)
        self._engine = None
        self.apply(self.init_bert_weights)

    # additive key-padding mask in the activation dtype (src/modeling.py:862-870)
    @staticmethod
    def additive_mask(attention_mask: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
        m = attention_mask[:, None, None, :].to(dtype)
        return (1.0 - m) * -10000.0

    def fused_engine(self):
        """The sm_90a execution engine bound to this module's parameters (built
        lazily the first time a CUDA forward is requested)."""
        if self._engine is None:
            from .fused import FusedEncoderEngine
            self._engine = FusedEncoderEngine(self)
        return self._engine

    def fusable_config(self) -> bool:
        """Whether the sm_90a kernel program implements this configuration.  The reference model runs any
        ``hidden_act`` of ``ACT2FN`` and any head size (src/modeling.py:118-139); the fused engine is specialised for
        erf-GELU and head_dim 64 with H a multiple of 64 and S <= 512 -- everything else takes the plain PyTorch path
        instead of raising (VERDICT r1, missing #4)."""
        cfg = self.config
        if cfg.hidden_act not in ("gelu", "bias_gelu"):
            return False
        H, h = cfg.hidden_size, cfg.num_attention_heads
        if H % 64 != 0 or H // h != 64:
            return False
        if cfg.intermediate_size % 8 != 0 or H > 8 * 256:
            return False
        return True

    def _can_fuse(self, input_ids: torch.Tensor) -> bool:
        if not (self.use_fused and input_ids.is_cuda):
            return False
        if not self.fusable_config() or input_ids.size(-1) > 512 or input_ids.size(-1) % 8 != 0:
            return False
        from .. import ops
        return ops.available()

    def forward(self, input_ids, token_type_ids=None, attention_mask=None):
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if self._can_fuse(input_ids) and not self.output_all_encoded_layers:
            seq = self.fused_engine().encode(input_ids, token_type_ids, attention_mask)
            layers = [seq]
        else:
            dtype = self.embeddings.word_embeddings.weight.dtype
            if torch.is_autocast_enabled():
                dtype = torch.get_autocast_dtype(input_ids.device.type)
            x = self.embeddings(input_ids, token_type_ids)
            layers = self.encoder(x, self.additive_mask(attention_mask, dtype))
        pooled = self.pooler(layers[-1]) if self.pooler is not None else None
        if not self.output_all_encoded_layers:
            layers = layers[-1:]            # a LIST, as in the reference (src/modeling.py:880-883): callers index [-1]
        return layers, pooled


def _metric_sums(scores: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """fp64 [3] {cross-entropy sum, correct count, count} of the rows of ``scores`` whose label is not -1
    (``torch.argmax``: the lowest index wins a tie)."""
    labels = labels.long().to(scores.device)
    keep = labels >= 0
    s, t = scores[keep].float(), labels[keep]
    loss = F.cross_entropy(s, t, reduction="none").double().sum()
    correct = (s.argmax(dim=-1) == t).sum().double()
    return torch.stack([loss, correct, torch.tensor(float(t.numel()), dtype=torch.float64, device=s.device)])


class BertForPreTraining(BertPreTrainedModel):
    """MLM + (optional) NSP heads; returns raw scores, the loss lives in the
    criterion (src/modeling.py:886-947)."""

    def __init__(self, config: BertConfig):
        super().__init__(config)
        self.bert = BertModel(config)
        self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight)
        self._pretrainer = None
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None):
        layers, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        seq = layers[-1]
        return self.cls(seq, pooled)

    def pretrain_engine(self):
        """The fused sm_90a forward+backward engine for MLM(+NSP) training, or ``None`` when the
        model is not on a CUDA device / fusion is disabled (then the autograd path runs)."""
        if not self.bert.use_fused or not self.bert.fusable_config():
            return None                   # e.g. relu / swish FFN or head_dim != 64: the autograd oracle path trains it
        if not self.bert.embeddings.word_embeddings.weight.is_cuda:
            return None
        from .. import ops
        if not ops.available():
            return None
        if self._pretrainer is None:
            from .fused import FusedPretrainer
            self._pretrainer = FusedPretrainer(self)
        return self._pretrainer

    @torch.no_grad()
    def evaluate(self, input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels, acc: torch.Tensor,
                 tokens: Optional[int] = None) -> torch.Tensor:
        """Adds the held-out metric sums of one batch into ``acc`` (fp64 [6]): ``[mlm_loss_sum, mlm_correct, mlm_count,
        nsp_loss_sum, nsp_correct, nsp_count]`` over the rows whose label is not -1.  Through the fused engine
        (:meth:`~.fused.FusedPretrainer.evaluate`) where it runs, else from the plain PyTorch forward with dropout off
        (autocast is the caller's), with the same rule for ties: the lowest index wins an argmax."""
        eng = self.pretrain_engine()
        if eng is not None:
            return eng.evaluate(input_ids, segment_ids, input_mask, masked_lm_labels, next_sentence_labels, acc,
                                tokens=tokens)
        was = self.training
        self.eval()
        try:
            scores, nsp = self(input_ids.long(), None if segment_ids is None else segment_ids.long(), input_mask.long())
        finally:
            self.train(was)
        acc[0:3] += _metric_sums(scores.reshape(-1, scores.size(-1)), masked_lm_labels.reshape(-1))
        if nsp is not None and next_sentence_labels is not None:
            acc[3:6] += _metric_sums(nsp.reshape(-1, 2), next_sentence_labels.reshape(-1))
        return acc


class BertForMaskedLM(BertPreTrainedModel):
    def __init__(self, config: BertConfig):
        super().__init__(config)
        self.bert = BertModel(config)
        self.cls = BertOnlyMLMHead(config, self.bert.embeddings.word_embeddings.weight)
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, masked_lm_labels=None):
        layers, _ = self.bert(input_ids, token_type_ids, attention_mask)
        seq = layers[-1]
        scores = self.cls(seq)
        if masked_lm_labels is not None:
            return F.cross_entropy(scores.view(-1, scores.size(-1)).float(), masked_lm_labels.view(-1),
                                   ignore_index=-1)
        return scores


def _require_pooled(pooled):
    if pooled is None:
        raise ValueError("this head needs the pooler, which only exists when config.next_sentence "
                         "is true (reference quirk Q13: it crashes with an AttributeError there)")
    return pooled


class BertForNextSentencePrediction(BertPreTrainedModel):
    def __init__(self, config: BertConfig):
        super().__init__(config)
        self.bert = BertModel(config)
        self.cls = BertOnlyNSPHead(config)
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, next_sentence_label=None):
        _, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        score = self.cls(_require_pooled(pooled))
        if next_sentence_label is not None:
            return F.cross_entropy(score.view(-1, 2).float(), next_sentence_label.view(-1), ignore_index=-1)
        return score


class BertForSequenceClassification(BertPreTrainedModel):
    def __init__(self, config: BertConfig, num_labels: int):
        super().__init__(config)
        self.num_labels = num_labels
        self.bert = BertModel(config)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.classifier = nn.Linear(config.hidden_size, num_labels)
        self._classifier = None
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        _, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        logits = self.classifier(self.dropout(_require_pooled(pooled)))
        if labels is not None:
            return F.cross_entropy(logits.view(-1, self.num_labels).float(), labels.view(-1))
        return logits

    def classifier_engine(self):
        """The fused sm_90a training / evaluation program of this model (:class:`~.fused.FusedClassifier`), or
        ``None`` where it cannot run: ``_can_fuse`` fails for ``input_ids``, the model has no pooler, or the label count
        is not one the classifier kernel is built for (2 or 3)."""
        from ..ops.api import CLS_CLASSES
        if self.bert.pooler is None or self.num_labels not in CLS_CLASSES:
            return None
        if self._classifier is None:
            from .fused import FusedClassifier
            self._classifier = FusedClassifier(self)
        return self._classifier

    def _fused(self, input_ids):
        return self.classifier_engine() if self.bert._can_fuse(input_ids) else None

    def train_step(self, input_ids, token_type_ids, attention_mask, labels, grad_scale: float = 1.0,
                   tokens: Optional[int] = None) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the mean cross-entropy over the rows whose label is not -1
        and accumulates the gradients (times ``grad_scale``) into ``.grad``.  Through the fused program
        (:meth:`~.fused.FusedClassifier.train_step`, dropout as ``self.training`` says) where it runs, else the plain
        PyTorch forward and backward (autocast is the caller's).  ``tokens``: the unmasked token count of the batch
        (a host int) for the unpadded program's bucket."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.train_step(input_ids, token_type_ids, attention_mask, labels, grad_scale, tokens=tokens)
        logits = self(input_ids.long(), None if token_type_ids is None else token_type_ids.long(), attention_mask.long())
        loss = F.cross_entropy(logits.view(-1, self.num_labels).float(), labels.long().view(-1), ignore_index=-1)
        if not bool((labels >= 0).any()):
            loss = logits.sum() * 0.0          # every row ignored: loss 0 and zero gradients, not NaN
        (loss * grad_scale).backward()
        return loss.detach()

    @torch.no_grad()
    def predict(self, input_ids, token_type_ids, attention_mask, tokens: Optional[int] = None) -> torch.Tensor:
        """fp32 logits [B, num_labels] without dropout.  Through the fused program
        (:meth:`~.fused.FusedClassifier.predict`) where it runs, else the plain PyTorch forward in eval mode (autocast
        is the caller's); ``self.training`` is left as it was."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.predict(input_ids, token_type_ids, attention_mask, tokens=tokens)
        was = self.training
        self.eval()
        try:
            logits = self(input_ids.long(), None if token_type_ids is None else token_type_ids.long(),
                          attention_mask.long())
        finally:
            self.train(was)
        return logits.float()


class BertForMultipleChoice(BertPreTrainedModel):
    def __init__(self, config: BertConfig, num_choices: int):
        super().__init__(config)
        self.num_choices = num_choices
        self.bert = BertModel(config)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.classifier = nn.Linear(config.hidden_size, 1)
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        flat = lambda t: None if t is None else t.view(-1, t.size(-1))
        _, pooled = self.bert(flat(input_ids), flat(token_type_ids), flat(attention_mask))
        logits = self.classifier(self.dropout(_require_pooled(pooled))).view(-1, self.num_choices)
        if labels is not None:
            return F.cross_entropy(logits.float(), labels)
        return logits


def _head(linear: nn.Linear, x: torch.Tensor) -> torch.Tensor:
    """Small-N head projection: the wgmma GEMM path on CUDA (models/fused.py:head_linear), ``linear(x)`` elsewhere."""
    if x.is_cuda:
        from .fused import head_linear
        return head_linear(linear, x)
    return linear(x)


class BertForTokenClassification(BertPreTrainedModel):
    """Per-token classifier; the loss only counts positions with
    ``attention_mask == 1`` (src/modeling.py:1259-1268)."""

    def __init__(self, config: BertConfig, num_labels: int):
        super().__init__(config)
        self.num_labels = num_labels
        self.bert = BertModel(config)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.classifier = nn.Linear(config.hidden_size, num_labels)
        self._token_program = None
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        layers, _ = self.bert(input_ids, token_type_ids, attention_mask)
        seq = layers[-1]
        logits = _head(self.classifier, self.dropout(seq))          # K29: own small-N GEMM on an H100
        if labels is not None:
            flat_logits = logits.view(-1, self.num_labels).float()
            flat_labels = labels.view(-1)
            if attention_mask is not None:
                keep = attention_mask.view(-1) == 1
                flat_logits, flat_labels = flat_logits[keep], flat_labels[keep]
            return F.cross_entropy(flat_logits, flat_labels)
        return logits

    def token_engine(self):
        """The fused sm_90a training / prediction program of this model (:class:`~.fused.FusedTokenClassifier`), or
        ``None`` where it cannot run: more labels than the per-token head kernels serve (64)."""
        from ..ops.api import TOKEN_HEAD_MAX_N
        if self.num_labels > TOKEN_HEAD_MAX_N:
            return None
        if self._token_program is None:
            from .fused import FusedTokenClassifier
            self._token_program = FusedTokenClassifier(self)
        return self._token_program

    def _fused(self, input_ids):
        return self.token_engine() if self.bert._can_fuse(input_ids) else None

    def train_step(self, input_ids, token_type_ids, attention_mask, labels, grad_scale: float = 1.0,
                   tokens: Optional[int] = None) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the mean cross-entropy over the positions whose
        ``attention_mask`` is 1 and whose label lies in [0, num_labels) (every other label, -100 or -1, is ignored; 0
        when nothing counts) and accumulates the gradients (times ``grad_scale``) into ``.grad``.  Through the fused
        program (:meth:`~.fused.FusedTokenClassifier.train_step`) where it runs, else the plain PyTorch forward and
        backward (autocast is the caller's).  ``tokens``: the unmasked token count (a host int) for the unpadded
        program's bucket."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.train_step(input_ids, token_type_ids, attention_mask, labels, grad_scale, tokens=tokens)
        logits = self(input_ids.long(), None if token_type_ids is None else token_type_ids.long(), attention_mask.long())
        loss = token_loss(logits, labels, attention_mask)
        (loss * grad_scale).backward()
        return loss.detach()

    @torch.no_grad()
    def predict(self, input_ids, token_type_ids, attention_mask, tokens: Optional[int] = None) -> torch.Tensor:
        """fp32 logits [B, S, num_labels] without dropout.  Through the fused program
        (:meth:`~.fused.FusedTokenClassifier.predict`) where it runs, else the plain PyTorch forward in eval mode
        (autocast is the caller's); ``self.training`` is left as it was."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.predict(input_ids, token_type_ids, attention_mask, tokens=tokens)
        return _eval_forward(self, input_ids, token_type_ids, attention_mask).float()


class BertForQuestionAnswering(BertPreTrainedModel):
    def __init__(self, config: BertConfig):
        super().__init__(config)
        self.bert = BertModel(config)
        self.qa_outputs = nn.Linear(config.hidden_size, 2)
        self._qa_program = None
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None):
        layers, _ = self.bert(input_ids, token_type_ids, attention_mask)
        seq = layers[-1]
        logits = _head(self.qa_outputs, seq)                        # K28: own small-N GEMM on an H100
        start, end = logits.split(1, dim=-1)
        return start.squeeze(-1), end.squeeze(-1)

    def qa_engine(self):
        """The fused sm_90a training / prediction program of this model (:class:`~.fused.FusedQuestionAnswering`)."""
        if self._qa_program is None:
            from .fused import FusedQuestionAnswering
            self._qa_program = FusedQuestionAnswering(self)
        return self._qa_program

    def _fused(self, input_ids):
        return self.qa_engine() if self.bert._can_fuse(input_ids) else None

    def train_step(self, input_ids, token_type_ids, attention_mask, start_positions, end_positions,
                   grad_scale: float = 1.0) -> torch.Tensor:
        """Forward, loss and backward of one batch: returns the SQuAD loss (:func:`span_loss`) and accumulates the
        gradients (times ``grad_scale``) into ``.grad``.  Through the fused program
        (:meth:`~.fused.FusedQuestionAnswering.train_step`, always padded) where it runs, else the plain PyTorch
        forward and backward (autocast is the caller's)."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.train_step(input_ids, token_type_ids, attention_mask, start_positions, end_positions, grad_scale)
        start, end = self(input_ids.long(), None if token_type_ids is None else token_type_ids.long(),
                          attention_mask.long())
        loss = span_loss(start, end, start_positions, end_positions)
        (loss * grad_scale).backward()
        return loss.detach()

    @torch.no_grad()
    def predict(self, input_ids, token_type_ids, attention_mask, tokens: Optional[int] = None):
        """fp32 ``(start, end)`` logits, each [B, S], without dropout.  Through the fused program
        (:meth:`~.fused.FusedQuestionAnswering.predict`) where it runs, else the plain PyTorch forward in eval mode
        (autocast is the caller's); ``self.training`` is left as it was."""
        eng = self._fused(input_ids)
        if eng is not None:
            return eng.predict(input_ids, token_type_ids, attention_mask, tokens=tokens)
        start, end = _eval_forward(self, input_ids, token_type_ids, attention_mask)
        return start.float(), end.float()


def _eval_forward(model, input_ids, token_type_ids, attention_mask):
    """``model``'s forward in eval mode (no dropout), ``model.training`` restored afterwards."""
    was = model.training
    model.eval()
    try:
        return model(input_ids.long(), None if token_type_ids is None else token_type_ids.long(), attention_mask.long())
    finally:
        model.train(was)


def span_loss(start_logits, end_logits, start_positions, end_positions):
    """The SQuAD loss (run_squad.py:1085-1092): positions are clamped to [0, S] and S is ignored; the mean start and
    the mean end cross-entropy, each over its own non-ignored sequences, averaged.  A column with no such sequence
    contributes 0 (and a zero gradient) instead of NaN."""
    S = start_logits.size(1)
    total = 0.0
    for logits, pos in ((start_logits, start_positions), (end_logits, end_positions)):
        y = pos.long().to(logits.device).clamp(0, S)
        n = (y != S).sum().clamp(min=1)
        total = total + F.cross_entropy(logits.float(), y, ignore_index=S, reduction="sum") / n
    return total / 2


def token_loss(logits, labels, attention_mask):
    """The NER loss: the mean cross-entropy over the positions whose ``attention_mask`` is 1 and whose label lies in
    [0, num_labels) (src/modeling.py:1259-1268 masks by attention_mask; -100 and -1 are ignored); 0 with a zero
    gradient when no position counts."""
    N = logits.size(-1)
    flat = logits.reshape(-1, N).float()
    y = labels.reshape(-1).long().to(flat.device)
    keep = (attention_mask.reshape(-1).to(flat.device) == 1) & (y >= 0) & (y < N)
    y = torch.where(keep, y, torch.full_like(y, -100))
    return F.cross_entropy(flat, y, ignore_index=-100, reduction="sum") / keep.sum().clamp(min=1)


class BertPretrainingCriterion(nn.Module):
    """Mean CE over labels != -1 (MLM) + mean CE (NSP), summed
    (run_pretraining.py:58-72)."""

    def __init__(self, vocab_size: int):
        super().__init__()
        self.vocab_size = vocab_size

    def forward(self, prediction_scores, masked_lm_labels, seq_relationship_score=None,
                next_sentence_labels=None):
        loss = F.cross_entropy(prediction_scores.view(-1, self.vocab_size).float(),
                               masked_lm_labels.view(-1), ignore_index=-1)
        if seq_relationship_score is not None and next_sentence_labels is not None:
            loss = loss + F.cross_entropy(seq_relationship_score.view(-1, 2).float(),
                                          next_sentence_labels.view(-1), ignore_index=-1)
        return loss


def count_parameters(model: nn.Module) -> Tuple[int, int]:
    """(number of elements, number of tensors), tied tensors counted once."""
    seen, n = set(), 0
    for p in model.parameters():          # parameters() already yields tied tensors once
        if id(p) in seen:
            continue
        seen.add(id(p))
        n += p.numel()
    return n, len(seen)
