"""Unpadded mode without a GPU: the runners' ``--unpad`` flags, the CPU path's indifference to ``BertModel.unpad``,
the packing record, and the attention bindings' argument checks (host tensors: everything is refused before a launch)."""
import os

import pytest
import torch

from bert_pytorch_b200.config import BertConfig
from bert_pytorch_b200.models import BertForTokenClassification
from bert_pytorch_b200.models.fused import pack_rows


def test_runners_parse_unpad_default_off():
    from bert_pytorch_b200 import finetune_ner, finetune_squad
    base = ["--train_file", "t", "--labels", "A", "--model_config_file", "c", "--model_checkpoint", "k"]
    assert finetune_ner.parse_arguments(base).unpad is False
    assert finetune_ner.parse_arguments(base + ["--unpad"]).unpad is True
    sq = ["--bert_model", "b", "--output_dir", "o", "--init_checkpoint", "i", "--config_file", "c"]
    assert finetune_squad.build_parser().parse_args(sq).unpad is False
    assert finetune_squad.build_parser().parse_args(sq + ["--unpad"]).unpad is True


def test_unpad_leaves_the_cpu_path_unchanged():
    torch.manual_seed(0)
    cfg = BertConfig(vocab_size_or_config_json_file=128, hidden_size=64, num_hidden_layers=2, num_attention_heads=1,
                     intermediate_size=128, max_position_embeddings=64)
    model = BertForTokenClassification(cfg, num_labels=5).eval()
    ids = torch.randint(1, 128, (3, 16))
    mask = torch.zeros(3, 16, dtype=torch.long)
    mask[0, :16] = 1
    mask[1, :5] = 1
    mask[2, [0, 1, 4, 9]] = 1
    assert model.bert.unpad is False
    with torch.no_grad():
        ref = model(ids, attention_mask=mask)
        model.bert.unpad = True
        got = model(ids, attention_mask=mask)
    assert torch.equal(ref, got)


def test_pack_rows_handles_masks_with_holes_and_empty_sequences():
    mask = torch.tensor([[1, 1, 0, 0], [0, 0, 0, 0], [1, 0, 1, 1]])
    pk = pack_rows(mask)
    assert pk.T == 5 and pk.S == 4
    assert pk.rows.dtype == torch.int32 and pk.rows.tolist() == [0, 1, 8, 10, 11]
    assert pk.cu_seqlens.tolist() == [0, 2, 2, 5]
    assert pk.pos_ids.tolist() == [0, 1, 0, 2, 3]
    assert pack_rows(torch.zeros(2, 8, dtype=torch.long)).T == 0


def _ext():
    from bert_pytorch_b200.ops import _loader
    if not os.path.exists(_loader.extension_path()):
        pytest.skip("extension not built (python -m bert_pytorch_b200.ops.build)")
    return _loader.load_extension()


def _fwd(C, qkv, seqlens, lse, heads, cu=None, S=0, fp8=False):
    ctx = torch.empty(*qkv.shape[:-1], qkv.size(-1) // 3, dtype=torch.bfloat16)
    q8 = torch.empty(ctx.shape, dtype=torch.uint8) if fp8 else None
    meta = torch.ones(4) if fp8 else None
    C.attention_fwd(qkv, seqlens, ctx, lse, heads, 0.125, 0.0, 0, 0, q8, meta, False, cu, S)


def _bwd(C, qkv, seqlens, lse, heads, cu=None, S=0, fp8=False):
    H = qkv.size(-1) // 3
    ctx = torch.empty(*qkv.shape[:-1], H, dtype=torch.bfloat16)
    q8 = torch.empty(qkv.shape, dtype=torch.uint8) if fp8 else None
    meta = torch.ones(4) if fp8 else None
    C.attention_bwd(qkv, seqlens, ctx, ctx, lse, torch.empty_like(qkv), torch.empty_like(lse),
                    torch.empty(ctx.numel()), heads, 0.125, 0.0, 0, 0, q8, meta, False, cu, S)


@pytest.mark.parametrize("call", [_fwd, _bwd], ids=["fwd", "bwd"])
def test_attention_bindings_reject_bad_arguments(call):
    C = _ext()
    B, S, heads, T = 3, 128, 2, 200
    qkv = torch.zeros(T, 3 * 64 * heads, dtype=torch.bfloat16)
    lse = torch.empty(B, heads, S)
    good = torch.tensor([0, 64, 64, T], dtype=torch.int32)
    for bad in (good.long(), good[:-1].contiguous(), torch.tensor([0, 64, 64, T, T], dtype=torch.int32),
                torch.stack([good, good], 1)[:, 0]):
        with pytest.raises(RuntimeError, match="cu_seqlens"):
            call(C, qkv, None, lse, heads, cu=bad, S=S)
    with pytest.raises(RuntimeError, match="fp8"):
        call(C, qkv, None, lse, heads, cu=good, S=S, fp8=True)
    with pytest.raises(RuntimeError, match="head dim"):
        call(C, torch.zeros(T, 3 * 96, dtype=torch.bfloat16), None, torch.empty(B, 1, S), 1, cu=good, S=S)
    for bad_S in (520, 100):
        with pytest.raises(RuntimeError, match="S <= 512"):
            call(C, qkv, None, torch.empty(B, heads, bad_S), heads, cu=good, S=bad_S)
    # the padded form: the same limits raise instead of aborting the process
    lens = torch.full((B,), 8, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="head dim"):
        call(C, torch.zeros(B, S, 3 * 96, dtype=torch.bfloat16), lens, torch.empty(B, 1, S), 1)
    with pytest.raises(RuntimeError, match="S <= 512"):
        call(C, torch.zeros(B, 520, 3 * 64, dtype=torch.bfloat16), lens, torch.empty(B, 1, 520), 1)
