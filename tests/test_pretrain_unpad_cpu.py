"""Unpadded pre-training without a GPU: the ``--unpad`` flag, the token buckets, the host token count against a numpy
packing oracle, the CPU path's indifference to the flag, and the argument checks of the new bindings (host tensors:
everything is refused before a launch)."""
import json
import os

import numpy as np
import pytest
import torch

from bert_pytorch_b200 import pretrain
from bert_pytorch_b200.models.fused import MAX_TOKEN_BUCKETS, packed_tokens, token_bucket


def np_pack(mask, ids, seg, T_cap, D):
    """numpy oracle of the device packing (ops.api.pack_tokens): -> dict of every output."""
    mask = np.asarray(mask)
    B, S = mask.shape
    keep = mask != 0
    keep[~keep.any(1)] = True                   # a row without unmasked tokens packs as S tokens
    rows = np.flatnonzero(keep.reshape(-1))
    T = rows.size
    assert T <= T_cap and D * S >= T_cap - T
    out = {"ids": np.zeros(T_cap, np.int32), "seg": np.zeros(T_cap, np.int32),
           "pos": (np.arange(T_cap) - T) % S, "row_map": np.full(B * S, -1, np.int32)}
    out["ids"][:T] = np.asarray(ids).reshape(-1)[rows]
    out["seg"][:T] = np.asarray(seg).reshape(-1)[rows]
    out["pos"][:T] = rows % S
    out["pos"] = out["pos"].astype(np.int32)
    out["row_map"][rows] = np.arange(T)
    lens = keep.sum(1)
    cu = np.concatenate([[0], np.cumsum(lens)])
    out["cls"] = cu[:-1].astype(np.int32)
    out["cu"] = np.concatenate([cu, np.minimum(T_cap, T + S * np.arange(1, D + 1))]).astype(np.int32)
    out["T"] = T
    return out


def masks(B=6, S=64, seed=0):
    """Prefix masks, holes, empty rows and full rows."""
    g = np.random.default_rng(seed)
    m = (np.arange(S)[None, :] < g.integers(1, S + 1, (B, 1))).astype(np.int32)
    m[0] = 1                                    # full
    m[1] = 0                                    # empty
    m[2, 3:9] = 0                               # holes
    m[3, 1::3] = 0
    return m


# ---- flag ------------------------------------------------------------------------------------------------------------
def test_unpad_flag_default_cli_and_json(tmp_path):
    base = ["--output_dir", "o"]
    assert pretrain.parse_arguments(base).unpad is False
    assert pretrain.parse_arguments(base + ["--unpad"]).unpad is True
    cfg = tmp_path / "c.json"
    cfg.write_text(json.dumps({"unpad": True}))
    assert pretrain.parse_arguments(base + ["--config_file", str(cfg)]).unpad is True


# ---- buckets ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S", [(96, 128), (16, 512), (8, 128), (3, 64), (1, 128), (5, 8), (64, 512)])
def test_token_bucket_bounds_alignment_tail_and_count(B, S):
    M = B * S
    caps = set()
    for T in range(1, M + 1):
        T_cap, D = token_bucket(T, B, S)
        assert T <= T_cap <= M
        assert T_cap % 128 == 0 or T_cap == M
        assert D * S >= T_cap - T and D >= 1
        caps.add(T_cap)
    assert len(caps) <= MAX_TOKEN_BUCKETS
    assert M in caps
    for T in (0, M + 1):
        with pytest.raises(ValueError):
            token_bucket(T, B, S)


def test_token_bucket_phase_shapes():
    assert token_bucket(96 * 128, 96, 128) == (12288, 6)       # phase 1: step 768 rows, 6 dummies of 128
    assert token_bucket(1, 96, 128) == (768, 6)
    assert token_bucket(16 * 512, 16, 512) == (8192, 1)        # phase 2: step 512 rows, one dummy of 512
    assert token_bucket(4097, 16, 512) == (4608, 1)


# ---- host count ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_packed_tokens_matches_numpy_oracle(seed):
    m = masks(seed=seed)
    want = np_pack(m, np.zeros_like(m), np.zeros_like(m), m.size, m.shape[0])["T"]
    for t in (torch.from_numpy(m), torch.from_numpy(m).long(), torch.from_numpy(m).bool()):
        assert packed_tokens(t) == want
    assert packed_tokens(torch.zeros(3, 16, dtype=torch.int32)) == 48
    assert packed_tokens(torch.ones(3, 16, dtype=torch.int32)) == 48
    assert packed_tokens(torch.tensor([[1, 0, 1, 0], [0, 0, 0, 0]])) == 2 + 4


def test_numpy_oracle_self_consistency():
    """The oracle's own invariants: packed rows in b*S+s order, sequences contiguous, dummies of at most S rows."""
    m = masks(B=5, S=32)
    ids = np.arange(m.size, dtype=np.int32).reshape(m.shape) + 100
    T = np_pack(m, ids, ids, m.size, 5)["T"]
    T_cap, D = token_bucket(T, 5, 32)
    o = np_pack(m, ids, ids, T_cap, D)
    assert (np.diff(o["cu"]) >= 0).all() and (np.diff(o["cu"][5:]) <= 32).all() and o["cu"][-1] == T_cap
    r = o["row_map"]
    assert (o["ids"][r[r >= 0]] == ids.reshape(-1)[r >= 0]).all()
    assert (o["ids"][T:] == 0).all() and (o["pos"][T:] < 32).all()


# ---- CPU path --------------------------------------------------------------------------------------------------------
def test_cpu_path_loss_is_the_same_with_unpad(tmp_path):
    from bert_pytorch_b200.data import synthetic
    data, model_json, _ = synthetic.make_workspace(str(tmp_path / "w"), num_shards=2, samples_per_shard=16, seq_len=64,
                                                   vocab_size=500, hidden_size=32, num_hidden_layers=1,
                                                   num_attention_heads=2, intermediate_size=64,
                                                   max_position_embeddings=64, hidden_dropout_prob=0.0,
                                                   attention_probs_dropout_prob=0.0)
    losses = []
    for extra in ([], ["--unpad"]):
        out = str(tmp_path / f"o{len(extra)}" / "out")
        os.makedirs(os.path.dirname(out))
        pretrain.cli(["--input_dir", data, "--output_dir", out, "--model_config_file", model_json, "--device", "cpu",
                      "--max_predictions_per_seq", "10", "--global_batch_size", "8", "--local_batch_size", "4",
                      "--max_steps", "2", "--steps", "2", "--skip_checkpoint", "--disable_progress_bar",
                      "--learning_rate", "1e-3", *extra])
        import csv
        rows = list(csv.DictReader(open(os.path.join(out, "logfile_metrics.csv"))))
        losses.append([float(r["average_loss"]) for r in rows])
    assert losses[0] == losses[1] and len(losses[0]) == 2


# ---- bindings --------------------------------------------------------------------------------------------------------
def _ext():
    from bert_pytorch_b200.ops import _loader
    if not os.path.exists(_loader.extension_path()):
        pytest.skip("extension not built (python -m bert_pytorch_b200.ops.build)")
    return _loader.load_extension()


def test_pack_tokens_binding_refuses_host_tensors_and_bad_shapes():
    C = _ext()
    B, S, T_cap, D = 3, 64, 128, 1
    i32 = dict(dtype=torch.int32)
    mask = torch.ones(B, S, **i32)

    def outs(T=T_cap, d=D):
        return (torch.empty(T, **i32), torch.empty(T, **i32), torch.empty(T, **i32), torch.empty(B + d + 1, **i32),
                torch.empty(B, **i32), torch.empty(B * S, **i32))
    for seg in (mask, None):
        with pytest.raises(RuntimeError, match="CUDA"):
            C.pack_tokens(mask, mask, seg, T_cap, D, *outs())


def test_mlm_compact_binding_refuses_a_host_row_map():
    C = _ext()
    labels = torch.full((2, 16), -1, dtype=torch.int32)
    idx, tgt, count = torch.empty(8, dtype=torch.int32), torch.empty(8, dtype=torch.int32), torch.empty(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        C.mlm_compact(labels, 4, idx, tgt, count, torch.zeros(32, dtype=torch.int32))
