import copy
import json
import math
import os

import numpy as np
import pytest
import torch

from bert_pytorch_b200 import BertConfig, kfac
from bert_pytorch_b200 import models as M
from bert_pytorch_b200.data import corpus, encode, hdf5, ner, squad
from bert_pytorch_b200.data.tokenization import BertTokenizer, get_wordpiece_tokenizer
from bert_pytorch_b200.parallel import FakeComm


def _cfg(**kw):
    base = dict(vocab_size_or_config_json_file=64, hidden_size=16, num_hidden_layers=1, num_attention_heads=2,
                intermediate_size=32, max_position_embeddings=32, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    base.update(kw)
    return BertConfig(**base)


# ---------------------------------------------------------------------------------------------- K-FAC
def test_kfac_registration_matches_reference_defaults():
    m = M.BertForPreTraining(_cfg())
    k = kfac.KFAC(m, skip_layers=["BertLMPredictionHead", "embedding"])
    names = k.layer_names()
    assert "cls.predictions.decoder" not in names                      # skipped through its parent class name
    assert {"bert.encoder.layer.0.attention.self.query", "bert.encoder.layer.0.attention.self.key",
            "bert.encoder.layer.0.attention.self.value", "bert.encoder.layer.0.attention.output.dense",
            "bert.encoder.layer.0.output.dense", "cls.seq_relationship"} == set(names)
    assert "lr" in k.param_groups[0]


def test_kfac_single_linear_matches_closed_form():
    torch.manual_seed(0)
    lin = torch.nn.Linear(5, 3)
    model = torch.nn.Sequential(lin)
    k = kfac.KFAC(model, lr=0.1, factor_decay=0.95, damping=0.003, kl_clip=None, factor_update_freq=1, inv_update_freq=1)
    x = torch.randn(7, 5)
    model.train()
    loss = model(x).pow(2).mean()
    loss.backward()
    gW, gb = lin.weight.grad.clone(), lin.bias.grad.clone()
    # closed form
    a = torch.cat([x, torch.ones(7, 1)], 1)
    A = a.t() @ a / 7
    gout = (2 * model(x) / (7 * 3)).detach()
    G = gout.t() @ gout * 7
    Wg = torch.cat([gW, gb[:, None]], 1)
    dA, QA = torch.linalg.eigh(A); dG, QG = torch.linalg.eigh(G)
    P = QG @ ((QG.t() @ Wg @ QA) / (dG[:, None] * dA[None, :] + 0.003)) @ QA.t()
    k.step()
    got = torch.cat([lin.weight.grad, lin.bias.grad[:, None]], 1)
    assert torch.allclose(got, P, rtol=1e-3, atol=1e-4)
    sd = k.state_dict()
    k2 = kfac.KFAC(torch.nn.Sequential(torch.nn.Linear(5, 3)), factor_update_freq=1, inv_update_freq=1)
    k2.load_state_dict(sd)
    assert k2.steps == 1 and torch.allclose(k2.layers[0].A, A, atol=1e-5)


def test_kfac_kl_clip_and_distributed_equivalence():
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.Tanh(), torch.nn.Linear(4, 2))
    xs = [torch.randn(8, 6) for _ in range(3)]

    def run(comm, x):
        m = copy.deepcopy(base).train()
        k = kfac.KFAC(m, lr=1.0, kl_clip=1e-3, factor_update_freq=1, inv_update_freq=1, comm=comm,
                      comm_method=kfac.CommMethod.HYBRID_OPT, grad_worker_fraction=0.5)
        m(x).pow(2).mean().backward()
        if comm is not None and comm.world_size > 1:
            for p in m.parameters():
                comm.all_reduce_(p.grad, op="avg")
        raw = sum(float((p.grad ** 2).sum()) for p in m.parameters())
        k.step()
        return [p.grad.clone() for p in m.parameters()], raw

    grads, raw = run(None, xs[0])
    assert all(torch.isfinite(g).all() for g in grads)
    # three ranks with different data agree with each other after the step
    outs = FakeComm.spawn(3, lambda c: run(c, xs[c.rank])[0])
    for g0, g1, g2 in zip(*outs):
        assert torch.allclose(g0, g1, atol=1e-6) and torch.allclose(g0, g2, atol=1e-6)


def _kfac_gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="env://")
    from bert_pytorch_b200.parallel import TorchComm
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.Tanh(), torch.nn.Linear(4, 3), torch.nn.Tanh(),
                               torch.nn.Linear(3, 2)).train()
    xs = [torch.randn(8, 6) for _ in range(world)]
    comm = TorchComm()
    k = kfac.KFAC(base, lr=1.0, kl_clip=1e-3, factor_update_freq=1, inv_update_freq=1, comm=comm,
                  comm_method=kfac.CommMethod.HYBRID_OPT, grad_worker_fraction=0.5, inv_dtype=torch.float32)
    for _ in range(2):                                   # second step: receivers re-use their allocated eigen buffers
        for p in base.parameters():
            p.grad = None
        base(xs[rank]).pow(2).mean().backward()
        for p in base.parameters():
            comm.all_reduce_(p.grad, op="avg")
        k.step()
    # by value: a tensor in a queue is a file descriptor served by this process, which may exit before the parent reads it
    q.put((rank, [p.grad.numpy().copy() for p in base.parameters()]))
    dist.barrier()
    dist.destroy_process_group()


def test_kfac_hybrid_groups_over_gloo_four_ranks_match_single_process():
    """HYBRID_OPT at 4 ranks = gradient-worker groups of 2 (reference recipe: run_pretraining.py:321-345): eigen-pairs go
    to the group, preconditioned gradients to the ranks outside it, through real sub-group broadcasts (eigh hands back
    column-major eigenvectors: the payloads must be made dense first -- the 4-GPU bench of round 2 tripped over that).
    Every rank must end with the single-process result on the concatenated batch."""
    import torch.multiprocessing as mp
    world, port = 4, 29671
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_kfac_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in range(world)], key=lambda t: t[0])
    res = [(r, [torch.from_numpy(a) for a in gs]) for r, gs in res]
    for p in procs:
        p.join(timeout=60)
    for r in range(1, world):
        for g0, g in zip(res[0][1], res[r][1]):
            assert torch.allclose(g0, g, atol=1e-5), (r, (g0 - g).abs().max())
    # single process, same data: factors are averages over micro-batches == averages over ranks
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(6, 4), torch.nn.Tanh(), torch.nn.Linear(4, 3), torch.nn.Tanh(),
                               torch.nn.Linear(3, 2)).train()
    xs = [torch.randn(8, 6) for _ in range(world)]
    k = kfac.KFAC(base, lr=1.0, kl_clip=1e-3, factor_update_freq=1, inv_update_freq=1, accumulate_data=True,
                  inv_dtype=torch.float32)
    for _ in range(2):
        for p in base.parameters():
            p.grad = None
        for x in xs:
            base(x).pow(2).mean().backward()         # unscaled micro-losses feed the taps exactly like one rank each
        for p in base.parameters():
            p.grad /= world
        k.step()
    for g0, g in zip(res[0][1], [p.grad for p in base.parameters()]):
        assert torch.allclose(g0, g, atol=1e-4, rtol=1e-3), (g0 - g).abs().max()


# ---------------------------------------------------------------------------------------------- SQuAD
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "the", "capital", "of", "france", "is", "paris", ".", "what", "?",
         "berlin", "germany", "and", "city", "a", "big", "##s", "river", "seine", "flows", "through", "who", "wrote",
         "hamlet", "shakespeare", "william", "play", "was", "by", "written"]


@pytest.fixture
def squad_files(tmp_path):
    vf = tmp_path / "vocab.txt"
    vf.write_text("\n".join(VOCAB) + "\n")
    data = {"version": "1.1", "data": [{"title": "t", "paragraphs": [
        {"context": "The capital of France is Paris. The river Seine flows through Paris.",
         "qas": [{"id": "q1", "question": "What is the capital of France?", "answers": [{"text": "Paris", "answer_start": 25}]},
                 {"id": "q2", "question": "What river flows through Paris?", "answers": [{"text": "Seine", "answer_start": 42}]}]},
        {"context": "Hamlet is a play. The play was written by William Shakespeare.",
         "qas": [{"id": "q3", "question": "Who wrote Hamlet?", "answers": [{"text": "William Shakespeare", "answer_start": 42}]}]}]}]}
    f = tmp_path / "train.json"
    f.write_text(json.dumps(data))
    return str(f), str(vf)


def test_squad_featurizer_windows_and_answer_alignment(squad_files):
    f, vf = squad_files
    tok = get_wordpiece_tokenizer(vf)
    ex = squad.read_squad_examples(f, True, False)
    assert len(ex) == 3 and ex[0].doc_tokens[ex[0].start_position] == "Paris."
    feats = squad.convert_examples_to_features(ex, tok, max_seq_length=18, doc_stride=3, max_query_length=8, is_training=True)
    assert len(feats) > 3                                           # sliding windows
    for ft in feats:
        assert len(ft.input_ids) == len(ft.input_mask) == len(ft.segment_ids) == 18
        assert ft.tokens[0] == "[CLS]" and ft.input_ids[0] == 2
        if ft.start_position:                                         # answer inside the window -> exact tokens
            span = ft.tokens[ft.start_position:ft.end_position + 1]
            e = ex[ft.example_index]
            assert " ".join(span).replace(" ##", "") in " ".join(tok.encode(e.orig_answer_text, add_special_tokens=False).tokens) \
                or " ".join(tok.encode(e.orig_answer_text, add_special_tokens=False).tokens) in " ".join(span).replace(" ##", "")
    # every doc token is 'max context' in exactly one window
    by_ex = {}
    for ft in feats:
        for pos, orig in ft.token_to_orig_map.items():
            if ft.token_is_max_context[pos]:
                by_ex.setdefault((ft.example_index, orig, ft.tokens[pos], pos - 0), 0)
    assert by_ex


def test_squad_postprocessing_em_f1(squad_files):
    f, vf = squad_files
    tok = get_wordpiece_tokenizer(vf)
    ex = squad.read_squad_examples(f, False, False)
    feats = squad.convert_examples_to_features(ex, tok, 48, 16, 12, False)
    results = []
    gold = {"q1": "paris", "q2": "seine", "q3": "shakespeare"}
    for ft in feats:
        s = [-5.0] * 48; e = [-5.0] * 48
        want = gold[ex[ft.example_index].qas_id]
        for i, t in enumerate(ft.tokens):
            if t == want and i in ft.token_to_orig_map:
                s[i] = e[i] = 5.0
                if want == "shakespeare":
                    s[i - 1] = 6.0
                break
        results.append(squad.RawResult(ft.unique_id, s, e))
    answers, nbest = squad.get_answers(ex, feats, results, n_best_size=5, max_answer_length=10, do_lower_case=True)
    assert answers["q1"] == "Paris" and answers["q2"] == "Seine" and answers["q3"] == "William Shakespeare"
    assert abs(sum(p["probability"] for p in nbest["q1"]) - 1.0) < 1e-6
    scores = squad.evaluate_predictions(f, answers)
    assert scores["exact_match"] == 100.0 and scores["f1"] == 100.0
    assert squad.f1_score("the William", "William Shakespeare") == pytest.approx(2 * 1.0 * 0.5 / 1.5)
    # v2: null answer wins when its score beats the best span by more than the threshold
    res2 = [squad.RawResult(r.unique_id, [9.0] + list(r.start_logits[1:]), [9.0] + list(r.end_logits[1:])) for r in results]
    ans2, _ = squad.get_answers(ex, feats, res2, version_2_with_negative=True, null_score_diff_threshold=0.0)
    assert ans2["q1"] == "" and ans2["q2"] == ""


def test_get_final_text_alignment():
    assert squad.get_final_text("steve smith", "Steve Smith's", do_lower_case=True) == "Steve Smith"
    assert squad.get_final_text("xyz", "Steve Smith", do_lower_case=True) == "Steve Smith"


def test_run_squad_cli_end_to_end_cpu(squad_files, tmp_path):
    from bert_pytorch_b200 import finetune_squad
    f, vf = squad_files
    cfg = {"vocab_size": len(VOCAB), "hidden_size": 16, "num_hidden_layers": 1, "num_attention_heads": 2,
           "intermediate_size": 32, "max_position_embeddings": 64, "vocab_file": vf, "tokenizer": "wordpiece",
           "next_sentence": True}
    cj = tmp_path / "model.json"; cj.write_text(json.dumps(cfg))
    m = M.BertForPreTraining(BertConfig.from_dict(dict(cfg)).pad_vocab(8))
    ck = tmp_path / "ckpt_1.pt"; torch.save({"model": m.state_dict()}, ck)
    out = tmp_path / "out"
    summary = finetune_squad.main(["--bert_model", "tiny", "--output_dir", str(out), "--init_checkpoint", str(ck),
                                   "--config_file", str(cj), "--train_file", f, "--predict_file", f, "--do_train",
                                   "--do_predict", "--do_eval", "--do_lower_case", "--train_batch_size", "2",
                                   "--num_train_epochs", "1", "--max_seq_length", "48", "--doc_stride", "16",
                                   "--max_query_length", "12", "--no_cuda", "--disable-progress-bar", "--skip_cache",
                                   "--eval_script", "/nonexistent"])
    for name in ("pytorch_model.bin", "bert_config.json", "predictions.json", "nbest_predictions.json", "squad_log.json"):
        assert (out / name).exists(), name
    assert set(json.load(open(out / "predictions.json"))) == {"q1", "q2", "q3"}
    for k in ("e2e_train_time", "training_sequences_per_second", "final_loss", "e2e_inference_time",
              "inference_sequences_per_second", "exact_match", "F1"):
        assert k in summary
    assert "model" in torch.load(out / "pytorch_model.bin", weights_only=False)


# ---------------------------------------------------------------------------------------------- NER
def test_ner_dataset_and_cli(tmp_path, squad_files):
    _, vf = squad_files
    conll = tmp_path / "train.txt"
    conll.write_text("-DOCSTART- -X- -X- O\n\nWilliam NNP B-NP B-PER\nShakespeare NNP I-NP I-PER\nwrote VBD B-VP O\nHamlet NNP B-NP B-MISC\n. . O O\n\n"
                     "Paris NNP B-NP B-LOC\nis VBZ B-VP O\nbig JJ B-ADJP O\n\n")
    tok = get_wordpiece_tokenizer(vf)
    ds = ner.NERDataset(str(conll), tok, ["O", "B-PER", "I-PER", "B-LOC", "B-MISC"], 12)
    assert len(ds) == 2
    ids, labels, mask = ds[0]
    assert ids.shape == (12,) and labels[0] == -100 and labels[1] == 2 and labels[2] == 3 and mask.sum() == 7
    assert labels[6] == -100 and (labels[7:] == 0).all()
    from bert_pytorch_b200 import finetune_ner
    cfg = {"vocab_size": len(VOCAB), "hidden_size": 16, "num_hidden_layers": 1, "num_attention_heads": 2,
           "intermediate_size": 32, "max_position_embeddings": 32, "vocab_file": vf, "tokenizer": "wordpiece"}
    cj = tmp_path / "m.json"; cj.write_text(json.dumps(cfg))
    ck = tmp_path / "c.pt"
    torch.save({"model": M.BertForPreTraining(BertConfig.from_dict(dict(cfg)).pad_vocab(8)).state_dict()}, ck)
    out = finetune_ner.main(["--train_file", str(conll), "--val_file", str(conll), "--test_file", str(conll), "--labels",
                             "O", "B-PER", "I-PER", "B-LOC", "B-MISC", "--model_config_file", str(cj),
                             "--model_checkpoint", str(ck), "--epochs", "2", "--lr", "0.01", "--batch_size", "2",
                             "--max_seq_len", "12", "--no_cuda"])
    assert set(out) >= {"train_loss", "val_loss", "val_f1", "test_loss", "test_f1"} and 0.0 <= out["test_f1"] <= 1.0
    assert finetune_ner.compute_metrics(np.eye(3)[None, [1, 2, 1]], np.array([[1, 2, 0]]), {1: "a", 2: "b"}) == 1.0


# ---------------------------------------------------------------------------------------------- corpus tooling
def test_encode_pipeline_and_corpus_tools(tmp_path, squad_files):
    _, vf = squad_files
    txt = tmp_path / "formatted" / "wiki_0.txt"
    txt.parent.mkdir()
    doc = ["the capital of france is paris .", "the river seine flows through paris .", "paris is a big city ."]
    txt.write_text("\n".join(doc) + "\n\n" + "\n".join(doc[::-1]) + "\n\n" + "\n".join(doc) + "\n")
    n = encode.encode_file(str(txt), str(tmp_path / "train_0.hdf5"), vf, "wordpiece", False, 32, 0.5, 0.1, seed=0)
    with hdf5.File(str(tmp_path / "train_0.hdf5"), "r") as f:
        ids, sp, nsl = f["input_ids"][:], f["special_token_positions"][:], f["next_sentence_labels"][:]
    assert ids.shape == (n, 32) and sp.shape == (n, 3) and nsl.dtype == np.int8
    assert (ids[:, 0] == 2).all() and (ids[np.arange(n), sp[:, 1]] == 3).all() and (ids[np.arange(n), sp[:, 2]] == 3).all()
    assert (ids[np.arange(n)[:, None], np.arange(32)[None, :]] * (np.arange(32)[None, :] > sp[:, 2:3]) == 0).all()
    n2 = encode.encode_file(str(txt), str(tmp_path / "train_1.hdf5"), vf, "wordpiece", False, 32, 0.0, 0.0, seed=0)
    with hdf5.File(str(tmp_path / "train_1.hdf5"), "r") as f:
        assert f["special_token_positions"].shape == (n2, 2) and (f["next_sentence_labels"][:] == 0).all()
    assert encode.output_dir_name(False, 128, True) == "sequences_lowercase_max_seq_len_128_next_seq_task_true"
    # sharding / sampling / helpers
    assert corpus.parse_value_as_int("100M") == 100_000_000 and corpus.parse_value_as_int("2.5K") == 2500
    nsh = corpus.shard_text(str(txt), str(tmp_path / "sh" / "shard_{index}.txt"), 80)
    assert nsh >= 2 and sum(len(corpus.file_to_articles(str(tmp_path / "sh" / f"shard_{i}.txt"))) for i in range(1, nsh + 1)) == 3
    corpus.sample_and_shard([str(txt)], str(tmp_path / "sam" / "shard_{index}.txt"), 10 ** 6, 3)
    assert len(corpus.file_to_articles(str(tmp_path / "sam" / "shard_0.txt"))) >= 1
    assert corpus.split_sentences("Dr. Smith went home. He slept! Did he? Yes.") == ["Dr. Smith went home.", "He slept!", "Did he?", "Yes."]
    wiki = tmp_path / "wiki_00"
    wiki.write_text('<doc id="1" url="u" title="T">\nT\nFirst sentence here. Second one.\n</doc>\n<doc id="2">\nU\nOther text.\n</doc>\n')
    corpus.format_files("wikicorpus", [str(wiki)], str(tmp_path / "fmt.txt"))
    assert (tmp_path / "fmt.txt").read_text() == "First sentence here.\nSecond one.\n\nOther text.\n\n"
    vocab = corpus.build_vocab([str(txt)], str(tmp_path / "v.txt"), size=60)
    assert vocab[0] == "[PAD]" and set(vocab[:5]) == {"[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"}
