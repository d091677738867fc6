"""GLUE data, features, metrics and the run_glue.py loop on the CPU: every task's processor against tiny TSVs in the
task's exact column layout, longest-first truncation and the [CLS] a [SEP] b [SEP] layout on a small vocabulary, the
metrics against hand-computed values and scipy, the classifier's dropout stream, and an end-to-end run on a learnable
synthetic task."""
import json
import os

import numpy as np
import pytest
import torch

from bert_pytorch_b200.data import glue as G

FILLER = [f"w{i}" for i in range(40)]
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "good", "bad", "the", "movie", "was", "a", "b", "c",
         "##s"] + FILLER


def _write(path, rows):
    with open(path, "w", encoding="utf-8") as f:
        for r in rows:
            f.write("\t".join(r) + "\n")


# ---------------------------------------------------------------------------------------------------------------------
# processors
# ---------------------------------------------------------------------------------------------------------------------
def _task_dir(tmp_path, name, files):
    d = tmp_path / name
    d.mkdir()
    for fname, rows in files.items():
        _write(d / fname, rows)
    return str(d)


def test_cola_headerless_train_dev_and_headed_test(tmp_path):
    d = _task_dir(tmp_path, "CoLA", {
        "train.tsv": [["gj04", "1", "", "Our friends won't buy this analysis."], ["gj04", "0", "*", "They drank the pub."]],
        "dev.tsv": [["clc95", "1", "", "The sailors rode the breeze."]],
        "test.tsv": [["index", "sentence"], ["0", "Bill whistled past the house."], ["1", "The car honked."]]})
    t = G.get_task("CoLA")
    tr = G.train_examples(t, d)
    assert [(e.text_a, e.text_b, e.label) for e in tr] == [("Our friends won't buy this analysis.", None, "1"),
                                                          ("They drank the pub.", None, "0")]
    (name, dev), = G.dev_sets(t, d)
    assert name == "CoLA" and dev[0].text_a == "The sailors rode the breeze." and dev[0].label == "1"
    (tname, test), = G.test_sets(t, d)
    assert tname == "CoLA" and [(e.guid, e.text_a, e.label) for e in test] == [
        ("0", "Bill whistled past the house.", None), ("1", "The car honked.", None)]
    assert t.metrics == ("mcc",) and t.num_labels == 2


def test_sst2_mrpc_qqp_qnli_rte_wnli_columns(tmp_path):
    cases = {
        "SST-2": ({"train.tsv": [["sentence", "label"], ["a fine film ", "1"]],
                   "test.tsv": [["index", "sentence"], ["7", "dull"]]}, ("a fine film ", None, "1"), ("7", "dull", None)),
        "MRPC": ({"train.tsv": [["Quality", "#1 ID", "#2 ID", "#1 String", "#2 String"], ["1", "11", "12", "He said.", "He stated."]],
                  "test.tsv": [["index", "#1 ID", "#2 ID", "#1 String", "#2 String"], ["3", "1", "2", "x y", "y x"]]},
                 ("He said.", "He stated.", "1"), ("3", "x y", "y x")),
        "QQP": ({"train.tsv": [["id", "qid1", "qid2", "question1", "question2", "is_duplicate"],
                               ["5", "1", "2", "How?", "Why?", "0"], ["6", "broken line"]],
                 "test.tsv": [["id", "question1", "question2"], ["9", "Who?", "What?"]]}, ("How?", "Why?", "0"),
                ("9", "Who?", "What?")),
        "QNLI": ({"train.tsv": [["index", "question", "sentence", "label"], ["0", "Q?", "S.", "not_entailment"]],
                  "test.tsv": [["index", "question", "sentence"], ["4", "Q2?", "S2."]]}, ("Q?", "S.", "not_entailment"),
                 ("4", "Q2?", "S2.")),
        "RTE": ({"train.tsv": [["index", "sentence1", "sentence2", "label"], ["0", "P.", "H.", "entailment"]],
                 "test.tsv": [["index", "sentence1", "sentence2"], ["2", "P2.", "H2."]]}, ("P.", "H.", "entailment"),
                ("2", "P2.", "H2.")),
        "WNLI": ({"train.tsv": [["index", "sentence1", "sentence2", "label"], ["0", "A.", "B.", "1"]],
                  "test.tsv": [["index", "sentence1", "sentence2"], ["8", "C.", "D."]]}, ("A.", "B.", "1"), ("8", "C.", "D.")),
    }
    for name, (files, train, test) in cases.items():
        files = dict(files)
        files["dev.tsv"] = files["train.tsv"]
        d = _task_dir(tmp_path, name, files)
        t = G.get_task(name)
        tr = G.train_examples(t, d)
        assert len(tr) == 1, name                                   # QQP's short line is skipped
        assert (tr[0].text_a, tr[0].text_b, tr[0].label) == train, name
        (_, te), = G.test_sets(t, d)
        assert (te[0].guid, te[0].text_a, te[0].text_b if te[0].text_b is not None else te[0].label) == test \
            or (te[0].guid, te[0].text_a, te[0].label) == test, name
        assert te[0].label is None
    assert G.get_task("mrpc").metrics == ("acc", "f1") and G.get_task("qqp").metrics == ("acc", "f1")


def test_mnli_matched_and_mismatched(tmp_path):
    head = ["index", "promptID", "pairID", "genre", "s1b", "s2b", "s1p", "s2p", "sentence1", "sentence2"]
    row = lambda i, a, b, *lab: [str(i), "p", "q", "g", "x", "x", "x", "x", a, b, *lab]   # noqa: E731
    d = _task_dir(tmp_path, "MNLI", {
        "train.tsv": [head + ["label1", "gold_label"], row(0, "A", "B", "neutral", "neutral")],
        "dev_matched.tsv": [head + ["label1", "label2", "label3", "label4", "label5", "gold_label"],
                            row(1, "Cm", "Dm", "neutral", "entailment", "x", "x", "x", "entailment")],
        "dev_mismatched.tsv": [head + ["label1", "label2", "label3", "label4", "label5", "gold_label"],
                               row(2, "Cmm", "Dmm", "x", "x", "x", "x", "x", "contradiction")],
        "test_matched.tsv": [head, row(10, "Tm", "Um")],
        "test_mismatched.tsv": [head, row(20, "Tmm", "Umm")]})
    t = G.get_task("MNLI")
    assert t.num_labels == 3
    assert [(e.text_a, e.text_b, e.label) for e in G.train_examples(t, d)] == [("A", "B", "neutral")]
    dev = G.dev_sets(t, d)
    assert [n for n, _ in dev] == ["MNLI-m", "MNLI-mm"]
    assert (dev[0][1][0].text_a, dev[0][1][0].label) == ("Cm", "entailment")
    assert (dev[1][1][0].text_b, dev[1][1][0].label) == ("Dmm", "contradiction")
    test = G.test_sets(t, d)
    assert [(n, ex[0].guid, ex[0].text_a, ex[0].text_b) for n, ex in test] == [("MNLI-m", "10", "Tm", "Um"),
                                                                             ("MNLI-mm", "20", "Tmm", "Umm")]


def test_unknown_tasks_labels_and_stsb_are_refused(tmp_path):
    with pytest.raises(ValueError, match="regression"):
        G.get_task("STS-B")
    with pytest.raises(ValueError, match="unknown GLUE task"):
        G.get_task("squad")
    d = _task_dir(tmp_path, "SST-2", {"train.tsv": [["sentence", "label"], ["x", "2"]]})
    with pytest.raises(ValueError, match="label '2'"):
        G.train_examples(G.get_task("sst-2"), d)


# ---------------------------------------------------------------------------------------------------------------------
# features
# ---------------------------------------------------------------------------------------------------------------------
def test_longest_first_truncation():
    a, b = [1, 2, 3, 4, 5], [6, 7]
    G.truncate_pair(a, b, 5)
    assert (a, b) == ([1, 2, 3], [6, 7])
    a, b = [1, 2, 3], [4, 5, 6]                                       # a tie takes from b first
    G.truncate_pair(a, b, 4)
    assert (a, b) == ([1, 2], [4, 5])
    a, b = [1, 2, 3], [4, 5, 6, 7, 8, 9]
    G.truncate_pair(a, b, 5)
    assert (a, b) == ([1, 2, 3], [4, 5])
    a = [1, 2, 3]
    G.truncate_pair(a, None, 2)
    assert a == [1, 2]


def test_features_special_tokens_segments_and_padding():
    ids, seg, mask = G.features([[10, 11], [10, 11, 12, 13, 14]], [[20], None], 7, cls_id=2, sep_id=3)
    assert ids.tolist() == [[2, 10, 11, 3, 20, 3, 0], [2, 10, 11, 12, 13, 14, 3]]
    assert seg.tolist() == [[0, 0, 0, 0, 1, 1, 0], [0] * 7]
    assert mask.tolist() == [[1, 1, 1, 1, 1, 1, 0], [1] * 7]
    ids, seg, mask = G.features([[10, 11, 12, 13]], [[20, 21, 22]], 8, cls_id=2, sep_id=3)   # 7 tokens into 5
    assert ids.tolist() == [[2, 10, 11, 12, 3, 20, 21, 3]] and seg.tolist() == [[0, 0, 0, 0, 0, 1, 1, 1]]


def test_featurizer_with_the_repo_tokenizer(tmp_path):
    vf = tmp_path / "vocab.txt"
    vf.write_text("\n".join(VOCAB) + "\n")
    fz = G.Featurizer(str(vf), do_lower_case=True, max_seq_length=10)
    t = G.get_task("mrpc")
    ids, seg, mask, labels = fz(t, [G.Example("x", "The movie was GOOD", "bads", "1"),
                                    G.Example("y", "zzz", "a", "0")])
    v = {w: i for i, w in enumerate(VOCAB)}
    assert ids[0].tolist() == [2, v["the"], v["movie"], v["was"], v["good"], 3, v["bad"], v["##s"], 3, 0]
    assert seg[0].tolist() == [0] * 6 + [1] * 3 + [0]
    assert ids[1].tolist()[:5] == [2, v["[UNK]"], 3, v["a"], 3] and mask[1].sum() == 5
    assert labels.tolist() == [1, 0]


def test_fill_batch_adds_inert_rows():
    ids = torch.arange(6).view(2, 3) + 5
    seg, mask, lab = torch.zeros_like(ids), torch.ones_like(ids), torch.tensor([1, 0])
    i2, s2, m2, l2 = G.fill_batch(ids, seg, mask, lab, 4)
    assert i2.shape == (4, 3) and torch.equal(i2[:2], ids) and (i2[2:] == 0).all()
    assert m2[2:].tolist() == [[1, 0, 0], [1, 0, 0]] and l2.tolist() == [1, 0, -1, -1] and (s2[2:] == 0).all()
    assert G.fill_batch(ids, seg, mask, lab, 2)[0] is ids


# ---------------------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------------------
def test_metrics_against_hand_values_and_scipy():
    from scipy import stats
    pred = np.array([1, 1, 0, 0, 1, 0, 1, 1])
    lab = np.array([1, 0, 0, 1, 1, 0, 1, 0])
    tp, tn, fp, fn = 3, 2, 2, 1
    assert G.accuracy(pred, lab) == 5 / 8
    assert G.f1_positive(pred, lab) == pytest.approx(2 * tp / (2 * tp + fp + fn))
    mcc = (tp * tn - fp * fn) / np.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn))
    assert G.matthews_corr(pred, lab) == pytest.approx(mcc)
    # for 0/1 variables the MCC is the Pearson correlation (the phi coefficient)
    assert G.matthews_corr(pred, lab) == pytest.approx(stats.pearsonr(pred, lab)[0])
    assert G.matthews_corr(1 - pred, lab) == pytest.approx(-mcc)
    # degenerate: one class predicted throughout, or one class in the labels -> 0, not NaN
    assert G.matthews_corr(np.ones(8, int), lab) == 0.0
    assert G.matthews_corr(pred, np.zeros(8, int)) == 0.0
    assert G.f1_positive(np.zeros(4, int), np.zeros(4, int)) == 0.0
    m = G.compute_metrics(G.get_task("mrpc"), pred, lab)
    assert m["acc"] == 5 / 8 and m["acc_and_f1"] == pytest.approx((5 / 8 + 2 * tp / (2 * tp + fp + fn)) / 2)
    assert set(G.compute_metrics(G.get_task("cola"), pred, lab)) == {"mcc"}
    assert set(G.compute_metrics(G.get_task("mnli"), pred, lab)) == {"acc"}


def test_submission_file(tmp_path):
    t = G.get_task("rte")
    ex = [G.Example("4", "a", "b", None), G.Example("9", "c", "d", None)]
    G.write_submission(t, tmp_path / "RTE.tsv", ex, np.array([1, 0]))
    assert (tmp_path / "RTE.tsv").read_text() == "index\tprediction\n4\tnot_entailment\n9\tentailment\n"


def test_classifier_dropout_stream_collides_with_no_encoder_or_embedding_stream():
    from bert_pytorch_b200.models import fused as F
    used = {F._stream(F._EMB_LAYER, F.SITE_EMB)}
    for layer in range(F._EMB_LAYER):
        used |= {F._stream(layer, s) for s in (F.SITE_ATTN_PROB, F.SITE_ATTN_OUT, F.SITE_FFN_OUT)}
    assert F.CLS_STREAM not in used and F.CLS_STREAM < 2 ** 32


# ---------------------------------------------------------------------------------------------------------------------
# run_glue.py end to end
# ---------------------------------------------------------------------------------------------------------------------
def write_synthetic_sst2(d, n_train, n_dev, n_test, seed=0, max_words=12):
    """An SST-2-layout task that a small model learns: label 1 iff the sentence holds "good" rather than "bad" (one of
    the two at a random place among filler words).  Returns the dev labels."""
    rng = np.random.default_rng(seed)

    def sent():
        k = int(rng.integers(2, max_words + 1))
        words = list(rng.choice(FILLER, k))
        y = int(rng.integers(0, 2))
        words.insert(int(rng.integers(0, k + 1)), "good" if y else "bad")
        return " ".join(words), y
    os.makedirs(d, exist_ok=True)
    tr = [sent() for _ in range(n_train)]
    dv = [sent() for _ in range(n_dev)]
    te = [sent() for _ in range(n_test)]
    _write(os.path.join(d, "train.tsv"), [["sentence", "label"]] + [[s, str(y)] for s, y in tr])
    _write(os.path.join(d, "dev.tsv"), [["sentence", "label"]] + [[s, str(y)] for s, y in dv])
    _write(os.path.join(d, "test.tsv"), [["index", "sentence"]] + [[str(i), s] for i, (s, _) in enumerate(te)])
    return [y for _, y in dv]


def _config_file(tmp_path, vf, **kw):
    cfg = {"vocab_size": len(VOCAB), "hidden_size": 32, "num_hidden_layers": 1, "num_attention_heads": 2,
           "intermediate_size": 64, "max_position_embeddings": 64, "vocab_file": str(vf), "next_sentence": True,
           "hidden_dropout_prob": 0.0, "attention_probs_dropout_prob": 0.0}
    cfg.update(kw)
    cj = tmp_path / "model.json"
    cj.write_text(json.dumps(cfg))
    return cj


def test_run_glue_end_to_end_cpu(tmp_path, monkeypatch):
    from bert_pytorch_b200 import finetune_glue
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    vf = tmp_path / "vocab.txt"
    vf.write_text("\n".join(VOCAB) + "\n")
    data = tmp_path / "SST-2"
    write_synthetic_sst2(str(data), 256, 64, 21)
    cj = _config_file(tmp_path, vf)
    out = tmp_path / "out"
    summary = finetune_glue.main(["--task_name", "SST-2", "--data_dir", str(data), "--config_file", str(cj),
                                  "--output_dir", str(out), "--do_train", "--do_eval", "--do_predict",
                                  "--do_lower_case", "--max_seq_length", "32", "--train_batch_size", "16",
                                  "--eval_batch_size", "16", "--learning_rate", "1e-3", "--num_train_epochs", "10",
                                  "--warmup_proportion", "0.1"])
    res = json.load(open(out / "eval_results.json"))
    assert set(res) == {"SST-2"} and res["SST-2"]["eval_samples"] == 64
    assert res["SST-2"]["acc"] > 0.75, res                            # chance is 0.5
    lines = (out / "SST-2.tsv").read_text().splitlines()
    assert lines[0] == "index\tprediction" and len(lines) == 22
    assert [ln.split("\t")[0] for ln in lines[1:]] == [str(i) for i in range(21)]
    assert all(ln.split("\t")[1] in ("0", "1") for ln in lines[1:])
    for name in ("pytorch_model.bin", "bert_config.json", "glue_log.json"):
        assert (out / name).exists(), name
    assert summary["final_loss"] == summary["final_loss"]
