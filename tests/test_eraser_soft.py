"""CPU: the ERASER soft-token scores and tokens to flip: the oracle (``oracle/eraser_soft.py``) and the host side of
``eraser.py`` against ``tests/golden/eraser_soft.npz`` (the reference's ``score_soft_tokens`` on the tiny-BERT word scores,
and tokens to flip by one reference forward per selection size), the restated curves against sklearn on random documents,
and the reference's ``metrics.py`` ``main`` on the written result files."""
import json
import math
import os
import sys
import warnings

import numpy as np
import pytest

from oracle import eraser_soft as osoft
from transformer_explainability_b200 import eraser as te

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser_soft.npz")
METHODS = te.METHODS


def load():
    import test_eraser as ce
    g, docids, docs, anns = ce.load()
    return np.load(GOLDEN), g, docids, docs, anns


def _close(a, b, tol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return bool(np.all((np.isnan(a) & np.isnan(b)) | (np.abs(a - b) <= tol)))


def _doc_truth(anns, docs, ranges, i):
    """(soft prediction truth vector, W, n_words, spans) of annotation i, keyed by (annotation id, docid)."""
    a = anns[i]
    d = te.annotation_docid(a)
    spans = te.TruthIndex(anns).spans_by_key.get((a.annotation_id, d), [])
    n = len(docs[d].split())
    return osoft.truth_vector(spans, n), len(ranges[d]), n, spans


@pytest.mark.parametrize("method", METHODS)
def test_oracle_reproduces_the_fixture(method):
    z, g, docids, docs, anns = load()
    dd = [te.annotation_docid(a) for a in anns]
    ranges = {d: te.word_piece_ranges(docs[d].split(), [str(p) for p in g["pieces." + d]]) for d in docids}
    words = [g["%s.words.%s" % (method, d)] for d in dd]
    n_words = [len(docs[d].split()) for d in dd]
    assert te.soft_lines(anns, dd, words, n_words) == [str(l) for l in z["%s.soft_lines" % method]]
    ref = json.loads(str(z["%s.soft_scores" % method]))
    per_doc, single = [], []
    try:
        for i in range(len(anns)):
            truth, W, n, spans = _doc_truth(anns, docs, ranges, i)
            assert te.soft_truth(te.TruthIndex(anns), anns[i], dd[i], W, n)[1] == osoft.tail_counts(spans, W, n)
            per_doc.append(osoft.soft_scores(osoft.soft_prediction(words[i], n), truth))
            single.append(len(set(truth)) < 2)
    except ValueError:
        assert method == "attn_gradcam" and "NaN" in ref["error"]               # the reference's maps are NaN there
        return
    assert _close(per_doc, z["%s.soft_doc" % method], 1e-12), method
    assert single == z["%s.single" % method].tolist()
    for got in (osoft.score_soft_tokens(per_doc, single), te.soft_token_scores(per_doc, single)):
        assert got.keys() == ref.keys() and all(abs(got[k] - ref[k]) <= 1e-12 for k in ref), (method, got, ref)
    # tokens to flip: the brute-force search, with the reference's recorded row margins as the classifier
    for tag in ("", "_shift"):
        flips, fl = [], []
        for i, d in enumerate(dd):
            ids = [int(x) for x in g["ids." + d]]
            margin = {}
            for k in range(1, len(words[i]) + 1):
                from oracle.eraser_faithfulness import reduce_rows
                margin[tuple(reduce_rows(ids, ranges[d], words[i], k)[0])] = z["%s.margins%s" % (method, tag)][i, k - 1]
            k, f = osoft.tokens_to_flip(lambda row: int(margin[tuple(row)] < 0), ids, ranges[d], words[i], n_words[i], 0)
            flips.append(k)
            fl.append(f)
        assert flips == z["%s.flip%s" % (method, tag)].tolist(), (method, tag)
        assert fl == z["%s.flipped%s" % (method, tag)].tolist()
        fs = te.flip_scores(anns, dd, n_words, flips, fl)
        assert fs["tokens_to_flip"] == float(z["%s.flip_fraction%s" % (method, tag)])
        assert fs["never_flipped"] == len(fl) - sum(fl)


def _random_doc(g, kind):
    """(W fp32 word scores, n_words, spans) of one random document of the given kind."""
    W = 1 if kind == "w1" else int(g.integers(1, 60))
    tail = int(g.integers(0, 40)) if kind in ("tail", "zeros", "signed_zero") else 0
    n = W + tail
    if kind == "ties":
        s = g.integers(0, 4, W).astype(np.float32) / 2
    elif kind == "zeros":
        s = np.zeros(W, dtype=np.float32)
    elif kind == "signed_zero":
        s = np.where(g.random(W) < 0.5, np.float32(-0.0), np.float32(0.0)) + \
            (g.random(W) < 0.3) * g.integers(1, 3, W).astype(np.float32)
    else:
        s = g.random(W).astype(np.float32)
    if kind == "single_pos":
        spans = [(0, n)]
    elif kind == "single_neg":
        spans = []
    else:
        spans = [(int(a), int(min(n, a + g.integers(1, 5)))) for a in g.integers(0, n, int(g.integers(1, 4)))]
    return s.astype(np.float32), n, spans


@pytest.mark.parametrize("seed", range(4))
def test_restatement_matches_sklearn(seed):
    skm = pytest.importorskip("sklearn.metrics")
    g = np.random.default_rng(seed)
    kinds = ["random", "ties", "zeros", "tail", "w1", "single_pos", "single_neg", "signed_zero"]
    per_doc, single = [], []
    for rep in range(30):
        s, n, spans = _random_doc(g, kinds[rep % len(kinds)])
        pred = osoft.soft_prediction(s, n)
        truth = [int(t) for t in osoft.truth_vector(spans, n)]
        got = osoft.soft_scores(pred, truth)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            p, r, _ = skm.precision_recall_curve(truth, pred)
            want = [skm.auc(r, p), skm.average_precision_score(truth, pred)]
            try:
                want.append(skm.roc_auc_score(truth, pred))
            except ValueError:                                 # older sklearn raises for one class
                want.append(math.nan)
        assert _close(got, want, 1e-12), (rep, got, want)
        per_doc.append(got)
        single.append(len(set(truth)) < 2)
    assert any(single) and not all(single)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = {"auprc": np.average([x[0] for x in per_doc]),
               "average_precision": np.average([x[1] for x, s in zip(per_doc, single) if not s]),
               "roc_auc_score": np.average([x[2] for x, s in zip(per_doc, single) if not s])}
    assert te.soft_token_scores(per_doc, single) == ref == osoft.score_soft_tokens(per_doc, single)


def test_tail_and_signed_zero_groups():
    # the tail joins the group of score 0 (either sign); a tail after positive scores is its own last group
    assert osoft.curve([0.5, -0.0, 0.0, 0.0], [1, 0, 1, 0]) == [(1, 0), (2, 2)]
    assert osoft.curve([0.5, 0.25, 0.0], [0, 1, 1]) == [(0, 1), (1, 1), (2, 1)]
    assert osoft.tail_counts([(1, 3), (4, 9)], 5, 7) == (2, 0)
    assert osoft.tail_counts([(0, 2)], 5, 8) == (0, 3)
    with pytest.raises(ValueError):
        osoft.curve([float("nan"), 1.0], [0, 1])
    a = te.Annotation("x", "", frozenset([(te.Evidence("", "x", 2, 9),)]), "POS")
    with pytest.raises(ValueError):
        te.soft_truth(te.TruthIndex([a]), a, "x", 3, 8)                     # a span past the document's 8 words


def test_reference_metrics_accepts_the_written_results(tmp_path, monkeypatch):
    from oracle import ref_harness as rh
    if not rh.available():
        pytest.skip("reference not present")
    import test_eraser_faithfulness as tf
    z, g, docids, docs, anns = load()
    zf = np.load(tf.GOLDEN)
    m = "transformer_attribution"
    dd = [te.annotation_docid(a) for a in anns]
    ranges = {d: te.word_piece_ranges(docs[d].split(), [str(p) for p in g["pieces." + d]]) for d in docids}
    words = [g["%s.words.%s" % (m, d)] for d in dd]
    n_words = [len(docs[d].split()) for d in dd]
    per_doc = [osoft.soft_scores(osoft.soft_prediction(words[i], n_words[i]), _doc_truth(anns, docs, ranges, i)[0])
               for i in range(len(anns))]
    single = z["%s.single" % m].tolist()
    pred, probs, comp, suff, thr = tf._arrays(zf["%s.lines" % m], tf.CLASSES)
    selected = [[h["start_token"] for h in json.loads(str(l))["rationales"][0]["hard_rationale_predictions"]]
                for l in zf["%s.lines" % m]]
    flips = z["%s.flip_shift" % m]
    aopc = [float(t) for t in zf["aopc_thresholds"]]
    res = {"lines": {}, "scores": {},
           "soft": {"lines": te.soft_lines(anns, dd, words, n_words), "scores": te.soft_token_scores(per_doc, single)},
           "faithfulness": {
               "lines": te.faithfulness_lines(anns, dd, tf.CLASSES, pred, probs, comp, suff, thr, selected, flips),
               "scores": te.classification_scores_from_probs(anns, tf.CLASSES, pred, probs, comp, suff, thr, aopc),
               "flip_scores": te.flip_scores(anns, dd, n_words, flips, z["%s.flipped_shift" % m])}}
    out = str(tmp_path / "out")
    te.write_results(res, out)
    assert sorted(os.listdir(out)) == ["faithfulness_results.jsonl", "faithfulness_scores.json", "soft_results.jsonl",
                                       "soft_scores.json", "tokens_to_flip.json"]
    # metrics.py pairs soft predictions with its flattened documents: a data directory whose docs.jsonl holds each
    # document as sentences of words flattens to the word lists (raw-text documents flatten to characters)
    data = str(tmp_path / "data")
    os.makedirs(data)
    with open(os.path.join(data, "docs.jsonl"), "w") as f:
        f.write("".join(json.dumps({"docid": d, "document": [docs[d].split()]}) + "\n" for d in docids))
    with open(os.path.join(data, "test.jsonl"), "w") as f:
        f.write("".join(str(l) + "\n" for l in g["annotations"]))
    rh._prepare_bert_imports()
    got = {}
    with rh._ref_imports():
        from BERT_rationale_benchmark import metrics as rmetrics
        for name in ("soft_results.jsonl", "faithfulness_results.jsonl"):
            score_file = str(tmp_path / (name + ".scores.json"))
            monkeypatch.setattr(sys, "argv", ["metrics.py", "--data_dir", data, "--split", "test", "--results",
                                              os.path.join(out, name), "--score_file", score_file])
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                rmetrics.main()
            with open(score_file) as f:
                got[name] = json.load(f)
    with open(os.path.join(out, "soft_scores.json")) as f:
        mine = json.load(f)
    ref = got["soft_results.jsonl"]["token_soft_metrics"]
    assert ref.keys() == mine.keys() and all(abs(ref[k] - mine[k]) <= 1e-12 for k in ref), (ref, mine)
    with open(os.path.join(out, "faithfulness_scores.json")) as f:
        assert got["faithfulness_results.jsonl"]["classification_scores"] == json.load(f)
    with open(os.path.join(out, "tokens_to_flip.json")) as f:
        t = json.load(f)
    assert t["tokens_to_flip"] == float(z["%s.flip_fraction_shift" % m]) and t["never_flipped"] == 0
    assert [x["tokens_to_flip"] for x in t["documents"]] == flips.tolist()


def test_cli_parsing():
    base = ["--data_dir", "d", "--output_dir", "o", "--model_params", "p"]
    a = te.parse_args(base)
    assert not a.soft_scores and not a.tokens_to_flip
    a = te.parse_args(base + ["--soft-scores", "--faithfulness", "--tokens-to-flip"])
    assert a.soft_scores and a.tokens_to_flip and a.faithfulness
    with pytest.raises(SystemExit):
        te.parse_args(base + ["--tokens-to-flip"])
    with pytest.raises(ValueError):
        te.eraser_eval(None, {}, [], {}, {}, tokens_to_flip=True)
    with pytest.raises(ValueError):
        te.eraser_eval(None, {}, [], {}, {}, faithfulness=True, tokens_to_flip=True, flip_chunk=65)


def test_flags_off_write_todays_files(tmp_path):
    import test_eraser_faithfulness as tf
    zf = np.load(tf.GOLDEN)
    _, g, docids, docs, anns = load()
    dd = [te.annotation_docid(a) for a in anns]
    m = "transformer_attribution"
    pred, probs, comp, suff, thr = tf._arrays(zf["%s.lines" % m], tf.CLASSES)
    selected = [[h["start_token"] for h in json.loads(str(l))["rationales"][0]["hard_rationale_predictions"]]
                for l in zf["%s.lines" % m]]
    lines = te.faithfulness_lines(anns, dd, tf.CLASSES, pred, probs, comp, suff, thr, selected)
    assert lines == [str(l) for l in zf["%s.lines" % m]]
    res = {"lines": {5: ["a"]}, "scores": {5: {"x": 1}}, "faithfulness": {"lines": lines, "scores": {"y": 2}}}
    te.write_results(res, str(tmp_path))
    assert sorted(os.listdir(str(tmp_path))) == ["faithfulness_results.jsonl", "faithfulness_scores.json",
                                                 "identifier_results_5.json", "scores_5.json"]
    with open(os.path.join(str(tmp_path), "faithfulness_results.jsonl")) as f:
        assert f.read() == "".join(str(l) + "\n" for l in zf["%s.lines" % m])


def test_fixture_covers_the_cases():
    z = np.load(GOLDEN)
    assert str(z["sklearn"])
    assert (z["n_words"] > z["W"]).any() and (z["n_words"] == z["W"]).any()              # truncated tails, and none
    for m in METHODS:
        assert not z["%s.flipped" % m].any()                                             # never flipped: fraction 1
        assert z["%s.flipped_shift" % m].all() and (z["%s.flip_shift" % m] < z["W"]).any()
