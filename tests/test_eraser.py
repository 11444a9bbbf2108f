"""CPU: the ERASER rationale-evaluation oracle (``oracle/eraser.py``) and the host side of ``eraser.py`` against the reference's
own pooling, top-k lines and ``metrics.py`` scores (``tests/golden/eraser.npz``), plus the reader, the word map's alignment
errors and the command line.

The metric dicts average over Python sets of string keys, so their last bits depend on the interpreter's hash seed; the
fixture was written with PYTHONHASHSEED=0, and the score comparisons run in a child interpreter with that seed."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import eraser as oe
from transformer_explainability_b200 import eraser as te

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser.npz")
METHODS = ("transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout")


def load():
    g = np.load(GOLDEN)
    docids = [str(d) for d in g["docids"]]
    docs = {d: str(t) for d, t in zip(docids, g["docs"])}
    anns = []
    for line in g["annotations"]:
        content = json.loads(str(line))
        content["evidences"] = frozenset(tuple(te.Evidence(**ev) for ev in grp) for grp in content["evidences"])
        anns.append(te.Annotation(**content))
    return g, docids, docs, anns


@pytest.fixture(scope="module")
def golden():
    return load()


def _bits(a):
    """fp32 bit patterns, every NaN as one pattern (its sign is not part of the result)."""
    a = np.array(a, dtype=np.float32)
    a[np.isnan(a)] = np.float32("nan")
    return a.view(np.int32)


@pytest.mark.parametrize("method", METHODS)
def test_oracle_pooling_bit_equal_to_reference(golden, method):
    g, docids, docs, _ = golden
    for d in docids:
        cam = np.maximum(g["%s.map.%s" % (method, d)], np.float32(0))
        cam = np.where(np.isnan(g["%s.map.%s" % (method, d)]), np.float32("nan"), cam)
        pooled = oe.pool_words(docs[d].split(), [str(p) for p in g["pieces." + d]], list(cam))
        assert np.array_equal(_bits(pooled), _bits(g["%s.words.%s" % (method, d)])), (method, d)


@pytest.mark.parametrize("method", METHODS)
def test_word_piece_ranges_pool_like_the_reference(golden, method):
    """max over each word's piece range of the clamped map == the reference's per-character pooling."""
    g, docids, docs, _ = golden
    for d in docids:
        ranges = te.word_piece_ranges(docs[d].split(), [str(p) for p in g["pieces." + d]])
        m = g["%s.map.%s" % (method, d)]
        ref = g["%s.words.%s" % (method, d)]
        assert len(ranges) == len(ref)
        for (a, b), r in zip(ranges, ref):
            v = m[a:b + 1]
            got = np.float32("nan") if np.isnan(v).any() else np.max(np.maximum(v, np.float32(0)))
            assert _bits(got) == _bits(r)


@pytest.mark.parametrize("method", METHODS)
def test_oracle_order_is_the_reference_topk_on_distinct_scores(golden, method):
    g, docids, _, _ = golden
    checked = 0
    for i, d in enumerate(docids):
        w = g["%s.words.%s" % (method, d)]
        order = oe.word_order(w)
        lines = [json.loads(str(g["%s.lines.%d" % (method, k)][i])) for k in g["ks"]]
        prev = 0
        for k, line in zip(g["ks"], lines):
            hard = line["rationales"][0]["hard_rationale_predictions"]
            n = min(int(k), len(w))
            got = [h["start_token"] for h in hard[prev:prev + n]]
            prev += n
            if len(set(w[~np.isnan(w)].tolist())) == len(w):           # distinct scores: the two orders agree
                assert got == order[:n].tolist(), (method, d, k)
                checked += 1
    assert method in ("attn_gradcam",) or checked > 0


def _child(fn):
    """Run ``fn`` of this module in a child interpreter with PYTHONHASHSEED=0 and return its JSON result."""
    if os.environ.get("PYTHONHASHSEED") == "0":
        return json.loads(json.dumps(globals()[fn]()))
    code = "import sys, json; sys.path[:0] = [%r, %r]; import test_eraser as t; print(json.dumps(t.%s()))" % (
        HERE, os.path.dirname(HERE), fn)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PYTHONHASHSEED="0"), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def oracle_scores():
    g, _, _, anns = load()
    return {"%s.%d" % (m, k): oe.hard_scores(anns, [str(l) for l in g["%s.lines.%d" % (m, k)]], list(g["thresholds"]))
            for m in METHODS for k in g["ks"]}


def host_scores():
    """``eraser.hard_scores`` fed the counts of the reference's own lines (the distinct words of each line, in order of
    first appearance)."""
    g, docids, _, anns = load()
    truth = te.TruthIndex(anns)
    thr = [float(t) for t in g["thresholds"]]
    out = {}
    for m in METHODS:
        for k in g["ks"]:
            orders, counts = [], []
            for d, line in zip(docids, g["%s.lines.%d" % (m, k)]):
                words = list(dict.fromkeys(h["start_token"] for h in json.loads(str(line))["rationales"][0]
                                           ["hard_rationale_predictions"]))
                orders.append(words)
                counts.append(oe.doc_counts(words, truth.spans_by_key.get((d, d), []), [len(words)], thr)[0])
            out["%s.%d" % (m, k)] = te.hard_scores(truth, docids, counts, orders, thr)
    return out


def test_oracle_scores_equal_the_reference_metrics(golden):
    g = golden[0]
    assert str(g["hashseed"]) == "0"
    got = _child("oracle_scores")
    for m in METHODS:
        for k in g["ks"]:
            assert got["%s.%d" % (m, k)] == json.loads(str(g["%s.scores.%d" % (m, k)])), (m, k)


def test_host_scores_from_counts_equal_the_reference_metrics(golden):
    g = golden[0]
    got = _child("host_scores")
    for m in METHODS:
        for k in g["ks"]:
            assert got["%s.%d" % (m, k)] == json.loads(str(g["%s.scores.%d" % (m, k)])), (m, k)


def test_fixture_covers_the_cases(golden):
    g, docids, docs, anns = golden
    truth = te.TruthIndex(anns)
    w = [len(g["transformer_attribution.words." + d]) for d in docids]
    assert min(w) < 5 and max(w) > 5                                     # k below and above W
    assert any(len(docs[d].split()) > n for d, n in zip(docids, w))       # truncated documents
    assert any(a.annotation_id != te.annotation_docid(a) for a in anns)  # a truth key without predictions
    spans = {d: truth.spans_by_key.get((d, d), []) for d in docids}
    assert any(e - s == 1 for v in spans.values() for s, e in v)                      # single words
    assert any(s >= n for d, n in zip(docids, w) for s, _ in spans[d])                 # evidence past the truncation
    assert any(s1 < e0 and s0 < e1 and (s0, e0) != (s1, e1) for v in spans.values() for s0, e0 in v for s1, e1 in v)
    assert any(np.isnan(g["attn_gradcam.words." + d]).any() for d in docids)


def test_doc_counts_match_sets():
    spans = [(0, 3), (2, 3), (5, 6), (7, 7)]
    c = oe.doc_counts([2, 5, 6, 0, 1], spans, [1, 2, 10], [0.5, 0.25, 1.0, 0.0])
    assert c.tolist() == [[1, 1, 1, 1, 1, 1, 1], [2, 2, 2, 2, 2, 2, 2], [5, 4, 2, 2, 4, 2, 5]]


def test_word_piece_ranges_alignment():
    assert te.word_piece_ranges(["ab", "c.", "de"], ["[CLS]", "a", "##b", "c", ".", "d", "##e", "[SEP]"]) == \
        [(1, 2), (3, 4), (5, 6)]
    # truncated: the last word is cut, and words past the stream are dropped
    assert te.word_piece_ranges(["ab", "cd", "ef"], ["[CLS]", "ab", "c", "[SEP]"]) == [(1, 1), (2, 2)]
    # pieces that straddle two words: both words see the piece
    assert te.word_piece_ranges(["ab", "cd"], ["[CLS]", "abc", "##d", "[SEP]"]) == [(1, 1), (1, 2)]
    with pytest.raises(ValueError, match="align"):
        te.word_piece_ranges(["ab", "☃", "cd"], ["[CLS]", "ab", "[UNK]", "cd", "[SEP]"])
    with pytest.raises(ValueError, match="align"):
        te.word_piece_ranges(["ab", "xy", "cd"], ["[CLS]", "ab", "cd", "xy", "[SEP]"])
    # an [UNK] in the last word is what the reference lets through
    assert te.word_piece_ranges(["ab", "c☃"], ["[CLS]", "ab", "[UNK]", "[SEP]"]) == [(1, 1)]


def test_encode_documents_with_any_tokenizer():
    class Tok:
        def __call__(self, text, add_special_tokens, max_length, truncation, padding, return_attention_mask):
            assert add_special_tokens and truncation and not padding
            ids = [2] + [10 + len(w) for w in text.split()][:max_length - 2] + [3]
            return {"input_ids": ids}

        def convert_ids_to_tokens(self, ids):
            return ["t%d" % i for i in ids]
    enc = te.encode_documents({"a": "x yy zzz"}, Tok(), 4)
    assert enc == {"a": ([2, 11, 12, 3], ["t2", "t11", "t12", "t3"])}


def _write_split(tmp, jsonl_docs):
    ann = {"annotation_id": "d1", "query": "q", "classification": "POS", "query_type": None,
           "evidences": [[{"text": "b", "docid": "d1", "start_token": 1, "end_token": 2, "start_sentence": -1,
                           "end_sentence": -1}], [{"text": "a b", "docid": "d1", "start_token": 0, "end_token": 2}]]}
    with open(os.path.join(tmp, "test.jsonl"), "w") as f:
        f.write(json.dumps(ann) + "\n")
    if jsonl_docs:
        with open(os.path.join(tmp, "docs.jsonl"), "w") as f:
            f.write(json.dumps({"docid": "d1", "document": "a b\nc\n"}) + "\n")
    else:
        os.makedirs(os.path.join(tmp, "docs"))
        with open(os.path.join(tmp, "docs", "d1"), "w") as f:
            f.write("a b\nc\n")


@pytest.mark.parametrize("jsonl_docs", [False, True])
def test_reader(tmp_path, jsonl_docs):
    _write_split(str(tmp_path), jsonl_docs)
    anns = te.load_split(str(tmp_path), "test")
    assert len(anns) == 1 and anns[0].classification == "POS"
    assert te.annotation_docid(anns[0]) == "d1"
    assert sorted(te.truth_rationales(anns)) == [("d1", "d1", 0, 2), ("d1", "d1", 1, 2)]
    assert te.load_documents(str(tmp_path), {"d1"}) == {"d1": "a b\nc\n"}
    truth = te.TruthIndex(anns)
    assert truth.spans_by_key == {("d1", "d1"): [(0, 2), (1, 2)]} and truth.n_tokens == 2 and truth.n_spans == 2


def test_records_hash_like_the_reference():
    """The metric key sets iterate in the reference's order only if the records hash as the tuple of their fields."""
    ev = te.Evidence("t", "d", 1, 2)
    assert hash(ev) == hash(("t", "d", 1, 2, -1, -1))
    from oracle import ref_harness as rh
    if not rh.available():
        pytest.skip("reference not present")
    with rh._ref_imports():
        from BERT_rationale_benchmark.utils import Evidence
    assert hash(Evidence("t", "d", 1, 2)) == hash(ev)


def test_cli_parsing(tmp_path):
    a = te.parse_args(["--data_dir", "data", "--output_dir", str(tmp_path), "--model_params", "p.json"])
    assert a.method == "transformer_attribution" and a.split == "test" and a.batch_size == 8
    assert a.iou_thresholds == [0.5]
    assert a.state_dict == os.path.join(str(tmp_path), "classifier", "classifier.pt")
    a = te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p", "--method", "rollout", "--split", "val",
                       "--state-dict", "w.pt", "--batch-size", "3", "--iou-thresholds", "0.5", "0.1"])
    assert (a.method, a.split, a.state_dict, a.batch_size, a.iou_thresholds) == ("rollout", "val", "w.pt", 3, [0.5, 0.1])
    assert set(te.METHOD_FOLDER) == set(te.METHODS) == set(te.METHOD_GENERATOR)
    for bad in (["--method", "lrp_x"], ["--batch-size", "0"]):
        with pytest.raises(SystemExit):
            te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p"] + bad)


def test_rationale_lines_from_an_order_nest_and_clip():
    lines = te.rationale_lines(["d"], ks=(1, 2, 5), order=[[4, 0, -1, -1, -1]])
    preds = [json.loads(lines[k][0])["rationales"][0]["hard_rationale_predictions"] for k in (1, 2, 5)]
    assert [p["start_token"] for p in preds[0]] == [4]
    assert [p["start_token"] for p in preds[1]] == [4, 4, 0]
    assert [p["start_token"] for p in preds[2]] == [4, 4, 0, 4, 0]
