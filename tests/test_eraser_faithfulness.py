"""CPU: the ERASER faithfulness evaluation's oracle (``oracle/eraser_faithfulness.py``) and the host side of ``eraser.py``
against ``tests/golden/eraser_faithfulness.npz``: the reduced rows of every method and selection, and ``metrics.py``'s
``score_classifications`` dict on the reference's own probabilities and on a hand-built corner set.

``score_classifications`` orders its labels by ``list(set(...))``, whose order follows the hash seed; the fixture was written
with PYTHONHASHSEED=0, and the score comparisons run in a child interpreter with that seed."""
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

from oracle import eraser_faithfulness as of
from transformer_explainability_b200 import eraser as te

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser_faithfulness.npz")
METHODS = te.METHODS
CLASSES = ["NEG", "POS"]


def load():
    import test_eraser as ce
    g, docids, docs, anns = ce.load()
    return np.load(GOLDEN), g, docids, docs, anns


def _annotations(lines):
    out = []
    for line in lines:
        content = json.loads(str(line))
        content["evidences"] = frozenset(tuple(te.Evidence(**ev) for ev in grp) for grp in content["evidences"])
        out.append(te.Annotation(**content))
    return out


def _arrays(lines, names):
    """The result lines as classification_scores_from_probs takes them: pred, probs, comp, suff, thresholds."""
    insts = [json.loads(str(l)) for l in lines]
    thr = [s["threshold"] for s in insts[0]["thresholded_scores"]]
    vec = lambda d: [d[c] for c in names]                                    # noqa: E731
    pred = [names.index(x["classification"]) for x in insts]
    probs = [vec(x["classification_scores"]) for x in insts]
    comp = [[vec(x["comprehensiveness_classification_scores"])] +
            [vec(s["comprehensiveness_classification_scores"]) for s in x["thresholded_scores"]] for x in insts]
    suff = [[vec(x["sufficiency_classification_scores"])] +
            [vec(s["sufficiency_classification_scores"]) for s in x["thresholded_scores"]] for x in insts]
    return pred, probs, comp, suff, thr


@pytest.mark.parametrize("method", METHODS)
def test_oracle_rows_reproduce_the_fixture(method):
    z, g, docids, docs, anns = load()
    fr = [float(f) for f in z["fractions"]]
    for i, a in enumerate(anns):
        d = te.annotation_docid(a)
        ids = [int(x) for x in g["ids." + d]]
        ranges = te.word_piece_ranges(docs[d].split(), [str(p) for p in g["pieces." + d]])
        words = g["%s.words.%s" % (method, d)]
        n = of.select_counts(fr, len(words))
        assert n == [te.select_count(f, len(words)) for f in fr] == z["%s.n_select" % method][i].tolist()
        for j, k in enumerate(n):
            for t, row in enumerate(of.reduce_rows(ids, ranges, words, k)):
                L = int(z["%s.red_len" % method][i, j, t])
                assert row == z["%s.red_ids" % method][i, j, t, :L].tolist(), (method, d, j, t)
                assert not z["%s.red_ids" % method][i, j, t, L:].any()
            assert z["%s.red_len" % method][i, j].sum() == len(ids) + 2


def test_default_k_is_the_human_fraction():
    z, g, docids, docs, anns = load()
    words = {d: len(te.word_piece_ranges(docs[d].split(), [str(p) for p in g["pieces." + d]])) for d in docids}
    dd = [te.annotation_docid(a) for a in anns]
    got = te.human_fraction(anns, dd, [words[d] for d in dd], te.TruthIndex(anns))
    assert got == float(z["fractions"][0])


def test_select_count_rounding_and_clipping():
    assert [te.select_count(f, 10) for f in (0.01, 0.05, 0.1, 0.14, 0.15, 0.25, 1.0)] == [1, 1, 1, 1, 2, 3, 10]
    assert te.select_count(0.5, 5) == 3 and te.select_count(0.3, 5) == 2          # 2.5 -> 3, 1.5 -> 2 (half up)
    assert te.select_count(0.01, 1) == 1 and te.select_count(0.5, 0) == 0
    assert of.select_counts([0.5, 0.3, 0.01, 1.0], 5) == [3, 2, 1, 5]


def _child(fn):
    """Run ``fn`` of this module in a child interpreter with PYTHONHASHSEED=0 and return its JSON result."""
    if os.environ.get("PYTHONHASHSEED") == "0":
        return json.loads(json.dumps(globals()[fn]()))
    code = "import sys, json; sys.path[:0] = [%r, %r]; import test_eraser_faithfulness as t; print(json.dumps(t.%s()))" % (
        HERE, os.path.dirname(HERE), fn)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PYTHONHASHSEED="0"), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def scores_of_both():
    """{set: (oracle dict, host dict)} for every method's lines and the corner set."""
    z, _, _, _, anns = load()
    aopc = [float(t) for t in z["aopc_thresholds"]]
    sets = {m: (anns, z["%s.lines" % m], CLASSES) for m in METHODS}
    sets["corner"] = (_annotations(z["corner.annotations"]), z["corner.instances"], ["a", "b", "c"])
    out = {}
    for name, (a, lines, names) in sets.items():
        pred, probs, comp, suff, thr = _arrays(lines, names)
        out[name] = (of.score_classifications([json.loads(str(l)) for l in lines], a, aopc),
                     te.classification_scores_from_probs(a, names, pred, probs, comp, suff, thr, aopc))
    return out


def test_scores_equal_the_reference_bit_for_bit():
    z = np.load(GOLDEN)
    assert str(z["hashseed"]) == "0"
    got = _child("scores_of_both")
    for name in list(METHODS) + ["corner"]:
        ref = json.loads(str(z["%s.scores" % name]))
        assert got[name][0] == ref, name
        assert got[name][1] == ref, name
    corner = json.loads(str(z["corner.scores"]))
    assert corner["comprehensiveness_kl"] == float("inf") and corner["prf"]["c"]["precision"] == 0.0


@pytest.mark.parametrize("seed", range(4))
def test_restatement_equals_sklearn_and_scipy(seed):
    skm = pytest.importorskip("sklearn.metrics")
    stats = pytest.importorskip("scipy.stats")
    g = np.random.default_rng(seed)
    for n, C in ((1, 2), (7, 3), (50, 2), (200, 5)):
        truth = g.integers(0, C, n)
        truth[:C] = np.arange(C)[:min(C, n)] if n >= C else truth[:C]
        if n < C:
            continue
        pred = g.integers(0, C - (seed % 2), n)                             # odd seeds: the last class is never predicted
        names = ["c%d" % i for i in range(C)]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = skm.classification_report(truth, pred, output_dict=True, target_names=names, digits=3)
        assert te._classification_report(truth, pred, names) == ref == of.class_report(truth, pred, names)
        assert float(np.average(truth == pred)) == skm.accuracy_score(truth, pred)
        for _ in range(20):
            p = g.random(C).astype(np.float32).astype(np.float64)
            q = g.random(C).astype(np.float32).astype(np.float64)
            p[g.random(C) < 0.3] = 0
            q[g.random(C) < 0.3] = 0
            if p.sum() == 0 or q.sum() == 0:
                continue
            for args in ((p.tolist(),), (p.tolist(), q.tolist())):
                want = stats.entropy(*args)
                assert te._entropy(*args) == want and of.entropy(*args) == want, args


def _data_dir(tmp, docs, anns_lines):
    os.makedirs(os.path.join(tmp, "docs"))
    for d, text in docs.items():
        with open(os.path.join(tmp, "docs", d), "w") as f:
            f.write(text)
    with open(os.path.join(tmp, "test.jsonl"), "w") as f:
        f.write("".join(str(l) + "\n" for l in anns_lines))


def test_reference_metrics_accepts_the_written_results(tmp_path, monkeypatch):
    from oracle import ref_harness as rh
    if not rh.available():
        pytest.skip("reference not present")
    z, g, docids, docs, anns = load()
    aopc = [float(t) for t in z["aopc_thresholds"]]
    m = "transformer_attribution"
    dd = [te.annotation_docid(a) for a in anns]
    pred, probs, comp, suff, thr = _arrays(z["%s.lines" % m], CLASSES)
    selected = [[h["start_token"] for h in json.loads(str(l))["rationales"][0]["hard_rationale_predictions"]]
                for l in z["%s.lines" % m]]
    res = {"lines": {}, "scores": {}, "faithfulness": {
        "lines": te.faithfulness_lines(anns, dd, CLASSES, pred, probs, comp, suff, thr, selected),
        "scores": te.classification_scores_from_probs(anns, CLASSES, pred, probs, comp, suff, thr, aopc)}}
    assert res["faithfulness"]["lines"] == [str(l) for l in z["%s.lines" % m]]
    out = str(tmp_path / "out")
    te.write_results(res, out)
    assert sorted(os.listdir(out)) == ["faithfulness_results.jsonl", "faithfulness_scores.json"]
    data = str(tmp_path / "data")
    _data_dir(data, docs, g["annotations"])
    rh._prepare_bert_imports()
    with rh._ref_imports():
        from BERT_rationale_benchmark import metrics as rmetrics
        results = rmetrics.load_jsonl(os.path.join(out, "faithfulness_results.jsonl"))
        flat = rmetrics.load_flattened_documents(data, set(dd))
        rmetrics.verify_instances(results, flat)                         # raises on any logged error
        score_file = str(tmp_path / "scores.json")
        monkeypatch.setattr(sys, "argv", ["metrics.py", "--data_dir", data, "--split", "test", "--results",
                                          os.path.join(out, "faithfulness_results.jsonl"), "--score_file", score_file])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            rmetrics.main()
    with open(score_file) as f:
        main_scores = json.load(f)
    with open(os.path.join(out, "faithfulness_scores.json")) as f:
        assert main_scores["classification_scores"] == json.load(f)
    assert "token_prf" in main_scores                                    # the main-k words score as hard predictions


def test_cli_parsing():
    base = ["--data_dir", "d", "--output_dir", "o", "--model_params", "p"]
    a = te.parse_args(base)
    assert not a.faithfulness and a.aopc_thresholds == [0.01, 0.05, 0.1, 0.2, 0.5] and a.k_fraction is None
    a = te.parse_args(base + ["--faithfulness", "--aopc-thresholds", "0.1", "0.3", "--k-fraction", "0.25"])
    assert a.faithfulness and a.aopc_thresholds == [0.1, 0.3] and a.k_fraction == 0.25
    for bad in (["--k-fraction", "0"], ["--k-fraction", "1.5"], ["--aopc-thresholds", "0.1", "0.1"],
                ["--aopc-thresholds", "0"], ["--aopc-thresholds"] + ["0.01"] * 64):
        with pytest.raises(SystemExit):
            te.parse_args(base + bad)


def test_faithfulness_off_writes_todays_files(tmp_path):
    res = {"lines": {5: ["a"], 10: ["b"]}, "scores": {5: {"x": 1}, 10: {"x": 2}}}
    te.write_results(res, str(tmp_path))
    assert sorted(os.listdir(str(tmp_path))) == ["identifier_results_10.json", "identifier_results_5.json",
                                                 "scores_10.json", "scores_5.json"]


def test_fixture_covers_the_cases():
    z = np.load(GOLDEN)
    corner = [json.loads(str(l)) for l in z["corner.instances"]]
    anns = _annotations(z["corner.annotations"])
    assert {x["classification"] for x in corner} == {"a", "b"} and {a.classification for a in anns} == {"a", "b", "c"}
    assert any(0.0 in x["classification_scores"].values() for x in corner)
    assert any(a.annotation_id != te.annotation_docid(a) for a in anns)
    assert str(z["sklearn"]) and str(z["scipy"])
    for m in METHODS:
        n = z["%s.n_select" % m]
        assert n.min() == 1 and (n[:, 0] > n[:, 1]).any()                  # clipped to 1 word, and a main k above it
