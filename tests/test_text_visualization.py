"""CPU checks of the BERT word-importance command (``transformer_explainability_b200.text_visualization``): argument
parsing, sentence-pair tokenisation from a local ``vocab.txt``, captum's colour rule at its boundaries, and the JSON and
HTML writers against ``oracle/text_visualization.py``."""
import json

import numpy as np
import pytest

from oracle import text_visualization as otv
from transformer_explainability_b200 import text_visualization as tv

VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "a", "b", "c", "d", "the", "movie", "##s", "was", "good", "bad",
         "."]


def write_vocab(path):
    path.mkdir(parents=True, exist_ok=True)
    (path / "vocab.txt").write_text("\n".join(VOCAB) + "\n")
    (path / "config.json").write_text(json.dumps({"model_type": "bert", "vocab_size": len(VOCAB)}))
    return str(path)


def test_parse_args():
    a = tv.parse_args(["--model-dir", "m", "--text", "a b", "--text", "c", "--text-pair", "x", "--text-pair", "y",
                       "--output-dir", "o"])
    assert a.text == ["a b", "c"] and a.text_pair == ["x", "y"] and a.start_layer == 0 and a.batch_size == 16
    assert a.method == "transformer_attribution" and a.class_index is None and a.labels is None
    a = tv.parse_args(["--model-dir", "m", "--text", "a", "--output-dir", "o", "--class-index", "1", "--labels",
                       "NEGATIVE", "POSITIVE", "--method", "attn_grad_rollout", "--batch-size", "4", "--start-layer", "11"])
    assert a.class_index == 1 and a.labels == ["NEGATIVE", "POSITIVE"] and a.method == "attn_grad_rollout"
    assert a.batch_size == 4 and a.start_layer == 11 and a.text_pair is None
    for bad in (["--text-pair", "x", "--text-pair", "y"], ["--batch-size", "0"], ["--method", "full"],
                ["--start-layer", "-1"]):
        with pytest.raises(SystemExit):
            tv.parse_args(["--model-dir", "m", "--text", "a", "--output-dir", "o"] + bad)
    with pytest.raises(SystemExit):
        tv.parse_args(["--model-dir", "m", "--output-dir", "o"])


def test_class_names():
    class C:
        num_labels = 2
        id2label = {0: "NEGATIVE", 1: "POSITIVE"}
    assert tv.class_names(C()) == ["NEGATIVE", "POSITIVE"]
    assert tv.class_names(C(), ["neg", "pos"]) == ["neg", "pos"]
    with pytest.raises(ValueError):
        tv.class_names(C(), ["only"])
    C.id2label = {}
    assert tv.class_names(C()) == ["LABEL_0", "LABEL_1"]


def test_tokenize_pairs(tmp_path):
    tok = tv.load_tokenizer(write_vocab(tmp_path / "m"))
    ids, tt, mask = tv.tokenize(tok, ["a b", "the movies was good ."], ["c d", "a"])
    assert ids.shape == tt.shape == mask.shape == (2, 10)
    assert tok.convert_ids_to_tokens(ids[0].tolist()) == ["[CLS]", "a", "b", "[SEP]", "c", "d", "[SEP]"] + ["[PAD]"] * 3
    assert tt[0].tolist() == [0, 0, 0, 0, 1, 1, 1, 0, 0, 0] and mask[0].tolist() == [1] * 7 + [0] * 3
    assert tok.convert_ids_to_tokens(ids[1].tolist()) == ["[CLS]", "the", "movie", "##s", "was", "good", ".", "[SEP]", "a",
                                                          "[SEP]"]
    assert tt[1].tolist() == [0] * 8 + [1, 1] and mask[1].tolist() == [1] * 10
    ids1, tt1, mask1 = tv.tokenize(tok, ["a b"])
    assert tok.convert_ids_to_tokens(ids1[0].tolist()) == ["[CLS]", "a", "b", "[SEP]"]
    assert tt1.tolist() == [[0, 0, 0, 0]] and mask1.tolist() == [[1, 1, 1, 1]]


@pytest.mark.parametrize("a,expected", [
    (1.0, "hsl(120, 75%, 50%)"), (-1.0, "hsl(0, 75%, 60%)"), (0.0, "hsl(0, 75%, 100%)"), (-0.0, "hsl(0, 75%, 100%)"),
    (3.0, "hsl(120, 75%, 50%)"), (-7.0, "hsl(0, 75%, 60%)"),
    # 50 a just below an integer in double: fp32 0.7 is 0.699999988..., 50 a = 34.9999994 -> 34 (an fp32 product rounds
    # to 35.0 and would give 65%)
    (np.float32(0.7), "hsl(120, 75%, 66%)"), (np.float32(0.3), "hsl(120, 75%, 85%)"),
    (np.float32(-0.7), "hsl(0, 75%, 73%)"), (np.float32(0.02), "hsl(120, 75%, 100%)"),
    (float("nan"), "hsl(120, 75%, 50%)"),
])
def test_color_rule(a, expected):
    assert tv.get_color(a) == expected == otv.color(a)


def test_color_rule_matches_oracle_on_a_grid():
    g = np.random.default_rng(0)
    vals = np.concatenate([g.uniform(-1.2, 1.2, 2000).astype(np.float32),
                           (np.arange(-50, 51) / 50).astype(np.float32),
                           np.nextafter((np.arange(-50, 51) / 50).astype(np.float32), np.float32(0))])
    for v in vals:
        assert tv.get_color(v) == otv.color(v)


def test_normalize_oracle_conventions():
    row = np.array([0.5, 1.5, 1.0, 9.0], np.float32)
    assert otv.normalize(row, 3, 1.0).tolist() == [0.0, 1.0, 0.5, 0.0]
    assert otv.normalize(row, 3, -1.0).tolist() == [-0.0, -1.0, -0.5, 0.0]
    assert otv.normalize(np.full(4, 2.0, np.float32), 4, -1.0).tolist() == [0.0] * 4
    n = otv.normalize(np.array([1.0, np.nan, 2.0, 5.0], np.float32), 3, 1.0)
    assert np.isnan(n[:3]).all() and n[3] == 0
    assert otv.sign_of("NEGATIVE") == -1.0 and otv.sign_of("POSITIVE") == 1.0 and otv.sign_of("negative") == 1.0


def _records():
    tokens = [["[CLS]", "a", "<b>", "[SEP]", "c", "[SEP]"], ["[CLS]", "the", "movie", "[SEP]"]]
    tts = [[0, 0, 0, 0, 1, 1], [0, 0, 0, 0]]
    g = np.random.default_rng(3)
    maps = g.standard_normal((2, 6)).astype(np.float32)
    probs = np.array([[0.25, 0.75], [0.9, 0.1]], np.float32)
    names = ["NEGATIVE", "POSITIVE"]
    pred = probs.argmax(1)
    scores = np.stack([otv.normalize(maps[b], len(tokens[b]), otv.sign_of(names[pred[b]])) for b in range(2)])
    return tokens, tts, scores, probs, names


def test_json_and_html_writers(tmp_path):
    tokens, tts, scores, probs, names = _records()
    recs = otv.records(tokens, tts, scores, probs, names)
    assert recs[1]["explained_label"] == "NEGATIVE" and max(recs[1]["scores"]) <= 0
    for r in recs:
        r.update(text="t", text_pair=None)
    jp, hp = tv.write_outputs(recs, str(tmp_path / "out"))
    assert json.load(open(jp)) == recs
    page = open(hp).read()
    assert page == otv.table(recs)
    assert page == tv.render_html(recs)
    assert "> #b </font>" in page                    # captum's special-token form of "<b>", never raw markup
    pos = 0
    for r in recs:                                   # every token's mark, in order, with its colour
        for t, a in zip(r["tokens"], r["scores"]):
            m = otv.mark(t, a)
            i = page.find(m, pos)
            assert i >= 0, (t, a)
            pos = i + len(m)
    assert "POSITIVE (0.75)" in page and "NEGATIVE (0.90)" in page
