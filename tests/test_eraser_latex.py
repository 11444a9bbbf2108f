"""CPU: the LaTeX heat maps of the ERASER pipeline (``eraser.latex_document``, ``ground_truth_documents``,
``comparison_figures``) and the fp32 restatement of ``generate()``'s weights (``oracle/eraser_latex.py``) against the
reference's own files (``tests/golden/eraser_latex.npz``).

- Every ``generate()`` file of the fixture (six methods, gold class and counterfactual, and the hand-built rows) is rebuilt
  byte for byte from its tokens and the weights printed in it; the ``ground_truth`` and ``generate_all`` files from the
  fixture's documents, annotations and logits.
- The restatement, fed the reference's own maps (clamped) and the hand-built rows (unclamped), gives the printed weights
  bit for bit.
The ground-truth spans come from each annotation's first evidence group, whose order follows the hash seed: the fixture was
written with PYTHONHASHSEED=0, and that comparison runs in a child interpreter with that seed."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import eraser_latex as ol
from transformer_explainability_b200 import eraser as te

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "eraser_latex.npz")
METHODS = ("transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout")
FOLDER = te.METHOD_FOLDER


def load():
    g = np.load(GOLDEN)
    docids = [str(d) for d in g["docids"]]
    docs = {d: str(t) for d, t in zip(docids, g["docs"])}
    anns = []
    for line in g["annotations"]:
        content = json.loads(str(line))
        content["evidences"] = frozenset(tuple(te.Evidence(**ev) for ev in grp) for grp in content["evidences"])
        anns.append(te.Annotation(**content))
    enc = {te.annotation_docid(a): ([int(i) for i in g["ids.%d" % j]], [str(p) for p in g["pieces.%d" % j]])
           for j, a in enumerate(anns)}
    return g, docs, anns, enc


@pytest.fixture(scope="module")
def golden():
    return load()


def text(g, name):
    return bytes(g["file." + name]).decode("utf-8")


def _bits(a):
    a = np.array(a, dtype=np.float32)
    a[np.isnan(a)] = np.float32("nan")
    return a.view(np.int32)


def method_files(g, anns):
    """(method, j, kind, file name) of every generate() file of the fixture."""
    names = set(str(f) for f in g["files"])
    out = []
    for m in METHODS:
        for j in range(len(anns)):
            gt = [n for n in names if n.startswith("%s/%d_GT_" % (FOLDER[m], j))]
            assert len(gt) == 1, (m, j)
            out.append((m, j, "GT", gt[0]))
            cf = "%s/%d_CF.tex" % (FOLDER[m], j)
            assert (cf in names) == (m in te.LATEX_CF_METHODS), (m, j)
            if cf in names:
                out.append((m, j, "CF", cf))
    return out


def test_fixture_covers_every_file(golden):
    g, _, anns, _ = golden
    n = len(anns)
    assert len(g["files"]) == len(method_files(g, anns)) + 2 * n      # + ground_truth + generate_all
    assert sum(str(f).startswith("ground_truth/") for f in g["files"]) == n
    assert sum(str(f).startswith("generate_all/") for f in g["files"]) == n


def test_latex_document_rebuilds_every_method_file(golden):
    g, _, anns, _ = golden
    for m, j, kind, name in method_files(g, anns):
        ref = text(g, name)
        w = ol.file_weights(ref)
        pieces = [str(p) for p in g["pieces.%d" % j]]
        assert len(w) == len(pieces)
        assert te.latex_document(pieces, w) == ref, (m, j, kind)


def test_oracle_weights_equal_the_reference_on_the_maps(golden):
    g, _, anns, _ = golden
    for m, j, kind, name in method_files(g, anns):
        cam = g["%s.%s.%d" % (m, "map" if kind == "GT" else "cf_map", j)]
        n = len(g["pieces.%d" % j])
        assert np.array_equal(_bits(ol.latex_weights(cam, n, clamp=True)), _bits(ol.file_weights(text(g, name)))), \
            (m, j, kind)


def test_hand_rows(golden):
    g = golden[0]
    nan_rows = 0
    for i in range(int(g["hand.count"])):
        tokens = [str(t) for t in g["hand.tokens.%d" % i]]
        ref = bytes(g["hand.file.%d" % i]).decode("utf-8")
        w = ol.latex_weights(g["hand.values.%d" % i], len(tokens), clamp=False)
        assert np.array_equal(_bits(w), _bits(ol.file_weights(ref))), i
        assert te.latex_document(tokens, w) == ref, i
        nan_rows += bool(np.isnan(w).any())
    assert nan_rows >= 3


def test_figure_pages(golden):
    g, _, anns, _ = golden
    classes = {"NEG": 0, "POS": 1}
    pred = [int(np.argmax(g["logits.%d" % j])) for j in range(len(anns))]
    docs = te.comparison_figures(anns, classes, pred, str(g["output_dir"]))
    assert sorted("generate_all/" + name for name, _ in docs.values()) == \
        sorted(str(f) for f in g["files"] if str(f).startswith("generate_all/"))
    for name, body in docs.values():
        assert body == text(g, "generate_all/" + name), name


def _ground_truth_check():
    g, docs, anns, enc = load()
    out = te.ground_truth_documents(anns, docs, enc)
    assert sorted(out) == list(range(len(anns)))
    for j, (name, body) in out.items():
        assert name == "visual_results_%d.tex" % j
        assert body == text(g, "ground_truth/" + name), j
    return len(out)


def test_ground_truth_documents():
    if os.environ.get("PYTHONHASHSEED") == "0":
        _ground_truth_check()
        return
    code = "import sys; sys.path[:0] = %r; import test_eraser_latex as t; print(t._ground_truth_check())" % (
        [HERE, os.path.dirname(HERE)],)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PYTHONHASHSEED="0"), capture_output=True,
                       text=True, cwd=os.path.dirname(HERE))
    assert r.returncode == 0, r.stderr[-3000:]
    assert int(r.stdout.split()[-1]) == 8


def test_input_words_cut_and_alignment():
    words = ["hello", "world", "again"]
    pieces = ["[CLS]", "hell", "##o", "wo", "[SEP]"]
    assert te.input_words(words, pieces) == ["hello", "wo"]
    with pytest.raises(ValueError):
        te.input_words(["help", "x", "y"], ["[CLS]", "hello", "wor", "[SEP]"])


def test_clean_word_order_and_glued_pieces():
    assert te.clean_word("a\\b{c}%#_^&") == "a\\\\b\\{c\\}\\%\\#\\_\\^\\&"
    doc = te.latex_document(["[CLS]", "play", "##ing", "$x$", "[SEP]"], [0.0, 100.0, 50.5, 1.0, 0.0])
    assert " \\colorbox{red!100.0}{\\strut play}\\colorbox{red!50.5}{\\strut ing} \\colorbox{red!1.0}{\\strut x}" in doc
    with pytest.raises(ValueError):
        te.latex_document(["a", "b"], [1.0])


def test_command_line_options():
    args = te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p", "--method", "partial_lrp",
                          "--latex"])
    assert args.latex and args.method == "partial_lrp"
    for mode in te.FIGURE_MODES:
        assert te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p", "--method", mode]).method == mode
        with pytest.raises(SystemExit):
            te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p", "--method", mode, "--latex"])
    assert not te.parse_args(["--data_dir", "d", "--output_dir", "o", "--model_params", "p"]).latex


def test_latex_needs_two_classes():
    with pytest.raises(ValueError, match="two classes"):
        te.eraser_eval(lambda **kw: None, {}, [], {}, {"A": 0, "B": 1, "C": 2}, latex=True)
