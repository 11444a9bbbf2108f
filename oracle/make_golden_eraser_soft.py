"""Generate ``tests/golden/eraser_soft.npz`` from ``tests/golden/eraser.npz`` and the UNMODIFIED reference's models and
``metrics.py`` on CPU (authoring container).

    python -m oracle.make_golden_eraser_soft          # from the repo root, needs /root/reference, transformers, sklearn

TEST INFRASTRUCTURE.  Everything scored here is the reference's own:
 * the documents, annotations, tiny BERT and per-method word scores (the reference's pooling of the reference's maps)
   are those of ``eraser.npz``; its longer documents are truncated at 32 pieces, so their words past truncation form a
   tail, some of it inside a truth span;
 * soft scores: per method one result line per annotation holds the W word scores followed by a 0 per tail word; the
   reference's ``PositionScoredDocument.from_results`` pairs them with the truth of the documents' word lists and
   ``score_soft_tokens`` scores them (the per-document values with the same sklearn calls); the reference's
   ``attn_gradcam`` maps of the tiny BERT are NaN throughout, and the error sklearn raises for them is kept instead;
 * tokens to flip, by brute force: per method and document, the comprehensiveness row of every selection size
   k = 1 .. W (``oracle.eraser_faithfulness.reduce_rows`` on the reference's word ranking) runs at batch 1 through the
   reference's own fp32 ``BertForSequenceClassification`` (``transformer_attribution``) or ``BERT_cls_lrp`` (the other
   five); the smallest k whose argmax differs from the original's is the document's value, the word count when none
   does.  The logit margin of every row (the original class's logit minus the other class's) is kept, so a test can
   tell a rounding tie from a disagreement; the mean fraction is ``metrics.py``'s (``:337-346``).
"""
import json
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                     # noqa: E402
from oracle import eraser_faithfulness as of             # noqa: E402
from oracle import eraser_soft as osoft                  # noqa: E402
from oracle.make_golden_eraser import CLASSES, METHODS, build, params   # noqa: E402
from oracle.make_golden_eraser_faithfulness import forward_probs   # noqa: E402

SRC = os.path.join(ROOT, "tests", "golden", "eraser.npz")
OUT = os.path.join(ROOT, "tests", "golden", "eraser_soft.npz")
FLIP_SHIFT = 0.0392                     # added to class 0's classifier bias: the predictions sit near the boundary


def run():
    import sklearn
    from sklearn.metrics import auc, average_precision_score, precision_recall_curve, roc_auc_score
    from transformer_explainability_b200 import eraser as te
    src = np.load(SRC)
    docids = [str(d) for d in src["docids"]]
    docs = {d: str(t) for d, t in zip(docids, src["docs"])}
    ann_lines = [str(a) for a in src["annotations"]]
    out = {"sklearn": np.array(sklearn.__version__)}
    rh._prepare_bert_imports()
    p = params()
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "test.jsonl"), "w") as f:
            f.write("".join(line + "\n" for line in ann_lines))
        with rh._ref_imports():
            from BERT_rationale_benchmark import metrics as rmetrics
            from BERT_rationale_benchmark import utils as rutils
            test = rutils.annotations_from_jsonl(os.path.join(tmp, "test.jsonl"))
            doc_of = [next(iter(a.evidences))[0].docid for a in test]
            flat = {d: docs[d].split() for d in docids}               # the documents' word lists
            ids = {d: [int(i) for i in src["ids." + d]] for d in docids}
            ranges = {d: te.word_piece_ranges(flat[d], [str(x) for x in src["pieces." + d]]) for d in docids}
            out["n_words"] = np.array([len(flat[d]) for d in doc_of])
            out["W"] = np.array([len(ranges[d]) for d in doc_of])
            Wmax = int(out["W"].max())
            for method, kind, which, kw in METHODS:
                lines = []
                per_doc = np.zeros((len(test), 3))
                single = np.zeros(len(test), dtype=bool)
                for i, (a, d) in enumerate(zip(test, doc_of)):
                    words = src["%s.words.%s" % (method, d)]
                    lines.append({"annotation_id": a.annotation_id, "rationales": [
                        {"docid": d, "soft_rationale_predictions": osoft.soft_prediction(words, len(flat[d]))}]})
                paired = rmetrics.PositionScoredDocument.from_results(lines, test, flat, use_tokens=True)
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    try:
                        scores = rmetrics.score_soft_tokens(paired)
                    except ValueError as e:                           # NaN word scores: sklearn rejects them
                        scores, paired = {"error": str(e)}, []
                        per_doc[:] = np.nan
                    for i, ps in enumerate(paired):
                        t = [int(x) for x in ps.truths]
                        pr, rc, _ = precision_recall_curve(t, ps.scores)
                        single[i] = len(set(t)) < 2
                        per_doc[i] = (auc(rc, pr), average_precision_score(t, ps.scores),
                                      np.nan if single[i] else roc_auc_score(t, ps.scores))
                out["%s.soft_lines" % method] = np.array([json.dumps(l) for l in lines])
                out["%s.soft_scores" % method] = np.array(json.dumps(scores))
                out["%s.soft_doc" % method] = per_doc
                out["%s.single" % method] = single
                # tokens to flip by brute force: one reference forward per selection size, with the classifier as
                # given (its predictions never flip on these documents) and with FLIP_SHIFT added to class 0's bias
                for tag, shift in (("", 0.0), ("_shift", FLIP_SHIFT)):
                    q = dict(p)
                    q["classifier.bias"] = p["classifier.bias"] + torch.tensor([shift, 0.0])
                    model = build(kind, q)
                    flip = np.zeros(len(test), dtype=np.int64)
                    flipped = np.zeros(len(test), dtype=bool)
                    margins = np.full((len(test), Wmax), np.nan)
                    margin0 = np.zeros(len(test))
                    for i, (a, d) in enumerate(zip(test, doc_of)):
                        words = src["%s.words.%s" % (method, d)]
                        if shift:                       # the bias moves the logits only: the maps stay the reference's
                            x = torch.tensor([ids[d]])
                            cam = rh.bert_generate(model, x, torch.ones_like(x), which, index=CLASSES.index(a.classification),
                                                   **kw)[0].numpy()
                            ref = src["%s.map.%s" % (method, d)]
                            assert np.array_equal(np.isnan(cam), np.isnan(ref)) and \
                                np.nanmax(np.abs(np.nan_to_num(cam) - np.nan_to_num(ref)), initial=0) <= 1e-6, (method, d)
                        rows = [ids[d]] + [of.reduce_rows(ids[d], ranges[d], words, k)[0] for k in range(1, len(words) + 1)]
                        logits = np.stack([lg.numpy() for _, lg in forward_probs(model, rows, torch.float32)])
                        pred0 = int(np.argmax(logits[0]))
                        m = logits[:, pred0] - logits[:, 1 - pred0]
                        margin0[i] = m[0]
                        margins[i, :len(words)] = m[1:]
                        k = next((k for k in range(1, len(words) + 1) if int(np.argmax(logits[k])) != pred0), None)
                        flip[i], flipped[i] = (k, True) if k is not None else (len(flat[d]), False)
                    frac = []
                    for a, t in zip(test, flip):                        # metrics.py:337-346
                        dd = set(ev.docid for grp in a.evidences for ev in grp)
                        frac.append(int(t) / sum(len(flat[x]) for x in dd))
                    out["%s.flip%s" % (method, tag)] = flip
                    out["%s.flipped%s" % (method, tag)] = flipped
                    out["%s.margins%s" % (method, tag)] = margins
                    out["%s.margin0%s" % (method, tag)] = margin0
                    out["%s.flip_fraction%s" % (method, tag)] = np.average(frac)
                    print(method, "flip%s" % tag, flip.tolist(), "never", int((~flipped).sum()))
                print(method, "soft", scores)
    np.savez_compressed(OUT, **out)
    print("eraser_soft.npz", len(out), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    run()
