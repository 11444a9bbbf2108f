"""ERASER soft-token and tokens-to-flip oracle (TEST INFRASTRUCTURE, numpy / plain Python).

Restates, on top of ``oracle/eraser.py``'s word ranking and ``oracle/eraser_faithfulness.py``'s reduced rows:

* ``tail_counts``        the positive and negative words of a document past truncation (they score 0)
* ``soft_prediction``    the soft prediction of one document: its W word scores, then one 0 per tail word
* ``curve``              sklearn's ``_binary_clf_curve``: one point per tie group (bit-equal scores, -0 == +0), in
                         descending score order, with the cumulative (tps, fps)
* ``soft_scores``        ``auc(recall, precision)`` of ``precision_recall_curve``, ``average_precision_score`` and
                         ``roc_auc_score`` (NaN for a single-class document) of one document, in fp64, from the curve
* ``score_soft_tokens``  ``metrics.py``'s aggregation (``:217-253``): AUPRC over every document, AP and ROC AUC over the
                         documents with both classes
* ``tokens_to_flip``     the brute-force search (DESIGN.md §1): the smallest k whose comprehensiveness row has another
                         argmax than the original prediction, else the document's word count
"""
import math
import warnings

import numpy as np

from oracle.eraser_faithfulness import reduce_rows


def tail_counts(spans, W, n_words):
    """(positives, negatives) among the words W .. n_words - 1 of a document, for truth spans [(start, end)]."""
    pos = set(t for s, e in spans for t in range(max(s, W), min(e, n_words)))
    return len(pos), n_words - W - len(pos)


def truth_vector(spans, n_words):
    """One bool per document word: inside some truth span (``PositionScoredDocument.from_results``)."""
    t = [False] * n_words
    for s, e in spans:
        for w in range(s, e):
            t[w] = True
    return t


def soft_prediction(words, n_words):
    """The W fp32 word scores (as Python floats), then 0.0 for each of the n_words - W words past truncation."""
    return [float(x) for x in np.asarray(words, dtype=np.float32)] + [0.0] * (n_words - len(words))


def curve(scores, truth):
    """[(tps, fps)] per tie group in descending score order; a NaN score raises ValueError (as sklearn)."""
    s = np.asarray(scores, dtype=np.float64)
    t = np.asarray(truth, dtype=bool)
    if np.isnan(s).any():
        raise ValueError("a soft score is NaN")
    out, tp, fp = [], 0, 0
    for v in sorted(set(s.tolist()), reverse=True):            # -0.0 == 0.0: one group
        m = s == v
        tp += int(np.sum(t & m))
        fp += int(np.sum(~t & m))
        out.append((tp, fp))
    return out


def soft_scores(scores, truth):
    """(auprc, average precision, roc auc) of one document; roc auc is NaN when it holds one class only."""
    pts = curve(scores, truth)
    P, N = pts[-1]
    pr = ap = 0.0
    roc = 0
    tq = fq = 0
    q, rq = 1.0, 0.0                                            # precision_recall_curve's end point (recall 0, precision 1)
    for tp, fp in pts:
        p = tp / (tp + fp)
        r = tp / P if P else 1.0
        pr += (r - rq) * (p + q) / 2.0
        ap += (r - rq) * p
        roc += (fp - fq) * (tp + tq)
        tq, fq, q, rq = tp, fp, p, r
    return pr, ap, (roc / (2.0 * P * N) if P and N else math.nan)


def score_soft_tokens(per_doc, single_class):
    """``score_soft_tokens``' dict from per-document (auprc, ap, roc auc) rows and single-class flags, in document
    order."""
    if len(per_doc) == 0:
        return {"auprc": 0.0, "average_precision": 0.0, "roc_auc_score": 0.0}
    keep = [i for i in range(len(per_doc)) if not single_class[i]]
    with warnings.catch_warnings():                            # no two-class document: numpy's mean of nothing, NaN
        warnings.simplefilter("ignore")
        return {"auprc": np.average([r[0] for r in per_doc]),
                "average_precision": np.average([per_doc[i][1] for i in keep]),
                "roc_auc_score": np.average([per_doc[i][2] for i in keep])}


def tokens_to_flip(predict, ids, ranges, scores, n_words, pred0):
    """(k, flipped): the smallest k = 1 .. W whose comprehensiveness row (``reduce_rows``) ``predict`` (id list -> class
    index) maps to a class other than pred0, or (n_words, False) when none does."""
    for k in range(1, len(ranges) + 1):
        if predict(reduce_rows(ids, ranges, scores, k)[0]) != pred0:
            return k, True
    return n_words, False
