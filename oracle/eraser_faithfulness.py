"""ERASER faithfulness oracle (TEST INFRASTRUCTURE, numpy / plain Python).

Restates, on top of ``oracle/eraser.py``'s word ranking:

* ``select_counts``          the selection size n(f, W) = min(W, max(1, floor(f * W + 0.5))) of each fraction f
* ``reduce_rows``            the comprehensiveness / sufficiency rows of one document (DESIGN.md §1): the rationale pieces
                             are the union of the piece ranges of the first n ranked words; comprehensiveness keeps
                             [CLS], the other inner pieces and [SEP], sufficiency [CLS], the rationale pieces and [SEP]
* ``score_classifications``  ``metrics.py``'s ``score_classifications`` (``:255-364``) with sklearn's
                             ``classification_report`` / ``accuracy_score`` and scipy's ``entropy`` written out, on the
                             result dicts of ``faithfulness_results.jsonl``; the label order is the reference's own
                             ``list(set(...))`` (it depends on the hash seed)
"""
import math

import numpy as np

from oracle.eraser import word_order


def select_counts(fractions, W):
    """n(f, W) = min(W, max(1, floor(f * W + 0.5))) for each fraction f in (0, 1], in Python floats."""
    return [min(W, max(1, int(math.floor(f * W + 0.5)))) for f in fractions]


def reduce_rows(ids, ranges, scores, n):
    """(comprehensiveness, sufficiency) id lists of one document [CLS] p_1 ... p_n [SEP] (ids, unpadded), its words'
    inclusive piece ranges, its word scores (the pooled clamped map) and a selection size n."""
    chosen = set()
    for w in word_order(scores)[:n]:
        a, b = ranges[int(w)]
        chosen.update(range(a, b + 1))
    inner = range(1, len(ids) - 1)
    comp = [ids[0]] + [ids[p] for p in inner if p not in chosen] + [ids[-1]]
    suff = [ids[0]] + [ids[p] for p in inner if p in chosen] + [ids[-1]]
    return comp, suff


def _log_ratio(x, y):
    """log(x / y) as scipy.special.rel_entr takes it: log1p((x - y) / y) for 0.5 < x / y < 2, else log(x / y)."""
    r = x / y
    return math.log1p((x - y) / y) if 0.5 < r < 2 else math.log(r)


def entropy(pk, qk=None):
    """scipy.stats.entropy: both inputs normalised; -x log x (0 at 0), or x log(x / y) (0 at x = 0, inf at y = 0 < x),
    summed with numpy; the logs are libm's (``math.log`` / ``math.log1p``), as scipy.special's."""
    pk = np.asarray(pk, dtype=np.float64)
    pk = pk / np.sum(pk, axis=0, keepdims=True)
    if qk is None:
        vec = [x if x != x else -x * math.log(x) if x > 0 else 0.0 if x == 0 else -math.inf for x in pk.tolist()]
    else:
        qk = np.asarray(qk, dtype=np.float64)
        qk = qk / np.sum(qk, axis=0, keepdims=True)
        vec = [math.nan if x != x or y != y else x * _log_ratio(x, y) if x > 0 and y > 0 else 0.0 if x == 0 and y >= 0
               else math.inf for x, y in zip(pk.tolist(), qk.tolist())]
    return np.sum(np.asarray(vec, dtype=np.float64))


def class_report(truth, pred, names):
    """sklearn's ``classification_report(truth, pred, output_dict=True, target_names=names)`` for labels
    0 .. len(names) - 1, each of which occurs in truth; a zero division gives 0."""
    truth, pred = np.asarray(truth), np.asarray(pred)
    L = range(len(names))
    tp = np.array([np.sum((truth == l) & (pred == l)) for l in L], dtype=np.int64)
    n_pred = np.array([np.sum(pred == l) for l in L], dtype=np.int64)
    n_true = np.array([np.sum(truth == l) for l in L], dtype=np.int64)

    def div(a, b):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        return np.where(b == 0, 0.0, a / np.where(b == 0, 1.0, b))
    p, r, f = div(tp, n_pred), div(tp, n_true), div(2.0 * tp, 1.0 * n_true + n_pred)
    out = {name: {"precision": float(p[i]), "recall": float(r[i]), "f1-score": float(f[i]), "support": float(n_true[i])}
           for i, name in enumerate(names)}
    support = float(np.sum(n_true))
    out["accuracy"] = float(div(tp.sum(), n_pred.sum()))
    out["macro avg"] = {"precision": float(np.average(p)), "recall": float(np.average(r)), "f1-score": float(np.average(f)),
                        "support": support}
    out["weighted avg"] = {"precision": float(np.average(p, weights=n_true)), "recall": float(np.average(r, weights=n_true)),
                           "f1-score": float(np.average(f, weights=n_true)), "support": support}
    return out


def score_classifications(instances, annotations, aopc_thresholds):
    """``metrics.py score_classifications`` (``:284-364``) on result dicts (one per annotation)."""
    labels = list(set(a.classification for a in annotations))
    label_to_int = {l: i for i, l in enumerate(labels)}
    by_id = {inst["annotation_id"]: inst for inst in instances}
    truth = [label_to_int[a.classification] for a in annotations]
    pred = [label_to_int[by_id[a.annotation_id]["classification"]] for a in annotations]
    comp, suff = "comprehensiveness_classification_scores", "sufficiency_classification_scores"

    def drop(key):
        return [x["classification_scores"][x["classification"]] - x[key][x["classification"]] for x in instances]

    def ent(key):
        return [entropy(list(x["classification_scores"].values())) - entropy(list(x[key].values())) for x in instances]

    def kl(key):
        out = []
        for x in instances:
            keys = list(x["classification_scores"].keys())
            out.append(entropy([x[key][k] for k in keys], [x["classification_scores"][k] for k in keys]))
        return out

    def aopc(key):
        rows = []
        for inst in instances:
            kls = inst["classification"]
            beta_0 = inst["classification_scores"][kls]
            rows.append([beta_0 - s[key][kls] for s in sorted(inst["thresholded_scores"], key=lambda x: x["threshold"])
                         if s["threshold"] in aopc_thresholds])
            assert len(rows[-1]) == len(aopc_thresholds)
        rows = np.array(rows)
        return np.average(rows), np.average(rows, axis=0).tolist()
    c_aopc, c_points = aopc(comp)
    s_aopc, s_points = aopc(suff)
    return {"accuracy": float(np.average(np.asarray(truth) == np.asarray(pred))),
            "prf": class_report(truth, pred, labels),
            "comprehensiveness": np.average(drop(comp)), "sufficiency": np.average(drop(suff)),
            "comprehensiveness_entropy": np.average(ent(comp)), "comprehensiveness_kl": np.average(kl(comp)),
            "sufficiency_entropy": np.average(ent(suff)), "sufficiency_kl": np.average(kl(suff)),
            "aopc_thresholds": aopc_thresholds, "comprehensiveness_aopc": c_aopc,
            "comprehensiveness_aopc_points": c_points, "sufficiency_aopc": s_aopc, "sufficiency_aopc_points": s_points}
