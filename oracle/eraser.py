"""ERASER rationale-evaluation oracle (TEST INFRASTRUCTURE, numpy / plain Python).

Restates, from the token map of one document on:

* ``pool_words``      ``bert_pipeline.py:96-138`` (``scores_per_word_from_scores_per_token``): one score per character of the
                      ``##``-stripped, special-token-free piece stream, then the max over each word's characters (np.max:
                      NaN propagates); words that start past the stream are dropped
* ``word_order``      the ranking ``te_eraser_rationales`` documents: NaN first, descending score, ascending word index
                      (-0 == +0); with distinct scores the order of ``cam.topk(k)`` (``:567-569``)
* ``doc_counts``      per k (n_pred, tok_hits, span_hits, iou_hits per threshold) of the first min(k, W) words, from sets
* ``prediction_lines`` / ``hard_scores``  the ``identifier_results_{k}.json`` lines (``:566-582``) and the dict that
                      ``metrics.py main()`` builds for hard predictions: ``partial_match_score`` (``:111-166``) and
                      ``score_hard_rationale_predictions`` (``:168-215``) at span and token level (``:628-640``), on tuples
                      (annotation_id, docid, start, end) that hash like the reference's ``Rationale``, so every key set
                      iterates in the reference's order
"""
import json

import numpy as np

SPECIAL = ("[CLS]", "[SEP]", "[UNK]", "[PAD]")


def pool_words(words, pieces, scores):
    """Per-word scores (float32) of the token scores [T] (already clamped), or ValueError on misalignment."""
    stream, per_char = [], []
    for p, s in zip((p.replace("##", "") for p in pieces), scores):
        if p in SPECIAL:
            continue
        stream.extend(p)
        per_char.extend([s] * len(p))
    out, seen = [], []
    pos = 0
    for w in words:
        if pos >= len(per_char):
            break
        out.append(np.max(np.asarray(per_char[pos:pos + len(w)], dtype=np.float32)))
        seen.append("".join(stream[pos:pos + len(w)]))
        pos += len(w)
    if seen[:-1] != list(words[:len(seen) - 1]):
        raise ValueError("pieces do not align with the words")
    return np.asarray(out, dtype=np.float32)


def word_order(scores):
    """Word indices ranked NaN first, then by descending score, then by ascending index."""
    s = np.asarray(scores, dtype=np.float32).astype(np.float64)
    nan = np.isnan(s)
    s = np.where(nan, 0.0, s) + 0.0                        # -0 -> +0
    return np.lexsort((np.arange(len(s)), -s, ~nan)).astype(np.int64)


def doc_counts(order, spans, ks, thresholds):
    """[len(ks), 3 + len(thresholds)] int64 for one document: the first min(k, W) ranked words against its truth spans
    [(start, end)] (end exclusive)."""
    spans = sorted(set((int(a), int(b)) for a, b in spans))
    out = np.zeros((len(ks), 3 + len(thresholds)), dtype=np.int64)
    for i, k in enumerate(ks):
        pred = [int(w) for w in order[:min(k, len(order))]]
        out[i, 0] = len(pred)
        out[i, 1] = sum(any(a <= w < b for a, b in spans) for w in pred)
        out[i, 2] = sum((w, w + 1) in spans for w in pred)
        for t, thr in enumerate(thresholds):
            out[i, 3 + t] = sum(max([1.0 / (b - a) for a, b in spans if a <= w < b] or [0.0]) >= thr for w in pred)
    return out


def prediction_lines(docids, per_doc_topk):
    """{position of k: [line]}: per document the accumulated ``hard_rationale_predictions`` (per_doc_topk[d][i] = the
    word indices of the i-th k, in order)."""
    out = {}
    for d, per_k in zip(docids, per_doc_topk):
        hard = []
        for i, idx in enumerate(per_k):
            hard.extend({"start_token": int(w), "end_token": int(w) + 1} for w in idx)
            out.setdefault(i, []).append(json.dumps({"annotation_id": d, "rationales": [{"docid": d,
                                                                                       "hard_rationale_predictions": list(hard)}]}))
    return out


def truth_tuples(annotations):
    """``Rationale.from_annotation`` of every annotation, in order (annotations as ``eraser.Annotation``)."""
    return [(a.annotation_id, ev.docid, ev.start_token, ev.end_token) for a in annotations for g in a.evidences for ev in g]


def pred_tuples(lines):
    """``Rationale.from_instance`` of every line, in order."""
    out = []
    for line in lines:
        inst = json.loads(line)
        for rat in inst["rationales"]:
            for p in rat.get("hard_rationale_predictions", []):
                out.append((inst["annotation_id"], rat["docid"], p["start_token"], p["end_token"]))
    return out


def _by_key(tuples):
    keyed = {}
    for t in tuples:
        keyed.setdefault(t[:2], set()).add(t)
    return keyed


def _f1(p, r):
    if p == 0 or r == 0:
        return 0
    return 2 * p * r / (p + r)


def _tokens(tuples):
    return [(a, d, t, t + 1) for a, d, s, e in tuples for t in range(s, e)]


def prf(truth, pred):
    """Instance micro / macro precision, recall and F1 of two lists of tuples (``metrics.py:168-215``)."""
    truth, pred = set(truth), set(pred)
    both = len(truth & pred)
    res = {"instance_micro": {"p": both / len(pred), "r": both / len(truth)}}
    res["instance_micro"]["f1"] = _f1(res["instance_micro"]["p"], res["instance_micro"]["r"])
    tk, pk = _by_key(truth), _by_key(pred)
    per = []
    for k in set(tk.keys()) | pk.keys():
        t, p = tk.get(k, set()), pk.get(k, set())
        prec = len(t & p) / len(p) if p else 0
        rec = len(t & p) / len(t) if t else 0
        per.append((prec, rec, _f1(prec, rec)))
    res["instance_macro"] = {n: sum(x[j] for x in per) / len(per) for j, n in enumerate(("p", "r", "f1"))}
    return res


def iou_scores(truth, pred, thresholds):
    """Partial-match precision / recall / F1 at each IoU threshold (``metrics.py:111-166``)."""
    tk, pk = _by_key(truth), _by_key(pred)
    best = {}
    for k in set(tk.keys()) | set(pk.keys()):
        for p in pk.get(k, []):
            b = 0.0
            for t in tk.get(k, []):
                ps, ts = set(range(p[2], p[3])), set(range(t[2], t[3]))
                u = len(ps | ts)
                iou = 0 if u == 0 else len(ps & ts) / u
                b = iou if iou > b else b
            best.setdefault(k, {})[p] = b
    n_truth = {k: len(v) for k, v in tk.items()}
    n_pred = {k: len(v) for k, v in pk.items()}
    out = []
    for thr in thresholds:
        tps = {k: sum(int(x >= thr) for x in v.values()) for k, v in best.items()}
        hit = sum(tps.values())
        r = hit / sum(n_truth.values()) if sum(n_truth.values()) > 0 else 0
        p = hit / sum(n_pred.values()) if sum(n_pred.values()) > 0 else 0
        rs = [tps.get(k, 0.0) / n if n > 0 else 0 for k, n in n_truth.items()]
        ps = [tps.get(k, 0.0) / n if n > 0 else 0 for k, n in n_pred.items()]
        mr = sum(rs) / len(rs) if rs else 0
        mp = sum(ps) / len(ps) if ps else 0
        out.append({"threshold": thr, "micro": {"p": p, "r": r, "f1": _f1(r, p)},
                    "macro": {"p": mp, "r": mr, "f1": _f1(mr, mp)}})
    return out


def hard_scores(annotations, lines, thresholds=(0.5,)):
    """The hard-prediction part of ``metrics.py main()`` (``:628-640``) for the truth of ``annotations`` and the lines of
    one ``identifier_results_{k}.json``."""
    truth, pred = truth_tuples(annotations), pred_tuples(lines)
    return {"iou_scores": iou_scores(truth, pred, list(thresholds)), "rationale_prf": prf(truth, pred),
            "token_prf": prf(_tokens(truth), _tokens(pred))}
