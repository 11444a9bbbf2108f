"""Generate ``tests/golden/eraser_faithfulness.npz`` from ``tests/golden/eraser.npz`` and the UNMODIFIED reference's models
and ``metrics.py`` on CPU (authoring container).

    python -m oracle.make_golden_eraser_faithfulness     # from the repo root, needs /root/reference, transformers, sklearn

TEST INFRASTRUCTURE.  The reference pipeline never fills the faithfulness fields (``pipeline_utils.py:540-541`` is a TODO),
so the reduced inputs follow the project's definitions (DESIGN.md §1), restated in ``oracle/eraser_faithfulness.py``;
everything they feed is the reference's own:
 * the vocabulary, documents, annotations, tiny BERT and per-method word scores (the reference's pooling of the
   reference's maps) are those of ``eraser.npz``;
 * for each method the words are ranked by those scores, and the comprehensiveness / sufficiency rows of every
   selection (the default k fraction, then ``metrics.py``'s AOPC bins) are built with ``oracle.eraser_faithfulness``;
 * every original and reduced row runs at batch 1 through the reference's own ``BertForSequenceClassification``
   (``transformer_attribution``) or ``BERT_cls_lrp`` (the other five) in fp32 and fp64; the fp32 softmax gives the
   result lines, which ``metrics.py``'s ``score_classifications`` scores;
 * a hand-built instance set reaches the corners of ``score_classifications``: three classes, one never predicted
   (sklearn's zero-division path), probabilities with exact zeros (an infinite KL divergence) and an annotation id that
   differs from its docid.
The label order of ``score_classifications`` follows the hash seed, so the script re-runs itself with PYTHONHASHSEED=0.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                     # noqa: E402
from oracle import eraser_faithfulness as of             # noqa: E402
from oracle.make_golden_eraser import CLASSES, METHODS, build, params   # noqa: E402

SRC = os.path.join(ROOT, "tests", "golden", "eraser.npz")
OUT = os.path.join(ROOT, "tests", "golden", "eraser_faithfulness.npz")
AOPC = [0.01, 0.05, 0.1, 0.2, 0.5]


def corner_set():
    """(annotation lines, result lines): three classes, 'c' never predicted, exact zeros, an id that is not its docid."""
    g = np.random.default_rng(7)
    classes = ("a", "b", "c")
    anns, insts = [], []
    for i in range(9):
        doc = "cdoc%d" % i
        ann_id = doc + ".q" if i == 4 else doc
        anns.append(json.dumps({"annotation_id": ann_id, "query": "q", "classification": classes[i % 3], "query_type": None,
                                "evidences": [[{"text": "x", "docid": doc, "start_token": 0, "end_token": 1,
                                                "start_sentence": -1, "end_sentence": -1}]]}))

        def dist(zero=None):
            p = g.random(3).astype(np.float32)
            if zero is not None:
                p[zero] = 0
            return {c: float(v) for c, v in zip(classes, (p / p.sum()).astype(np.float32))}
        orig = dist(zero=2 if i % 2 else None)
        pred = "a" if orig["a"] >= orig["b"] else "b"
        inst = {"annotation_id": ann_id, "rationales": [{"docid": doc, "hard_rationale_predictions": [
                    {"start_token": 0, "end_token": 1}]}],
                "classification": pred, "classification_scores": orig,
                "comprehensiveness_classification_scores": dist(), "sufficiency_classification_scores": dist(zero=0),
                "thresholded_scores": [{"threshold": t, "comprehensiveness_classification_scores": dist(zero=1),
                                        "sufficiency_classification_scores": dist()} for t in AOPC[::-1]]}
        insts.append(json.dumps(inst))
    return anns, insts


def forward_probs(model, rows, dtype):
    """Softmax probabilities of each id list at batch 1 through the reference model (fp32 or fp64)."""
    out = []
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        for r in rows:                                  # the reference's forward registers gradient hooks
            ids = torch.tensor([r], dtype=torch.long)
            logits = model(input_ids=ids, attention_mask=torch.ones_like(ids))[0].detach()
            out.append((torch.softmax(logits, dim=-1)[0], logits[0]))
    finally:
        torch.set_default_dtype(prev)
    return out


def run():
    import scipy
    import sklearn
    from transformer_explainability_b200 import eraser as te
    src = np.load(SRC)
    docids = [str(d) for d in src["docids"]]
    docs = {d: str(t) for d, t in zip(docids, src["docs"])}
    ann_lines = [str(a) for a in src["annotations"]]
    out = {"sklearn": np.array(sklearn.__version__), "scipy": np.array(scipy.__version__),
           "hashseed": np.array(os.environ["PYTHONHASHSEED"]), "aopc_thresholds": np.array(AOPC)}
    corner_anns, corner_insts = corner_set()
    out["corner.annotations"] = np.array(corner_anns)
    out["corner.instances"] = np.array(corner_insts)
    rh._prepare_bert_imports()
    p = params()
    with tempfile.TemporaryDirectory() as tmp:
        for name, lines in (("test", ann_lines), ("corner", corner_anns)):
            with open(os.path.join(tmp, name + ".jsonl"), "w") as f:
                f.write("".join(line + "\n" for line in lines))
        with rh._ref_imports():
            from BERT_rationale_benchmark import metrics as rmetrics
            from BERT_rationale_benchmark import utils as rutils
            test = rutils.annotations_from_jsonl(os.path.join(tmp, "test.jsonl"))
            corner = rutils.annotations_from_jsonl(os.path.join(tmp, "corner.jsonl"))
            out["corner.scores"] = np.array(json.dumps(rmetrics.score_classifications(
                [json.loads(l) for l in corner_insts], corner, {}, AOPC)))
            doc_of = [next(iter(a.evidences))[0].docid for a in test]
            ids = {d: [int(i) for i in src["ids." + d]] for d in docids}
            ranges = {d: te.word_piece_ranges(docs[d].split(), [str(x) for x in src["pieces." + d]]) for d in docids}
            # the default k fraction: mean over documents of (words < W inside a truth span) / W
            fr = []
            for a, d in zip(test, doc_of):
                W = len(ranges[d])
                cov = set(t for grp in a.evidences for ev in grp if ev.docid == d
                          for t in range(ev.start_token, min(ev.end_token, W)))
                fr.append(len(cov) / W)
            fracs = [sum(fr) / len(fr)] + AOPC
            out["fractions"] = np.array(fracs)
            J = len(fracs)
            S = max(len(v) for v in ids.values())
            for method, kind, _, _ in METHODS:
                model32 = build(kind, p)
                model64 = build(kind, {k: v.double() for k, v in p.items()}).double()
                nsel = np.zeros((len(test), J), dtype=np.int64)
                red_ids = np.zeros((len(test), J, 2, S), dtype=np.int64)
                red_len = np.zeros((len(test), J, 2), dtype=np.int64)
                rows = []
                for i, d in enumerate(doc_of):
                    words = src["%s.words.%s" % (method, d)]
                    nsel[i] = of.select_counts(fracs, len(words))
                    rows.append(ids[d])
                    for j, n in enumerate(nsel[i]):
                        for t, r in enumerate(of.reduce_rows(ids[d], ranges[d], words, int(n))):
                            red_ids[i, j, t, :len(r)] = r
                            red_len[i, j, t] = len(r)
                            rows.append(r)
                res = {}
                for dt, tag, model in ((torch.float32, "f32", model32), (torch.float64, "f64", model64)):
                    pr = forward_probs(model, rows, dt)
                    probs = np.stack([q.numpy() for q, _ in pr]).reshape(len(test), 1 + 2 * J, -1)
                    logits = np.stack([lg.numpy() for _, lg in pr]).reshape(len(test), 1 + 2 * J, -1)
                    out["%s.probs_%s" % (method, tag)] = probs[:, 0]
                    out["%s.red_probs_%s" % (method, tag)] = probs[:, 1:].reshape(len(test), J, 2, -1)
                    out["%s.logits_%s" % (method, tag)] = logits[:, 0]
                    res[tag] = probs
                probs = res["f32"]
                lines = []
                for i, (a, d) in enumerate(zip(test, doc_of)):
                    pred = int(np.argmax(out["%s.logits_f32" % method][i]))
                    sc = lambda v: {c: float(x) for c, x in zip(CLASSES, v)}          # noqa: E731
                    order = of.word_order(src["%s.words.%s" % (method, d)])[:int(nsel[i, 0])]
                    lines.append({"annotation_id": a.annotation_id,
                                  "rationales": [{"docid": d, "hard_rationale_predictions": [
                                      {"start_token": int(w), "end_token": int(w) + 1} for w in order]}],
                                  "classification": CLASSES[pred], "classification_scores": sc(probs[i, 0]),
                                  "comprehensiveness_classification_scores": sc(probs[i, 1]),
                                  "sufficiency_classification_scores": sc(probs[i, 2]),
                                  "thresholded_scores": [{"threshold": t,
                                                          "comprehensiveness_classification_scores": sc(probs[i, 1 + 2 * j]),
                                                          "sufficiency_classification_scores": sc(probs[i, 2 + 2 * j])}
                                                         for j, t in enumerate(fracs) if j > 0]})
                out["%s.n_select" % method] = nsel
                out["%s.red_ids" % method] = red_ids
                out["%s.red_len" % method] = red_len
                out["%s.lines" % method] = np.array([json.dumps(l) for l in lines])
                scores = rmetrics.score_classifications(lines, test, {}, AOPC)
                out["%s.scores" % method] = np.array(json.dumps(scores))
                print(method, "comprehensiveness %.4f sufficiency %.4f aopc %.4f / %.4f" % (
                    scores["comprehensiveness"], scores["sufficiency"], scores["comprehensiveness_aopc"],
                    scores["sufficiency_aopc"]))
    np.savez_compressed(OUT, **out)
    print("eraser_faithfulness.npz", len(out), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if os.environ.get("PYTHONHASHSEED") != "0":
        sys.exit(subprocess.call([sys.executable, "-m", "oracle.make_golden_eraser_faithfulness"], cwd=ROOT,
                                 env=dict(os.environ, PYTHONHASHSEED="0")))
    torch.set_num_threads(os.cpu_count())
    run()
