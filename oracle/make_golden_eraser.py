"""Generate ``tests/golden/eraser.npz`` by running the UNMODIFIED reference's ERASER pieces on CPU (authoring container).

    python -m oracle.make_golden_eraser          # from the repo root, needs /root/reference, transformers and sklearn

TEST INFRASTRUCTURE.  The pipeline's ``main()`` trains a classifier before it explains, so its test loop
(``bert_pipeline.py:456-582``) is restated here around the reference's own functions:
 * documents are interned with a real ``BertTokenizer`` (called with the pipeline's ``encode_plus`` arguments,
   ``:262-271``; transformers 5 keeps only the call) on a
   seeded synthetic vocabulary of 100 entries (the tiny golden BERT's vocabulary size) with ``##`` pieces;
 * each annotation is explained for its gold class with the six ``Generator`` methods the pipeline compares (``:437-448``)
   on the tiny BERT of ``bert_tiny.npz`` (3 layers, ``max_length`` 32): ``generate_LRP`` on
   ``BertForSequenceClassification``, the other five on ``BERT_cls_lrp``.  ``generate_LRP`` runs with start_layer 2, the
   last layer, which is what the pipeline's default 11 is at BERT-base depth (11 is out of range at depth 3);
 * the clamped map goes through the reference's ``scores_per_word_from_scores_per_token``; the top-k is ``cam.topk(k)``
   with k clipped to the number of words (the reference's ``topk`` raises past it; the engine clips the same way);
 * ``metrics.py``'s ``partial_match_score`` and ``score_hard_rationale_predictions`` score the lines, with the truth read
   by the reference's ``annotations_from_jsonl`` from a data directory written here.
The metric dicts depend on Python's set iteration order, so the script re-runs itself with PYTHONHASHSEED=0; the tests
compare against them under the same seed.

Cases: document 0 has 3 words (every k above W), the longer ones are truncated at 32 pieces with evidence past the
truncation, spans overlap and repeat, several are single words, and annotation 5's id differs from its docid, so its truth
key never meets a prediction and its document's predictions have no truth.
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

from oracle import ref_harness as rh         # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "eraser.npz")
SEED = 41
MAX_LENGTH = 32
KS = tuple(range(5, 85, 5))
THRESHOLDS = (0.5, 0.25, 1.0)
CLASSES = ("NEG", "POS")
# (method, model, Generator method, kwargs)
METHODS = (("transformer_attribution", "ours", "LRP", dict(start_layer=2)),
           ("partial_lrp", "cls_lrp", "LRP_last_layer", {}),
           ("last_attn", "cls_lrp", "attn_last_layer", {}),
           ("attn_gradcam", "cls_lrp", "attn_gradcam", {}),
           ("lrp", "cls_lrp", "full_lrp", {}),
           ("rollout", "cls_lrp", "rollout", {}))
WORDS_PER_DOC = (3, 6, 12, 25, 40, 9, 30, 18)
NO_MATCH = 5                                  # annotation whose id differs from its docid


def vocabulary():
    """100 entries: the five specials, '.', ',', the 26 letters as words and as '##' pieces, and 41 seeded multi-letter
    words / pieces (so every lower-case word tokenises without [UNK])."""
    g = np.random.default_rng(SEED)
    letters = [chr(c) for c in range(ord("a"), ord("z") + 1)]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", ".", ","] + letters + ["##" + c for c in letters]
    while len(vocab) < 100:
        w = "".join(g.choice(letters, size=int(g.integers(2, 5))))
        w = w if g.random() < 0.5 else "##" + w
        if w not in vocab:
            vocab.append(w)
    return vocab


def documents(vocab):
    g = np.random.default_rng(SEED + 1)
    whole = [v for v in vocab[7:] if not v.startswith("##")]
    pieces = [v[2:] for v in vocab if v.startswith("##")]
    docs = {}
    for i, n in enumerate(WORDS_PER_DOC):
        words = []
        for _ in range(n):
            w = str(g.choice(whole)) + "".join(g.choice(pieces, size=int(g.integers(0, 3))))
            if g.random() < 0.1:
                w += "."
            words.append(w)
        docs["doc%d.txt" % i] = " ".join(words) + "\n"
    return docs


def annotations(docs):
    """The split as JSON lines (``utils.annotations_to_jsonl`` fields)."""
    g = np.random.default_rng(SEED + 2)
    lines = []
    for i, (d, text) in enumerate(sorted(docs.items())):
        n = len(text.split())
        spans = []
        for _ in range(int(g.integers(2, 5))):
            s = int(g.integers(0, n))
            spans.append((s, min(n, s + int(g.integers(1, 4)))))
        spans.append((int(g.integers(0, n)),) * 2)
        spans[-1] = (spans[-1][0], spans[-1][0] + 1)                    # a single word
        spans.append(spans[0])                                           # a repeated span
        if n > 20:
            spans.append((n - 3, n))                                     # past the truncation
        ann_id = d + ".other" if i == NO_MATCH else d
        ev = [[{"text": " ".join(text.split()[s:e]), "docid": d, "start_token": s, "end_token": e,
                "start_sentence": -1, "end_sentence": -1}] for s, e in spans]
        lines.append(json.dumps({"annotation_id": ann_id, "query": "what is the sentiment?", "evidences": ev,
                                 "classification": CLASSES[int(g.integers(0, 2))], "query_type": None}))
    return lines


def params():
    z = np.load(os.path.join(ROOT, "tests", "golden", "bert_tiny.npz"))
    return {k[len("param."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("param.")}


def build(kind, p):
    if kind == "ours":
        from oracle.make_golden import BERT_TINY
        model = rh.build_bert(seed=3, **BERT_TINY)
        res = model.load_state_dict(p, strict=False)
        assert not res.unexpected_keys
        return model
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import bert_lrp_oracle as olrp
    return olrp._build_ref_cls_lrp(p, torch.float32)


def run():
    from transformers import BertTokenizer
    vocab = vocabulary()
    docs = documents(vocab)
    ann_lines = annotations(docs)
    out = {"vocab": np.array(vocab), "docids": np.array(sorted(docs)), "docs": np.array([docs[d] for d in sorted(docs)]),
           "annotations": np.array(ann_lines), "ks": np.array(KS), "thresholds": np.array(THRESHOLDS),
           "max_length": np.int64(MAX_LENGTH), "hashseed": np.array(os.environ["PYTHONHASHSEED"])}
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "vocab.txt"), "w") as f:
            f.write("".join(v + "\n" for v in vocab))
        tok = BertTokenizer(os.path.join(tmp, "vocab.txt"), do_lower_case=True)
        os.makedirs(os.path.join(tmp, "docs"))
        for d, text in docs.items():
            with open(os.path.join(tmp, "docs", d), "w") as f:
                f.write(text)
        with open(os.path.join(tmp, "test.jsonl"), "w") as f:
            f.write("".join(line + "\n" for line in ann_lines))
        rh._prepare_bert_imports()
        with rh._ref_imports():
            from BERT_rationale_benchmark import utils as rutils
            from BERT_rationale_benchmark import metrics as rmetrics
            from BERT_rationale_benchmark.models.pipeline import bert_pipeline as rpipe
            test = rutils.annotations_from_jsonl(os.path.join(tmp, "test.jsonl"))
            texts = rutils.load_documents(tmp, set(docs))
            enc = {d: tok(texts[d], add_special_tokens=True, max_length=MAX_LENGTH,
                                      return_token_type_ids=False, padding=False, return_attention_mask=True,
                                      return_tensors="pt", truncation=True) for d in texts}
            for d in sorted(docs):
                ids = enc[d]["input_ids"][0]
                out["ids." + d] = ids.numpy().astype(np.int64)
                out["pieces." + d] = np.array(tok.convert_ids_to_tokens(ids))
            p = params()
            truth = list(rpipe.chain.from_iterable(rmetrics.Rationale.from_annotation(a) for a in test))
            classes = {c: i for i, c in enumerate(CLASSES)}
            for name, kind, which, kw in METHODS:
                model = build(kind, p)
                files = {k: [] for k in KS}
                for a in test:
                    d = rpipe.extract_docid_from_dataset_element(a)
                    ids = enc[d]["input_ids"]
                    mask = enc[d]["attention_mask"]
                    target = classes[a.classification]
                    cam = rh.bert_generate(model, ids, mask, which, index=target, **kw)[0]
                    out["%s.map.%s" % (name, d)] = cam.numpy()
                    cam = cam.clamp(min=0)
                    words = rpipe.scores_per_word_from_scores_per_token(texts[d].split(), tok, ids[0], cam)
                    out["%s.words.%s" % (name, d)] = words.numpy()
                    hard = []
                    for k in KS:
                        _, idx = words.topk(k=min(k, len(words)))
                        hard.extend({"start_token": i, "end_token": i + 1} for i in idx.tolist())
                        files[k].append(json.dumps({"annotation_id": d, "rationales": [
                            {"docid": d, "hard_rationale_predictions": list(hard)}]}))
                for k in KS:
                    out["%s.lines.%d" % (name, k)] = np.array(files[k])
                    pred = list(rpipe.chain.from_iterable(rmetrics.Rationale.from_instance(json.loads(l)) for l in files[k]))
                    scores = {"iou_scores": rmetrics.partial_match_score(truth, pred, list(THRESHOLDS)),
                              "rationale_prf": rmetrics.score_hard_rationale_predictions(truth, pred)}
                    tt = list(rpipe.chain.from_iterable(r.to_token_level() for r in truth))
                    tp = list(rpipe.chain.from_iterable(r.to_token_level() for r in pred))
                    scores["token_prf"] = rmetrics.score_hard_rationale_predictions(tt, tp)
                    out["%s.scores.%d" % (name, k)] = np.array(json.dumps(scores))
                print(name, "token F1 @5 / @80:", json.loads(str(out["%s.scores.5" % name]))["token_prf"]["instance_micro"]["f1"],
                      json.loads(str(out["%s.scores.80" % name]))["token_prf"]["instance_micro"]["f1"])
    np.savez_compressed(OUT, **out)
    print("eraser.npz", len(out), "arrays,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if os.environ.get("PYTHONHASHSEED") != "0":
        sys.exit(subprocess.call([sys.executable, "-m", "oracle.make_golden_eraser"], cwd=ROOT,
                                 env=dict(os.environ, PYTHONHASHSEED="0")))
    torch.set_num_threads(os.cpu_count())
    run()
