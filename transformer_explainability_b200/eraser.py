"""ERASER rationale evaluation of the BERT explanation methods (``BERT_rationale_benchmark/models/pipeline/bert_pipeline.py``
``:96-138, 260-273, 456-582`` and ``BERT_rationale_benchmark/metrics.py``): token-level F1 of each method's top-k words
against the human rationales, for k = 5, 10, ..., 80.

The reference explains one document at a time (``test_batch_size = 1``), clamps the scores at zero, pools word-piece scores
to words (``scores_per_word_from_scores_per_token``), takes the top-k words for each k and appends one JSON line per document
to ``identifier_results_{k}.json``; ``metrics.py`` then scores the files.  Here, per batch of length-sorted documents, one
engine call makes the maps, one ``te_eraser_rationales`` call pools them to words, ranks the words and counts the hits of
every k against the truth spans, and one small device-to-host copy brings back the order and the counts.  The files keep the
reference's format, including its quirk that ``hard_rationale_predictions`` is never reset between the k's of a document
(the k = 10 line holds the top-5 words followed by the top-10 words, ``:566-582``), and ``metrics.py``'s hard-prediction
scores (``token_prf``, ``rationale_prf``, ``iou_scores``) are computed on the host from the counts with its Python float
arithmetic and its key sets.

    python -m transformer_explainability_b200.eraser --data_dir movies --output_dir out --model_params movies_bert.json \\
        --method transformer_attribution

Deviations from the reference (DESIGN.md §1):
 * ties: the reference calls ``cam.topk(k)`` for each k and may pick different tied words for different k; here one order
   (NaN first, descending score, ascending word index) serves every k, so the lines nest.  With distinct scores the two agree;
 * short documents: for k > W (the number of words) the reference's ``topk`` raises; here k is clipped to W;
 * batches larger than 1: padding changes a real token's map only by rounding; ``generate_LRP`` sets the ``[CLS]`` entry to
   the row minimum, which sees the padded zeros, and pooling never reads that entry.  ``generate_attn_gradcam`` averages
   the gradients and min-max normalises over the whole [S, S] map, padded query rows included, so its batches only hold
   documents of one length;
 * one annotation per document and split (the pipeline keys its predictions by docid: two annotations of one document would
   merge into one key), and every annotation needs an evidence; otherwise ``ValueError``;
 * soft-token metrics (AUPRC, AP) are not computed.
"""
import argparse
import json
import os
from dataclasses import dataclass
from typing import FrozenSet, Optional, Tuple, Union

import numpy as np
import torch

KS = tuple(range(5, 85, 5))
SPECIAL_PIECES = ("[CLS]", "[SEP]", "[UNK]", "[PAD]")
METHODS = ("transformer_attribution", "partial_lrp", "last_attn", "attn_gradcam", "lrp", "rollout")
METHOD_FOLDER = {"transformer_attribution": "ours", "partial_lrp": "partial_lrp", "last_attn": "last_attn",
                 "attn_gradcam": "attn_gradcam", "lrp": "lrp", "rollout": "rollout"}
# method -> (model: "ours" = BertForSequenceClassification, "cls_lrp" = BERT_cls_lrp; Generator method)   (:437-448)
METHOD_GENERATOR = {"transformer_attribution": ("ours", "generate_LRP"),
                    "partial_lrp": ("cls_lrp", "generate_LRP_last_layer"),
                    "last_attn": ("cls_lrp", "generate_attn_last_layer"),
                    "attn_gradcam": ("cls_lrp", "generate_attn_gradcam"),
                    "lrp": ("cls_lrp", "generate_full_lrp"),
                    "rollout": ("cls_lrp", "generate_rollout")}


def topk_rationales(scores, ks=KS):
    """scores [B,T] (GPU or CPU) -> list (per document) of list (per k) of index lists, ``cam.topk(k)`` order."""
    scores = scores.clamp(min=0)
    kmax = min(max(ks), scores.shape[1])
    idx = scores.topk(kmax, dim=1).indices.cpu()
    return [[idx[b, :min(k, kmax)].tolist() for k in ks] for b in range(scores.shape[0])]


def rationale_lines(doc_ids, scores=None, ks=KS, order=None):
    """One JSON string per (k, document) in the reference's accumulation order: returns {k: [line, ...]}.  The words of
    each k come from ``topk_rationales(scores)``, or with ``order`` (per document a ranked list of word indices, as
    ``te_eraser_rationales`` returns it; -1 entries are ignored) from its first k entries."""
    if order is None:
        per_doc = topk_rationales(scores, ks)
    else:
        per_doc = []
        for o in order:
            o = [int(i) for i in o if int(i) >= 0]
            per_doc.append([o[:k] for k in ks])
    out = {k: [] for k in ks}
    for doc, per_k in zip(doc_ids, per_doc):
        hard = []
        for k, indices in zip(ks, per_k):
            hard.extend({"start_token": i, "end_token": i + 1} for i in indices)
            out[k].append(json.dumps({"annotation_id": doc,
                                      "rationales": [{"docid": doc, "hard_rationale_predictions": list(hard)}]}))
    return out


def write_identifier_results(generator, input_ids, attention_mask, targets, doc_ids, output_dir, method="generate_LRP",
                             folder="ours", word_scores=None, ks=KS, **kw):
    """Explain a batch for its target classes with ``getattr(generator, method)`` and append to
    ``output_dir/folder/identifier_results_{k}.json``.  Returns the [B,T] scores."""
    scores = getattr(generator, method)(input_ids, attention_mask, index=targets, **kw)
    if word_scores is not None:
        scores = word_scores(scores)
    os.makedirs(os.path.join(output_dir, folder), exist_ok=True)
    for k, lines in rationale_lines(doc_ids, scores, ks).items():
        with open(os.path.join(output_dir, folder, "identifier_results_%d.json" % k), "a") as f:
            f.write("".join(line + "\n" for line in lines))
    return scores


# ---- data (BERT_rationale_benchmark/utils.py) ----------------------------------------------------------------------------
# The two records have the reference's fields in the reference's order: a frozen dataclass hashes as the tuple of its
# fields, so the evidence sets iterate in the reference's order, and so do the metric key sets built from them.
@dataclass(eq=True, frozen=True)
class Evidence:
    """One evidence span: ``(docid, start_token, end_token)`` words, end exclusive (``utils.py:9-26``)."""
    text: Union[str, Tuple[int], Tuple[str]]
    docid: str
    start_token: int = -1
    end_token: int = -1
    start_sentence: int = -1
    end_sentence: int = -1


@dataclass(eq=True, frozen=True)
class Annotation:
    """One annotation: ``evidences`` is a frozenset of evidence groups (tuples of ``Evidence``) (``utils.py:29-54``)."""
    annotation_id: str
    query: Union[str, Tuple[int]]
    evidences: FrozenSet[Tuple[Evidence]]
    classification: str
    query_type: Optional[str] = None
    docids: Optional[Tuple[str]] = None


def annotations_from_jsonl(path):
    """The annotations of one ``{split}.jsonl`` file, in file order (``utils.py:109-120``)."""
    out = []
    with open(path, "r") as f:
        for line in f:
            content = json.loads(line)
            content["evidences"] = frozenset(tuple(Evidence(**ev) for ev in group) for group in content["evidences"])
            out.append(Annotation(**content))
    return out


def load_split(data_dir, split="test"):
    return annotations_from_jsonl(os.path.join(data_dir, split + ".jsonl"))


def load_documents(data_dir, docids=None):
    """{docid: raw text} from ``docs.jsonl`` (every document in it) or from ``docs/<docid>`` (``utils.py:135-154, 205-223``)."""
    if os.path.exists(os.path.join(data_dir, "docs.jsonl")):
        if os.path.exists(os.path.join(data_dir, "docs")):
            raise ValueError("%s holds both docs.jsonl and docs/" % data_dir)
        with open(os.path.join(data_dir, "docs.jsonl"), "r") as f:
            return {d["docid"]: d["document"] for d in map(json.loads, f)}
    docs_dir = os.path.join(data_dir, "docs")
    docids = sorted(os.listdir(docs_dir)) if docids is None else sorted(set(str(d) for d in docids))
    out = {}
    for d in docids:
        with open(os.path.join(docs_dir, d), "r") as f:
            out[d] = f.read()
    return out


def annotation_docid(ann):
    """``extract_docid_from_dataset_element`` (``bert_pipeline.py:206-207``): the docid of the first evidence."""
    for group in ann.evidences:
        if group:
            return group[0].docid
        break
    raise ValueError("annotation %r has no evidence" % (ann.annotation_id,))


def truth_rationales(annotations):
    """``Rationale.from_annotation`` over the split (``metrics.py:43-49``): [(annotation_id, docid, start, end)]."""
    return [(ann.annotation_id, ev.docid, ev.start_token, ev.end_token)
            for ann in annotations for group in ann.evidences for ev in group]


# ---- tokenisation and the word map -----------------------------------------------------------------------------------------
def encode_documents(documents, tokenizer, max_length):
    """{docid: (input ids, word-piece strings)} as the pipeline interns them (``:262-271``: special tokens, truncation to
    ``max_length``, no padding).  ``tokenizer`` is any object with ``__call__`` and ``convert_ids_to_tokens`` in the manner
    of transformers' ``BertTokenizer``."""
    out = {}
    for d, doc in documents.items():
        ids = list(tokenizer(doc, add_special_tokens=True, max_length=max_length, truncation=True, padding=False,
                             return_attention_mask=False)["input_ids"])
        out[d] = (ids, list(tokenizer.convert_ids_to_tokens(ids)))
    return out


def word_piece_ranges(words, pieces):
    """Each word's inclusive word-piece range [first, last]: ``scores_per_word_from_scores_per_token``
    (``bert_pipeline.py:96-138``) as an index map.  The pieces, ``##`` stripped and ``[CLS]`` / ``[SEP]`` / ``[UNK]`` /
    ``[PAD]`` skipped, form one character stream; word i covers the next ``len(words[i])`` characters; words that start past
    the stream are dropped (truncation), and a word's score is the max over the pieces that overlap its characters.
    Raises ``ValueError`` where the reference's alignment check fails (every word but the last kept one must equal its
    characters; an ``[UNK]`` that swallowed characters breaks it), and when a piece that contributes no character lies
    inside a word's range."""
    piece_of_char, chars = [], []
    for i, p in enumerate(pieces):
        p = p.replace("##", "")
        if p in SPECIAL_PIECES:
            continue
        chars.extend(p)
        piece_of_char.extend([i] * len(p))
    ranges, got = [], []
    start = 0
    for w in words:
        if start >= len(chars):
            break
        end = start + len(w)
        seg = piece_of_char[start:end]
        ranges.append((seg[0], seg[-1]))
        got.append("".join(chars[start:end]))
        if len(set(seg)) != seg[-1] - seg[0] + 1:
            raise ValueError("word %d (%r): a piece without characters lies inside its piece range" % (len(ranges) - 1, w))
        start = end
    if got[:-1] != list(words[:len(got) - 1]):
        bad = next(i for i, (a, b) in enumerate(zip(got, words)) if a != b)
        raise ValueError("word pieces do not align with the document's words: word %d is %r, its characters are %r"
                         % (bad, words[bad], got[bad]))
    return ranges


# ---- metrics.py's hard-prediction scores from counts ----------------------------------------------------------------------
def _f1(p, r):
    return 0 if p == 0 or r == 0 else 2 * p * r / (p + r)


def _key_order(tuples):
    """The keys (first two fields) in the order the reference's ``_keyed_rationale_from_list`` meets them."""
    return dict.fromkeys(t[:2] for t in tuples)


class TruthIndex:
    """The truth side of ``metrics.py``'s hard-prediction scores for one split: per key (annotation_id, docid) the distinct
    spans and tokens, with the key orders of the reference's dicts and sets (all annotation data, host only)."""

    def __init__(self, annotations):
        spans = truth_rationales(annotations)
        span_set = set(spans)
        tokens = [(a, d, t, t + 1) for a, d, s, e in spans for t in range(s, e)]
        token_set = set(tokens)
        self.span_keys = {}                       # score_hard_rationale_predictions (spans): over set(truth)
        for t in span_set:
            self.span_keys[t[:2]] = self.span_keys.get(t[:2], 0) + 1
        self.token_keys = {}                      # ... (tokens)
        for t in token_set:
            self.token_keys[t[:2]] = self.token_keys.get(t[:2], 0) + 1
        self.iou_keys = {k: self.span_keys[k] for k in _key_order(spans)}      # partial_match_score: over the truth list
        self.n_spans = len(span_set)
        self.n_tokens = len(token_set)
        by_key = {}
        for a, d, s, e in spans:
            by_key.setdefault((a, d), set()).add((s, e))
        self.spans_by_key = {k: sorted(v) for k, v in by_key.items()}


def _prf(truth_keys, n_truth, pred_keys, pred_order):
    """``score_hard_rationale_predictions`` (``metrics.py:168-215``) from counts: truth_keys {key: distinct truth items},
    n_truth = their total; pred_keys {key: (n_pred, hits)} in the order of the prediction list; pred_order() -> the pred
    keys in the order of the reference's ``set(pred)`` iteration (only needed for keys without truth)."""
    hits = sum(h for _, h in pred_keys.values())
    n_pred = sum(n for n, _ in pred_keys.values())
    micro_p = hits / n_pred
    micro_r = hits / n_truth
    out = {"instance_micro": {"p": micro_p, "r": micro_r, "f1": _f1(micro_p, micro_r)}}
    pred_in_set_order = pred_order() if any(k not in truth_keys for k in pred_keys) else pred_keys
    per = {}
    for k in set(truth_keys.keys()) | dict.fromkeys(pred_in_set_order).keys():
        n, h = pred_keys.get(k, (0, 0))
        p = h / n if n > 0 else 0
        r = h / truth_keys[k] if truth_keys.get(k, 0) > 0 else 0
        per[k] = {"p": p, "r": r, "f1": _f1(p, r)}
    out["instance_macro"] = {"p": sum(i["p"] for i in per.values()) / len(per),
                             "r": sum(i["r"] for i in per.values()) / len(per),
                             "f1": sum(i["f1"] for i in per.values()) / len(per)}
    return out


def _iou_scores(truth_keys, pred_keys, thresholds):
    """``partial_match_score`` (``metrics.py:111-166``) from counts: truth_keys {key: distinct spans} in truth-list order,
    pred_keys {key: (n_pred, [hits per threshold])} in prediction-list order."""
    n_truth = sum(truth_keys.values())
    n_pred = sum(n for n, _ in pred_keys.values())
    out = []
    for t, threshold in enumerate(thresholds):
        tps = {k: h[t] for k, (_, h) in pred_keys.items()}
        micro_r = sum(tps.values()) / n_truth if n_truth > 0 else 0
        micro_p = sum(tps.values()) / n_pred if n_pred > 0 else 0
        rs = [tps.get(k, 0.0) / n if n > 0 else 0 for k, n in truth_keys.items()]
        ps = [tps.get(k, 0.0) / n if n > 0 else 0 for k, (n, _) in pred_keys.items()]
        macro_r = sum(rs) / len(rs) if rs else 0
        macro_p = sum(ps) / len(ps) if ps else 0
        out.append({"threshold": threshold, "micro": {"p": micro_p, "r": micro_r, "f1": _f1(micro_r, micro_p)},
                    "macro": {"p": macro_p, "r": macro_r, "f1": _f1(macro_r, macro_p)}})
    return out


def hard_scores(truth, docids, counts, orders, thresholds=(0.5,)):
    """The dict ``metrics.py main()`` builds for hard predictions (``iou_scores``, ``rationale_prf``, ``token_prf``) of one
    k.  truth: ``TruthIndex``; docids: the documents in file (dataset) order; counts [docs, 3 + len(thresholds)] =
    (n_pred, tok_hits, span_hits, iou_hits...) counted against the spans of the key (docid, docid), as
    ``te_eraser_rationales`` returns them; orders: per document its predicted word indices (used only to rebuild the
    reference's set order for predicted keys that have no truth)."""
    counts = np.asarray(counts, dtype=np.int64)
    span_pred, token_pred, iou_pred = {}, {}, {}
    for d, c in zip(docids, counts):
        n = int(c[0])
        if n == 0:                                 # no prediction: the key does not occur on the prediction side
            continue
        k = (d, d)
        span_pred[k] = (n, int(c[2]))
        token_pred[k] = (n, int(c[1]))
        iou_pred[k] = (n, [int(x) for x in c[3:]])

    def pred_order():
        keys = {}
        for t in set((d, d, int(w), int(w) + 1) for d, o, c in zip(docids, orders, counts) for w in list(o)[:int(c[0])]):
            keys[t[:2]] = None
        return keys
    return {"iou_scores": _iou_scores(truth.iou_keys, iou_pred, list(thresholds)),
            "rationale_prf": _prf(truth.span_keys, truth.n_spans, span_pred, pred_order),
            "token_prf": _prf(truth.token_keys, truth.n_tokens, token_pred, pred_order)}


# ---- the evaluation ---------------------------------------------------------------------------------------------------------
def eraser_eval(generator_method, documents, annotations, encodings, evidence_classes, batch_size=8, ks=KS,
                iou_thresholds=(0.5,), pad_id=0, device=None, same_length=None):
    """The test loop of the pipeline (``bert_pipeline.py:456-582``) and ``metrics.py``'s hard scores on the engine.

    generator_method: a bound ``Generator`` method (``generate_LRP`` keeps its ``start_layer = 11``), called as
    ``generator_method(input_ids=, attention_mask=, index=)`` for a padded batch; documents {docid: text};
    annotations: the split in dataset order; encodings {docid: (input ids, pieces)} (``encode_documents``);
    evidence_classes {class name: index}.  Every annotation is explained for its gold class.  With ``same_length`` a batch
    only holds documents of one token length (no padding); it defaults to on for ``generate_attn_gradcam``, whose gradient
    weights and min-max normalisation run over the whole [S, S] map, padded query rows included.
    Returns {"docids": [...], "word_ranges", "order" [docs, max(ks)] (-1 past the last word), "counts" [docs, len(ks),
    3 + len(iou_thresholds)], "lines" {k: [...]}, "scores" {k: metrics dict}}, all in dataset order."""
    ks = tuple(int(k) for k in ks)
    docids = [annotation_docid(a) for a in annotations]
    if len(set(docids)) != len(docids):
        raise ValueError("two annotations of the split share a document; the pipeline keys its predictions by docid")
    truth = TruthIndex(annotations)
    ranges = {d: word_piece_ranges(documents[d].split(), encodings[d][1]) for d in set(docids)}
    targets = [evidence_classes[a.classification] for a in annotations]
    if device is None:
        owner = getattr(generator_method, "__self__", None)
        model = getattr(owner, "model", None)
        device = next(model.parameters()).device if model is not None else torch.device("cuda")
    from . import ops
    n, kmax, ncol = len(annotations), max(ks), 3 + len(iou_thresholds)
    order = np.full((n, kmax), -1, dtype=np.int64)
    counts = np.zeros((n, len(ks), ncol), dtype=np.int64)
    if same_length is None:
        name = getattr(getattr(generator_method, "func", generator_method), "__name__", "")
        same_length = name == "generate_attn_gradcam"
    by_len = sorted(range(n), key=lambda i: len(encodings[docids[i]][0]))
    batches = []
    for i in by_len:
        if not batches or len(batches[-1]) == batch_size or \
                (same_length and len(encodings[docids[i]][0]) != len(encodings[docids[batches[-1][0]]][0])):
            batches.append([])
        batches[-1].append(i)
    for idx in batches:
        S = max(len(encodings[docids[i]][0]) for i in idx)
        ids = torch.full((len(idx), S), pad_id, dtype=torch.long)
        mask = torch.zeros((len(idx), S), dtype=torch.long)
        wr, woff, sp, soff = [], [0], [], [0]
        for r, i in enumerate(idx):
            d = docids[i]
            e = encodings[d][0]
            ids[r, :len(e)] = torch.as_tensor(e, dtype=torch.long)
            mask[r, :len(e)] = 1
            wr.extend(ranges[d])
            woff.append(len(wr))
            sp.extend(truth.spans_by_key.get((d, d), []))
            soff.append(len(sp))
        maps = generator_method(input_ids=ids.to(device), attention_mask=mask.to(device),
                                index=torch.as_tensor([targets[i] for i in idx], device=device))
        res = ops.eraser_rationales(maps.reshape(len(idx), S).to(torch.float32).contiguous(), wr, woff, sp, soff, ks,
                                    iou_thresholds)
        host = torch.cat([res["order"].reshape(len(idx), -1), res["counts"].reshape(len(idx), -1)], dim=1).cpu().numpy()
        order[idx] = host[:, :kmax]
        counts[idx] = host[:, kmax:].reshape(len(idx), len(ks), ncol)
    lines = rationale_lines(docids, ks=ks, order=order)
    scores = {k: hard_scores(truth, docids, counts[:, i], order, iou_thresholds) for i, k in enumerate(ks)}
    return {"docids": docids, "word_ranges": [ranges[d] for d in docids], "order": order, "counts": counts,
            "lines": lines, "scores": scores}


def write_results(results, folder):
    """``identifier_results_{k}.json`` (the pipeline's files) and ``scores_{k}.json`` (``metrics.py``'s ``--score_file``
    layout: indent 4, sorted keys) under ``folder``."""
    os.makedirs(folder, exist_ok=True)
    for k, lines in results["lines"].items():
        with open(os.path.join(folder, "identifier_results_%d.json" % k), "w") as f:
            f.write("".join(line + "\n" for line in lines))
        with open(os.path.join(folder, "scores_%d.json" % k), "w") as f:
            json.dump(results["scores"][k], f, indent=4, sort_keys=True)


# ---- command line ---------------------------------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description="ERASER rationale evaluation (token F1 at top-k) of the BERT explanation methods")
    p.add_argument("--data_dir", dest="data_dir", required=True, help="directory with {split}.jsonl and docs/ or docs.jsonl")
    p.add_argument("--output_dir", dest="output_dir", required=True)
    p.add_argument("--model_params", dest="model_params", required=True,
                   help="the pipeline's JSON parameters (bert_vocab, bert_dir, max_length, evidence_classifier.classes)")
    p.add_argument("--method", default="transformer_attribution", choices=METHODS)
    p.add_argument("--split", default="test")
    p.add_argument("--state-dict", dest="state_dict", default=None,
                   help="classifier weights (default: output_dir/classifier/classifier.pt, where the pipeline saves them)")
    p.add_argument("--batch-size", dest="batch_size", type=int, default=8)
    p.add_argument("--iou-thresholds", dest="iou_thresholds", type=float, nargs="+", default=[0.5])
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if not 1 <= len(args.iou_thresholds) <= 8:
        p.error("--iou-thresholds takes 1 to 8 values")
    if args.state_dict is None:
        args.state_dict = os.path.join(args.output_dir, "classifier", "classifier.pt")
    return args


def build_generator(method, bert_dir, num_labels, state_dict=None, device="cuda"):
    """The bound ``Generator`` method of ``method`` on the one façade model it needs (``:422-448``)."""
    import transformers
    from .BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    kind, fn = METHOD_GENERATOR[method]
    if kind == "ours":
        from .BERT_explainability.modules.BERT.BertForSequenceClassification import BertForSequenceClassification
    else:
        from .BERT_explainability.modules.BERT.BERT_cls_lrp import BertForSequenceClassification
    config = transformers.BertConfig.from_pretrained(bert_dir, num_labels=num_labels)
    model = BertForSequenceClassification(config)
    if state_dict:
        model.load_state_dict(torch.load(state_dict, map_location="cpu"), strict=False)
    model = model.to(device).eval()
    return getattr(Generator(model), fn)


def main(argv=None):
    args = parse_args(argv)
    try:
        import transformers
    except ImportError as e:
        raise ImportError("the ERASER command line tokenises with transformers' BertTokenizer; install transformers") from e
    with open(args.model_params) as f:
        params = json.load(f)
    annotations = load_split(args.data_dir, args.split)
    documents = load_documents(args.data_dir, set(annotation_docid(a) for a in annotations))
    tokenizer = transformers.BertTokenizer.from_pretrained(params["bert_vocab"])
    encodings = encode_documents({d: documents[d] for d in set(annotation_docid(a) for a in annotations)}, tokenizer,
                                 params["max_length"])
    classes = params["evidence_classifier"]["classes"]
    evidence_classes = {c: i for i, c in enumerate(classes)}
    gen = build_generator(args.method, params["bert_dir"], len(classes), args.state_dict)
    res = eraser_eval(gen, documents, annotations, encodings, evidence_classes, batch_size=args.batch_size,
                      iou_thresholds=args.iou_thresholds)
    write_results(res, os.path.join(args.output_dir, METHOD_FOLDER[args.method]))
    for k in KS:
        print("top-%d token F1 %.4f (instance macro %.4f)" % (k, res["scores"][k]["token_prf"]["instance_micro"]["f1"],
                                                              res["scores"][k]["token_prf"]["instance_macro"]["f1"]))
    return res


if __name__ == "__main__":
    main()
