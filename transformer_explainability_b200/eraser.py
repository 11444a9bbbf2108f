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
   merge into one key), and every annotation needs an evidence; otherwise ``ValueError``.

With ``faithfulness=True`` (CLI ``--faithfulness``) the same pass also measures ``metrics.py``'s faithfulness
(``score_classifications``, ``:255-364``): per batch one more engine forward gives the original logits, one
``te_eraser_reduce_inputs`` call builds the comprehensiveness (rationale words removed) and sufficiency (only the rationale
words kept) rows of every selection size, the rows run through the engine forward in length-sorted chunks, and
``te_class_probs`` turns each chunk's logits into probabilities on the device.  The selection sizes, the default k and the
row layout are defined in DESIGN.md §1; the result lines go to ``faithfulness_results.jsonl`` and ``metrics.py``'s
``classification_scores`` dict to ``faithfulness_scores.json``.

With ``tokens_to_flip=True`` (CLI ``--tokens-to-flip``, with ``--faithfulness``) each batch also searches, in rounds of
``flip_chunk`` selection sizes, for each document's smallest k whose comprehensiveness row changes the prediction
(``te_eraser_reduce_inputs`` rows, the chunked engine forward, ``te_logit_stats``' argmax): the ``tokens_to_flip`` field of
``faithfulness_results.jsonl`` and ``tokens_to_flip.json``.  With ``soft_scores=True`` (CLI ``--soft-scores``) one
``te_eraser_soft_scores`` call per batch scores the word scores, followed by a 0 per word past truncation, as
``metrics.py``'s soft predictions (``score_soft_tokens``: AUPRC, average precision, ROC AUC): ``soft_results.jsonl`` and
``soft_scores.json``.  Both are defined in DESIGN.md §1.

With ``latex=True`` (CLI ``--latex``) each batch also draws the pipeline's LaTeX heat maps (``generate()``, ``:49-93,
547-561``): one ``te_eraser_latex_weights`` launch turns the gold-class maps, and for the methods of ``LATEX_CF_METHODS``
the maps of one more generator call for the class 1 - target, into ``generate()``'s colour weights, which join the batch's
one device-to-host copy; ``latex_document`` writes the reference's bytes (``{j}_GT_{neg|pos}_{correct}.tex``,
``{j}_CF.tex``).  ``--method ground_truth`` and ``--method generate_all`` write only the pipeline's other two figure
files (``ground_truth_documents``, ``comparison_figures``); ``generate_all`` writes into ``{output_dir}/generate_all/``
rather than the current directory.
"""
import argparse
import functools
import json
import math
import os
import warnings
from dataclasses import dataclass
from types import SimpleNamespace
from typing import FrozenSet, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib, ops
from ._host import to_host

KS = tuple(range(5, 85, 5))
AOPC_THRESHOLDS = (0.01, 0.05, 0.1, 0.2, 0.5)              # metrics.py --aopc_thresholds
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
# one more choice besides the pipeline's METHODS: the LRP-free gradient-weighted attention rollout of the authors'
# follow-up paper (Chefer, Gur, Wolf, ICCV 2021) on the BertForSequenceClassification model.  Padded keys and queries
# contribute exactly nothing to it, so it takes length-sorted padded batches like transformer_attribution.
FOLLOW_UP_FOLDER = {"attn_grad_rollout": "attn_grad_rollout"}
FOLLOW_UP_GENERATOR = {"attn_grad_rollout": ("ours", "generate_attn_grad_rollout")}
CHOICES = METHODS + tuple(FOLLOW_UP_GENERATOR)
FIGURE_MODES = ("ground_truth", "generate_all")         # the pipeline's two figure-only modes (bert_pipeline.py:474-546)


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


# ---- faithfulness: selection sizes and metrics.py's score_classifications --------------------------------------------------
def select_count(fraction, W):
    """The number of words selected at fraction f in (0, 1] of W words: min(W, max(1, floor(f * W + 0.5)))."""
    return min(W, max(1, int(math.floor(fraction * W + 0.5))))


def human_fraction(annotations, docids, word_counts, truth):
    """The default k fraction: the mean over the split's documents of (words < W covered by a truth span) / W."""
    fr = []
    for a, d, W in zip(annotations, docids, word_counts):
        covered = set(t for s, e in truth.spans_by_key.get((a.annotation_id, d), []) for t in range(s, min(e, W)))
        fr.append(len(covered) / W if W else 0.0)
    return sum(fr) / len(fr)


def _log_ratio(x, y):
    """log(x / y) as scipy.special.rel_entr takes it: log1p((x - y) / y) for 0.5 < x / y < 2, else log(x / y)."""
    r = x / y
    return math.log1p((x - y) / y) if 0.5 < r < 2 else math.log(r)


def _entropy(pk, qk=None):
    """scipy.stats.entropy of one distribution (or the KL divergence of pk from qk): both normalised, -x log x (0 at 0)
    or x log(x / y) (0 at x = 0, inf at y = 0 < x) with rel_entr's log, summed with numpy."""
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


def _classification_report(truth, pred, names):
    """sklearn's ``classification_report(truth, pred, output_dict=True, target_names=names)`` for the labels
    0 .. len(names) - 1, each of which occurs in truth; a zero division gives 0 (sklearn's ``zero_division="warn"``)."""
    truth, pred = np.asarray(truth), np.asarray(pred)
    tp = np.array([np.sum((truth == l) & (pred == l)) for l in range(len(names))], dtype=np.int64)
    n_pred = np.array([np.sum(pred == l) for l in range(len(names))], dtype=np.int64)
    n_true = np.array([np.sum(truth == l) for l in range(len(names))], dtype=np.int64)

    def div(a, b):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        return np.where(b == 0, 0.0, a / np.where(b == 0, 1.0, b))
    cols = {"precision": div(tp, n_pred), "recall": div(tp, n_true), "f1-score": div(2.0 * tp, 1.0 * n_true + n_pred)}
    out = {name: dict({k: float(v[i]) for k, v in cols.items()}, support=float(n_true[i])) for i, name in enumerate(names)}
    out["accuracy"] = float(div(tp.sum(), n_pred.sum()))
    out["macro avg"] = dict({k: float(np.average(v)) for k, v in cols.items()}, support=float(np.sum(n_true)))
    out["weighted avg"] = dict({k: float(np.average(v, weights=n_true)) for k, v in cols.items()},
                               support=float(np.sum(n_true)))
    return out


def classification_scores_from_probs(annotations, class_names, pred, probs, comp, suff, thresholds, aopc_thresholds):
    """``metrics.py``'s ``score_classifications`` (``:284-364``) for one result line per annotation, in annotation order:
    pred [N] predicted class indices, probs [N, C] (``classification_scores``), comp / suff [N, 1 + T, C] (the main k,
    then one entry per value of ``thresholds``: ``thresholded_scores``), classes in the order of ``class_names``.  The
    averages and their Python float / numpy arithmetic are the reference's, so the values are its values; ``labels`` is
    rebuilt as the reference builds it (``list(set(...))``, whose order follows the hash seed)."""
    probs = np.asarray(probs, dtype=np.float64)
    comp, suff = np.asarray(comp, dtype=np.float64), np.asarray(suff, dtype=np.float64)
    labels = list(set(a.classification for a in annotations))
    label_to_int = {l: i for i, l in enumerate(labels)}
    truth = [label_to_int[a.classification] for a in annotations]
    predicted = [label_to_int[class_names[int(p)]] for p in pred]
    rows = range(len(annotations))
    beta0 = [float(probs[i, int(pred[i])]) for i in rows]
    cols = [1 + t for t in sorted(range(len(thresholds)), key=lambda t: thresholds[t]) if thresholds[t] in aopc_thresholds]
    if len(cols) != len(aopc_thresholds):
        raise ValueError("every AOPC threshold needs its own thresholded scores")
    out = {"accuracy": float(np.average(np.asarray(truth) == np.asarray(predicted))),
           "prf": _classification_report(truth, predicted, labels)}
    for name, red in (("comprehensiveness", comp), ("sufficiency", suff)):
        out[name] = np.average([beta0[i] - float(red[i, 0, int(pred[i])]) for i in rows])
        out[name + "_entropy"] = np.average([_entropy(probs[i].tolist()) - _entropy(red[i, 0].tolist()) for i in rows])
        out[name + "_kl"] = np.average([_entropy(red[i, 0].tolist(), probs[i].tolist()) for i in rows])
        points = np.array([[beta0[i] - float(red[i, c, int(pred[i])]) for c in cols] for i in rows])
        out[name + "_aopc"] = np.average(points)
        out[name + "_aopc_points"] = np.average(points, axis=0).tolist()
    out["aopc_thresholds"] = list(aopc_thresholds)
    return out


def faithfulness_lines(annotations, docids, class_names, pred, probs, comp, suff, thresholds, selected, tokens_to_flip=None):
    """One ``metrics.py`` result line per annotation (keyed by its own annotation id): the main-k words as
    ``hard_rationale_predictions``, ``classification``, ``classification_scores``, the main-k comprehensiveness and
    sufficiency scores and one ``thresholded_scores`` entry per threshold; with ``tokens_to_flip`` (one int per
    annotation) also that field, last."""
    def scores(p):
        return {c: float(v) for c, v in zip(class_names, p)}
    out = []
    for i, (a, d) in enumerate(zip(annotations, docids)):
        extra = {} if tokens_to_flip is None else {"tokens_to_flip": int(tokens_to_flip[i])}
        out.append(json.dumps(dict({
            "annotation_id": a.annotation_id,
            "rationales": [{"docid": d, "hard_rationale_predictions": [{"start_token": int(w), "end_token": int(w) + 1}
                                                                       for w in selected[i]]}],
            "classification": class_names[int(pred[i])], "classification_scores": scores(probs[i]),
            "comprehensiveness_classification_scores": scores(comp[i][0]),
            "sufficiency_classification_scores": scores(suff[i][0]),
            "thresholded_scores": [{"threshold": float(t), "comprehensiveness_classification_scores": scores(comp[i][1 + j]),
                                    "sufficiency_classification_scores": scores(suff[i][1 + j])}
                                   for j, t in enumerate(thresholds)]}, **extra)))
    return out


def flip_scores(annotations, docids, n_words, tokens, flipped):
    """``tokens_to_flip.json``: the mean fraction of the document's words, as ``metrics.py`` averages it (``:337-346``:
    tokens / document words per annotation, ``np.average``), the number of documents that never flipped and the
    per-document values, in annotation order."""
    frac = [int(t) / int(n) for t, n in zip(tokens, n_words)]
    return {"tokens_to_flip": np.average(frac), "never_flipped": int(len(flipped) - np.count_nonzero(flipped)),
            "documents": [{"annotation_id": a.annotation_id, "docid": d, "tokens_to_flip": int(t), "words": int(n),
                           "fraction": f, "flipped": bool(fl)}
                          for a, d, t, n, f, fl in zip(annotations, docids, tokens, n_words, frac, flipped)]}


# ---- soft-token scores: metrics.py's score_soft_tokens ----------------------------------------------------------------------
def soft_truth(truth, annotation, docid, W, n_words):
    """(the truth spans of (annotation id, docid), (positives, negatives) past the W scored words): the truth side of
    ``PositionScoredDocument.from_results`` for a document of n_words words.  A span past the document raises
    ``ValueError`` (the reference's truth vector has no room for it)."""
    spans = truth.spans_by_key.get((annotation.annotation_id, docid), [])
    if any(e > n_words for _, e in spans):
        raise ValueError("annotation %r: a truth span ends past document %r's %d words"
                         % (annotation.annotation_id, docid, n_words))
    pos = len(set(t for s, e in spans for t in range(max(s, W), e)))
    return spans, (pos, n_words - W - pos)


def soft_token_scores(per_doc, single_class):
    """``score_soft_tokens``' dict (``metrics.py:217-253``) from the per-document (AUPRC, AP, ROC AUC) rows and
    single-class flags, in annotation order: AUPRC averaged over every document, AP and ROC AUC over the documents that
    hold both classes (``_score_aggregator(..., True)``; none: numpy's mean of nothing, NaN)."""
    if len(per_doc) == 0:
        return {"auprc": 0.0, "average_precision": 0.0, "roc_auc_score": 0.0}
    per_doc = np.asarray(per_doc, dtype=np.float64)
    keep = [i for i in range(len(per_doc)) if not single_class[i]]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return {"auprc": np.average(per_doc[:, 0].tolist()), "average_precision": np.average(per_doc[keep, 1].tolist()),
                "roc_auc_score": np.average(per_doc[keep, 2].tolist())}


def soft_lines(annotations, docids, word_scores, n_words):
    """One ``metrics.py`` result line per annotation: ``soft_rationale_predictions`` = the W fp32 word scores, then a 0
    for each word past truncation (one score per document word, as ``PositionScoredDocument.from_results`` asserts)."""
    return [json.dumps({"annotation_id": a.annotation_id, "rationales": [{"docid": d, "soft_rationale_predictions":
                                                                          [float(x) for x in s] + [0.0] * (n - len(s))}]})
            for a, d, s, n in zip(annotations, docids, word_scores, n_words)]


# ---- LaTeX heat maps: bert_pipeline.py's generate() and its ground_truth / generate_all modes -------------------------------
# the methods whose counterfactual (index = 1 - target) map the pipeline also draws (:556-561), plus this port's
# class-dependent attn_grad_rollout
LATEX_CF_METHODS = ("transformer_attribution", "partial_lrp", "attn_gradcam", "lrp", "attn_grad_rollout")
LATEX_ESCAPED = ("\\", "%", "&", "^", "#", "_", "{", "}")          # clean_word's characters, in its order
_TCBSET = r"\tcbset{width=0.9\textwidth,boxrule=0pt,colback=red,arc=0pt,auto outer arc,left=0pt,right=0pt,boxsep=5pt}"
_PARBOX = r"{\setlength{\fboxsep}{0pt}\colorbox{white!0}{\parbox{0.9\textwidth}{"
_CJK_END = r"\end{CJK*}" + "\n" + r"\end{document}"
LATEX_HEADER = "\n".join([r"\documentclass[varwidth=150mm]{standalone}", r"\special{papersize=210mm,297mm}",
                          r"\usepackage{color}", r"\usepackage{tcolorbox}", r"\usepackage{CJK}", r"\usepackage{adjustbox}",
                          _TCBSET, r"\begin{document}", r"\begin{CJK*}{UTF8}{gbsn}", _PARBOX]) + "\n"
LATEX_FOOTER = "\n}}}\n" + _CJK_END


def clean_word(word):
    """One token as ``clean_word`` escapes it: a backslash before each of ``\\ % & ^ # _ { }``, in that order."""
    for c in LATEX_ESCAPED:
        word = word.replace(c, "\\" + c)
    return word


def latex_document(tokens, weights, color="red"):
    """The text of the file ``generate(tokens, cam, ..., color)`` writes (``bert_pipeline.py:49-84``), from the tokens and
    the colour weights (the host copy of ``ops.eraser_latex_weights``, one per token; extra weights are ignored).  Each
    weight is printed as Python prints the float (``%s``); a token is stripped of ``$`` and escaped by ``clean_word``; a
    token holding an escaped ``##`` joins the previous box with the ``\\#\\#`` removed, every other one follows a space."""
    if len(weights) < len(tokens):
        raise ValueError("latex_document: %d weights for %d tokens" % (len(weights), len(tokens)))
    boxes = []
    for t, w in zip(tokens, weights):
        t = clean_word(t.replace("$", ""))
        glued = "\\#\\#" in t
        box = "\\colorbox{%s!%s}{\\strut %s}" % (color, float(w), t.replace("\\#\\#", "") if glued else t)
        boxes.append(box if glued else " " + box)
    return LATEX_HEADER + "".join(boxes) + LATEX_FOOTER


def generate(text_list, attention_list, latex_file, color="red"):
    """``generate()`` (``bert_pipeline.py:49-84``) with its signature: the weights of the first ``len(text_list)`` entries
    of the CUDA tensor ``attention_list`` come from one ``te_eraser_latex_weights`` launch (no clamp: the pipeline
    clamps before it calls), and ``latex_file`` receives ``latex_document``'s text."""
    if not (torch.is_tensor(attention_list) and attention_list.is_cuda):
        raise ValueError("generate: attention_list must be a CUDA tensor (the weights are computed on the GPU)")
    n = len(text_list)
    a = attention_list.reshape(1, -1).to(torch.float32).contiguous()
    if not 1 <= n <= a.shape[1]:
        raise ValueError("generate: %d tokens for %d attention values" % (n, a.shape[1]))
    w = ops.eraser_latex_weights(a, [n], clamp=False)[0, :n].cpu().numpy()
    with open(latex_file, "w", encoding="utf-8") as f:
        f.write(latex_document(text_list, w.tolist(), color))


def input_words(words, pieces):
    """``get_input_words`` (``bert_pipeline.py:140-166``): the words that survive truncation, each as the characters of
    the pieces it covers (``##`` stripped, ``[CLS]`` / ``[SEP]`` / ``[UNK]`` / ``[PAD]`` skipped), so a word cut by the
    truncation keeps only its covered prefix.  Raises ``ValueError`` where the reference's alignment check fails."""
    chars = "".join(p.replace("##", "") for p in pieces if p.replace("##", "") not in SPECIAL_PIECES)
    out, start = [], 0
    for w in words:
        if start >= len(chars):
            break
        out.append(chars[start:start + len(w)])
        start += len(w)
    if out[:-1] != list(words[:len(out) - 1]):
        raise ValueError("word pieces do not align with the document's words")
    return out


def _neg_pos(target):
    return "neg" if target == 0 else "pos"


def ground_truth_documents(annotations, documents, encodings):
    """The ``ground_truth`` mode (``bert_pipeline.py:533-546``): {j: (``visual_results_{j}.tex``, text)} per annotation j
    in dataset order.  The human rationale over ``input_words``: every evidence span of the annotation's first evidence
    group marks its words, up to the first span that starts past the kept words; drawn in green (100 marked, 0 not; a
    document marked everywhere or nowhere is a constant map, all 0)."""
    out = {}
    for j, ann in enumerate(annotations):
        d = annotation_docid(ann)
        words = input_words(documents[d].split(), encodings[d][1])
        cam = [0] * len(words)
        for ev in next(iter(ann.evidences)):
            if ev.start_token >= len(cam):
                break
            for i in range(len(cam))[ev.start_token:ev.end_token]:
                cam[i] = 1
        weights = [0.0] * len(cam) if len(set(cam)) <= 1 else [100.0 * c for c in cam]
        out[j] = ("visual_results_%d.tex" % j, latex_document(words, weights, color="green"))
    return out


# the eleven panels of the comparison page (bert_pipeline.py:476-497): (method folder, GT or CF), three per row
FIGURE_PANELS = (("ground_truth", None), ("ours", "GT"), ("ours", "CF"), ("partial_lrp", "GT"), ("partial_lrp", "CF"),
                 ("attn_gradcam", "GT"), ("attn_gradcam", "CF"), ("lrp", "GT"), ("lrp", "CF"), ("last_attn", "GT"),
                 ("rollout", "GT"))


def comparison_figure(j, target, correct, output_dir):
    """The ``generate_all`` page of annotation j (``bert_pipeline.py:474-528``): (``{j}_{neg|pos}_{correct}.tex``, text),
    a tabular of the eleven PDFs the other modes' files compile to under ``output_dir``."""
    cls, ok = _neg_pos(target), int(correct)
    paths = []
    for folder, kind in FIGURE_PANELS:
        name = ("visual_results_%d" % j if kind is None else "%d_GT_%s_%d" % (j, cls, ok) if kind == "GT"
                else "%d_CF" % j)
        paths.append(os.path.join(output_dir, "%s/%s.pdf" % (folder, name)))
    pad = " " * 8
    cells = [pad + r"\includegraphics[width=0.32\linewidth]{" + p + "}" for p in paths]
    labels = ["(%s)" % chr(ord("a") + i) for i in range(len(paths))]
    rows = []
    for r in range(0, len(paths), 3):                       # the last row holds two panels and an empty third cell
        row, lab = "&\n".join(cells[r:r + 3]), " & ".join(labels[r:r + 3])
        if r + 3 > len(paths):
            row, lab = row + "&", lab + "&"
        rows.append(row + "\\\\\n" + pad + lab + "\\\\\n")
    text = "\n".join([r"\documentclass[varwidth]{standalone}", r"\usepackage{color}", r"\usepackage{tcolorbox}",
                      r"\usepackage{CJK}", _TCBSET, r"\begin{document}", r"\begin{CJK*}{UTF8}{gbsn}", _PARBOX,
                      r"    \setlength{\tabcolsep}{2pt} % Default value: 6pt", r"    \begin{tabular}{ccc}", ""])
    text += "".join(rows) + "    \\end{tabular}\n}}}\n" + _CJK_END + "\n)"
    return "%d_%s_%d.tex" % (j, cls, ok), text


def comparison_figures(annotations, evidence_classes, pred, output_dir):
    """The ``generate_all`` mode: {j: (name, text)} per annotation j in dataset order; ``pred`` [annotations] holds the
    predicted class indices (``predictions``), the correctness flag of each file name is pred == gold class."""
    out = {}
    for j, ann in enumerate(annotations):
        t = evidence_classes[ann.classification]
        out[j] = comparison_figure(j, t, int(pred[j]) == t, output_dir)
    return out


def _batch(idx, docids, encodings, pad_id, device, ranges=None, spans=None):
    """The padded batch of the documents of annotations ``idx`` (length-sorted by the caller): ``ids`` / ``mask``
    int64 [B, S] on ``device``, the token lengths ``lens``, and with ``ranges`` {docid: word ranges} and ``spans``
    {(docid, docid): truth spans} the documents' word ranges and truth spans, flattened with their offsets
    (``ranges[woff[b]:woff[b + 1]]``, ``spans[soff[b]:soff[b + 1]]``)."""
    lens = [len(encodings[docids[i]][0]) for i in idx]
    ids = torch.full((len(idx), max(lens)), pad_id, dtype=torch.long)
    mask = torch.zeros((len(idx), max(lens)), dtype=torch.long)
    wr, woff, sp, soff = [], [0], [], [0]
    for r, i in enumerate(idx):
        ids[r, :lens[r]] = torch.as_tensor(encodings[docids[i]][0], dtype=torch.long)
        mask[r, :lens[r]] = 1
        if ranges is not None:
            wr.extend(ranges[docids[i]])
            woff.append(len(wr))
            sp.extend(spans.get((docids[i], docids[i]), []))
            soff.append(len(sp))
    return SimpleNamespace(idx=idx, docids=[docids[i] for i in idx], ids=ids.to(device), mask=mask.to(device), lens=lens,
                           S=max(lens), ranges=wr, woff=woff, spans=sp, soff=soff)


def predictions(model, annotations, encodings, batch_size=8, pad_id=0):
    """The first-maximum argmax of the engine forward's logits for every annotation's document, in dataset order: one
    forward per length-sorted padded batch, no attribution."""
    eng = model.engine()
    device = next(model.parameters()).device
    docids = [annotation_docid(a) for a in annotations]
    order = sorted(range(len(docids)), key=lambda i: -len(encodings[docids[i]][0]))
    pred = np.zeros(len(docids), dtype=np.int64)
    for s0 in range(0, len(order), batch_size):
        b = _batch(order[s0:s0 + batch_size], docids, encodings, pad_id, device)
        pred[b.idx] = np.argmax(to_host(eng.forward(b.ids, b.mask))[0], axis=1)
    return pred


def write_documents(docs, folder):
    """Write {j: (name, text)} (``ground_truth_documents``, ``comparison_figures``) under ``folder``."""
    os.makedirs(folder, exist_ok=True)
    for name, text in docs.values():
        with open(os.path.join(folder, name), "w", encoding="utf-8") as f:
            f.write(text)


def _sorted_chunks(eng, flat, lens, rows, cap, device):
    """The rows ``rows`` of flat [R, S] (host lengths ``lens[q]``), longest first, through the engine forward in padded
    chunks of at most ``cap`` rows (default: the engine's ``max_chunk`` at the chunk's length): yields (chunk, L, logits)."""
    rows = sorted(rows, key=lambda q: -int(lens[q]))               # longest first: each chunk's first row sets S
    s0 = 0
    while s0 < len(rows):
        L = int(lens[rows[s0]])
        chunk = rows[s0:s0 + (cap or eng.max_chunk(L))]
        sel = torch.as_tensor(chunk, device=device)
        x = flat.index_select(0, sel)[:, :L].contiguous()
        m = (torch.arange(L, device=device)[None, :] <
             torch.as_tensor(lens[chunk], device=device)[:, None]).to(torch.int64)
        yield chunk, L, eng.forward(x, m)
        s0 += len(chunk)


def _flip_search(eng, maps, ids, lens, ranges, woff, orders, pred0, n_words, flip_chunk, cap):
    """Tokens to flip of one batch (DESIGN.md §1): in rounds, every unfinished document b runs the comprehensiveness
    rows of its next ``flip_chunk`` selection sizes (``te_eraser_reduce_inputs``; their lengths follow on the host from
    the full word order ``orders[b]``), in length-sorted chunks, and ``te_logit_stats`` gives their argmax; one copy of
    the round's predictions finds each document's first flip.  Returns (tokens [B], flipped [B], rows, real tokens,
    padded tokens)."""
    B, device = len(lens), maps.device
    W = np.diff(np.asarray(woff))
    comp_len = []                                                  # comp_len[b][k - 1]: the row length at selection k
    for b in range(B):
        seen, cl = set(), []
        for w in orders[b][:W[b]]:
            a, e = ranges[woff[b] + int(w)]
            seen.update(range(a, e + 1))
            cl.append(lens[b] - len(seen))
        comp_len.append(cl)
    nxt = [1] * B
    tokens = [None if W[b] else n_words[b] for b in range(B)]
    flipped = [False] * B
    n_rows = real = padded = 0
    while any(t is None for t in tokens):
        live = [b for b in range(B) if tokens[b] is None]
        J = min(flip_chunk, max(W[b] - nxt[b] + 1 for b in live))
        nsel = np.zeros((B, J), dtype=np.int64)
        rows, rlen = [], np.zeros(B * J * 2, dtype=np.int64)
        for b in live:
            for j, k in enumerate(range(nxt[b], min(nxt[b] + J, W[b] + 1))):
                nsel[b, j] = k
                rows.append((b * J + j) * 2)
                rlen[rows[-1]] = comp_len[b][k - 1]
        red = ops.eraser_reduce_inputs(maps, ids, lens, ranges, woff, nsel)
        flat = red["ids"].reshape(B * J * 2, -1)
        preds, order = [], []
        for chunk, L, logits in _sorted_chunks(eng, flat, rlen, rows, cap, device):
            preds.append(ops.logit_stats(logits, torch.zeros(len(chunk), dtype=torch.int32, device=device))[0])
            order += chunk
            real += int(rlen[chunk].sum())
            padded += len(chunk) * L
        n_rows += len(rows)
        ph = dict(zip(order, np.concatenate(to_host(*preds))))           # row -> its prediction
        for b in live:
            ks = range(nxt[b], min(nxt[b] + J, W[b] + 1))
            hit = next((k for j, k in enumerate(ks) if ph[(b * J + j) * 2] != pred0[b]), None)
            if hit is not None:
                tokens[b], flipped[b] = hit, True
            else:
                nxt[b] += len(ks)
                if nxt[b] > W[b]:
                    tokens[b] = n_words[b]
    return tokens, flipped, n_rows, real, padded


LATEX_CF_GENERATORS = tuple({**METHOD_GENERATOR, **FOLLOW_UP_GENERATOR}[m][1] for m in LATEX_CF_METHODS)


def latex_logits(eng, input_ids, attention_mask):
    """A copy of the logits [B, C] of the engine's last forward when it ran on this whole batch (the generator's own
    forward: no extra pass); otherwise (the generator chunked the batch) one forward of the batch."""
    if tuple(eng.last) == tuple(input_ids.shape):
        return eng.tensor("logits").to(torch.float32).clone()
    return eng.forward(input_ids, attention_mask)


def _generator_model(generator_method):
    f = generator_method
    while isinstance(f, functools.partial):
        f = f.func
    model = getattr(getattr(f, "__self__", None), "model", None)
    if model is None or not hasattr(model, "engine"):
        raise ValueError("faithfulness needs a Generator method bound to a façade BERT model (its engine runs the "
                         "forwards of the reduced inputs)")
    return model


def _check_fraction(f, what):
    if not (isinstance(f, float) and 0.0 < f <= 1.0):
        raise ValueError("%s must lie in (0, 1], got %r" % (what, f))


# ---- the evaluation ---------------------------------------------------------------------------------------------------------
# One unit per optional evaluation: the constructor sets it up and checks its arguments; per batch ``device(b, res)`` (b:
# ``_batch`` with its gold-class maps and targets, res: ``eraser_rationales``' tensors) returns named tensors for the
# batch's one ``to_host`` copy, and ``host(b, h)`` reads their host arrays; ``result()`` is its entry of the result.
class _Latex:
    """The pipeline's LaTeX heat maps: the weights of the gold-class maps and, for ``LATEX_CF_GENERATORS``, of one more
    generator call for the class 1 - target, with the logits of the batch's engine forward."""
    def __init__(self, generator_method, gen_name, encodings, evidence_classes):
        if len(evidence_classes) != 2:
            raise ValueError("latex needs exactly two classes: the counterfactual class is 1 - target")
        self.eng = _generator_model(generator_method).engine()
        self.generator_method, self.cf = generator_method, gen_name in LATEX_CF_GENERATORS
        self.encodings, self.docs = encodings, {}

    def device(self, b, res):
        out = {"latex_logits": latex_logits(self.eng, b.ids, b.mask), "latex_gt": ops.eraser_latex_weights(b.maps, b.lens)}
        if self.cf:
            cf = self.generator_method(input_ids=b.ids, attention_mask=b.mask,
                                       index=torch.as_tensor([1 - t for t in b.targets], device=b.ids.device))
            out["latex_cf"] = ops.eraser_latex_weights(cf.reshape(len(b.idx), b.S).to(torch.float32).contiguous(), b.lens)
        return out

    def host(self, b, h):
        for r, (i, d) in enumerate(zip(b.idx, b.docids)):
            t, L, pieces = b.targets[r], b.lens[r], self.encodings[d][1]
            correct = int(np.argmax(h["latex_logits"][r])) == t
            doc = {"GT": ("%d_GT_%s_%d.tex" % (i, _neg_pos(t), correct), latex_document(pieces, h["latex_gt"][r, :L]))}
            if self.cf:
                doc["CF"] = ("%d_CF.tex" % i, latex_document(pieces, h["latex_cf"][r, :L]))
            self.docs[i] = doc

    def result(self):
        return dict(sorted(self.docs.items()))


class _Soft:
    """``metrics.py``'s soft-token scores of the word scores (one ``te_eraser_soft_scores`` call per batch)."""
    def __init__(self, truth, annotations, docids, ranges, n_words):
        self.annotations, self.docids, self.n_words = annotations, docids, n_words
        self.truths = [soft_truth(truth, a, d, len(ranges[d]), nw) for a, d, nw in zip(annotations, docids, n_words)]
        self.per_doc, self.single = np.zeros((len(docids), 3), dtype=np.float64), np.zeros(len(docids), dtype=bool)
        self.words = [None] * len(docids)

    def device(self, b, res):
        sp, soff = [], [0]
        for i in b.idx:
            sp.extend(self.truths[i][0])
            soff.append(len(sp))
        soft = ops.eraser_soft_scores(res["word_scores"], b.woff, sp, soff, [self.truths[i][1] for i in b.idx])
        return {"soft_scores": soft["scores"], "soft_flags": soft["flags"], "word_scores": res["word_scores"]}

    def host(self, b, h):
        self.per_doc[b.idx] = h["soft_scores"]
        self.single[b.idx] = h["soft_flags"][:, 0] != 0
        bad = [d for d, nan in zip(b.docids, h["soft_flags"][:, 1]) if nan]
        if bad:
            raise ValueError("document %r has a NaN word score; metrics.py's soft-token scores (sklearn) reject NaN"
                             % bad[0])
        for r, i in enumerate(b.idx):
            self.words[i] = h["word_scores"][b.woff[r]:b.woff[r + 1]]

    def result(self):
        return {"per_document": self.per_doc, "single_class": self.single,
                "lines": soft_lines(self.annotations, self.docids, self.words, self.n_words),
                "scores": soft_token_scores(self.per_doc, self.single)}


class _Faithfulness:
    """``metrics.py``'s faithfulness and, with ``tokens_to_flip``, the tokens-to-flip search.  The probabilities of the
    reduced rows collect in one device buffer, which comes back at the end; ``kfull``: the largest k of the word orders."""
    def __init__(self, generator_method, annotations, docids, ranges, truth, n_words, evidence_classes, aopc_thresholds,
                 k_fraction, faith_chunk, tokens_to_flip, flip_chunk, kmax, device):
        fracs = [float(f) for f in aopc_thresholds]
        for f in fracs:
            _check_fraction(f, "an AOPC threshold")
        if not fracs:
            raise ValueError("faithfulness needs at least one AOPC threshold")
        if k_fraction is None:
            k_fraction = human_fraction(annotations, docids, [len(ranges[d]) for d in docids], truth)
        _check_fraction(float(k_fraction), "k_fraction")
        self.fracs = [float(k_fraction)] + fracs
        n, J = len(docids), len(self.fracs)
        self.nsel = np.array([[select_count(f, len(ranges[d])) for f in self.fracs] for d in docids],
                             dtype=np.int64).reshape(n, J)
        self.eng = _generator_model(generator_method).engine()
        self.names = [c for c, _ in sorted(evidence_classes.items(), key=lambda kv: kv[1])]
        C = self.eng.cfg.num_labels
        self.buf = torch.empty(n * 2 * J, C, dtype=torch.float32, device=device)
        self.logits, self.probs = np.zeros((n, C), dtype=np.float32), np.zeros((n, C), dtype=np.float32)
        self.red_slot, self.slot, self.real_tok, self.padded_tok = np.zeros((n, J, 2), dtype=np.int64), 0, 0, 0
        self.selected = [None] * n
        self.kfull = max(kmax, int(self.nsel[:, 0].max()) if n else 0)
        self.flip = tokens_to_flip
        if tokens_to_flip:                                          # the search needs every document's full order
            if C < 2:
                raise ValueError("tokens_to_flip needs at least two classes")
            self.kfull = max([self.kfull] + [len(ranges[d]) for d in docids])
            self.flip_tok, self.flipped, self.flip_stats = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=bool), [0, 0, 0]
        self.annotations, self.docids, self.n_words = annotations, docids, n_words
        self.faith_chunk, self.flip_chunk = faith_chunk, int(flip_chunk)

    def device(self, b, res):
        logits = self.eng.forward(b.ids, b.mask)
        out = {"logits": logits, "probs": ops.class_probs(logits)}
        self.red = ops.eraser_reduce_inputs(b.maps, b.ids, b.lens, b.ranges, b.woff, self.nsel[b.idx])
        out["red_lengths"] = self.red["lengths"]
        if self.flip:                                               # te_logit_stats' pred: the first maximum
            out["pred0"] = ops.logit_stats(logits, torch.zeros(len(b.idx), dtype=torch.int32, device=logits.device))[0]
        return out

    def host(self, b, h):
        J = len(self.fracs)
        self.logits[b.idx], self.probs[b.idx] = h["logits"], h["probs"]
        for r, i in enumerate(b.idx):
            self.selected[i] = h["order"][r, :self.nsel[i, 0]].tolist()
        lens = h["red_lengths"].reshape(-1)                         # [B * J * 2], rows (document, selection, kind)
        flat = self.red["ids"].reshape(len(lens), b.S)
        for chunk, L, logits in _sorted_chunks(self.eng, flat, lens, range(len(lens)), self.faith_chunk, b.ids.device):
            ops.class_probs(logits, out=self.buf[self.slot:self.slot + len(chunk)])
            for q_i, q in enumerate(chunk):
                r, rest = divmod(q, 2 * J)
                self.red_slot[b.idx[r], rest // 2, rest % 2] = self.slot + q_i
            self.slot += len(chunk)
            self.real_tok += int(lens[chunk].sum())
            self.padded_tok += len(chunk) * L
        if self.flip:                                               # the batch's maps stay on the device until it ends
            t, fl, *st = _flip_search(self.eng, b.maps, b.ids, b.lens, b.ranges, b.woff, h["order"], h["pred0"],
                                      [self.n_words[i] for i in b.idx], self.flip_chunk, self.faith_chunk)
            self.flip_tok[b.idx], self.flipped[b.idx] = t, fl
            self.flip_stats = [a + c for a, c in zip(self.flip_stats, st)]

    def result(self):
        allp, = to_host(self.buf)
        anns, docids, logits, probs = self.annotations, self.docids, self.logits, self.probs
        pred = np.argmax(logits, axis=1)                                # the first maximum
        comp, suff = allp[self.red_slot[:, :, 0]], allp[self.red_slot[:, :, 1]]
        thr = self.fracs[1:]
        out = {"fractions": self.fracs, "n_select": self.nsel, "pred": pred, "logits": logits, "probs": probs,
               "comp": comp, "suff": suff,
               "lines": faithfulness_lines(anns, docids, self.names, pred, probs, comp, suff, thr, self.selected,
                                           self.flip_tok if self.flip else None),
               "scores": classification_scores_from_probs(anns, self.names, pred, probs, comp, suff, thr, thr),
               "real_tokens": self.real_tok, "padded_tokens": self.padded_tok}
        if self.flip:
            out.update({"tokens_to_flip": self.flip_tok, "flipped": self.flipped,
                        "flip_scores": flip_scores(anns, docids, self.n_words, self.flip_tok, self.flipped),
                        "flip_rows": self.flip_stats[0], "flip_real_tokens": self.flip_stats[1],
                        "flip_padded_tokens": self.flip_stats[2]})
        return out


def eraser_eval(generator_method, documents, annotations, encodings, evidence_classes, batch_size=8, ks=KS,
                iou_thresholds=(0.5,), pad_id=0, device=None, same_length=None, faithfulness=False,
                aopc_thresholds=AOPC_THRESHOLDS, k_fraction=None, faith_chunk=None, soft_scores=False,
                tokens_to_flip=False, flip_chunk=16, latex=False):
    """The test loop of the pipeline (``bert_pipeline.py:456-582``) and ``metrics.py``'s hard scores on the engine.

    generator_method: a bound ``Generator`` method (``generate_LRP`` keeps its ``start_layer = 11``), called as
    ``generator_method(input_ids=, attention_mask=, index=)`` for a padded batch; documents {docid: text};
    annotations: the split in dataset order; encodings {docid: (input ids, pieces)} (``encode_documents``);
    evidence_classes {class name: index}.  Every annotation is explained for its gold class.  With ``same_length`` a batch
    only holds documents of one token length (no padding); it defaults to on for ``generate_attn_gradcam``, whose gradient
    weights and min-max normalisation run over the whole [S, S] map, padded query rows included.
    Returns {"docids": [...], "word_ranges", "order" [docs, max(ks)] (-1 past the last word), "counts" [docs, len(ks),
    3 + len(iou_thresholds)], "lines" {k: [...]}, "scores" {k: metrics dict}}, all in dataset order.

    With ``faithfulness`` (the generator must be bound to a façade model, whose engine runs the forwards) the same maps
    also give ``metrics.py``'s faithfulness at the fractions (k_fraction, *aopc_thresholds) of each document's words
    (``k_fraction`` defaults to ``human_fraction``); the reduced rows run in length-sorted chunks of at most
    ``faith_chunk`` rows (default: the engine's ``max_chunk`` at the chunk's length).  The other keys are unchanged, and
    a key "faithfulness" holds {"fractions", "n_select" [docs, 1 + T], "pred" [docs], "logits" [docs, C], "probs"
    [docs, C], "comp" / "suff" [docs, 1 + T, C] (fp32 probabilities), "lines", "scores", "real_tokens",
    "padded_tokens"}.

    With ``soft_scores`` the same word scores also give ``metrics.py``'s soft-token scores (one ``te_eraser_soft_scores``
    call per batch), in a key "soft": {"per_document" [docs, 3] (AUPRC, AP, ROC AUC), "single_class" [docs], "lines",
    "scores"}; a NaN word score raises ``ValueError``.  With ``tokens_to_flip`` (needs ``faithfulness``) each batch's
    maps also drive the tokens-to-flip search (DESIGN.md §1) in rounds of ``flip_chunk`` selection sizes per document;
    "faithfulness" gains "tokens_to_flip" [docs], "flipped" [docs], "flip_scores" (``tokens_to_flip.json``),
    "flip_rows", "flip_real_tokens" and "flip_padded_tokens", and its lines the ``tokens_to_flip`` field.

    With ``latex`` (two classes only; the generator must be bound to a façade model) each batch also draws the
    pipeline's LaTeX heat maps (``bert_pipeline.py:547-561``): the gold-class maps above and, for the generators of
    ``LATEX_CF_METHODS`` (``generate_LRP``, ``generate_LRP_last_layer``, ``generate_attn_gradcam``, ``generate_full_lrp``,
    ``generate_attn_grad_rollout``), one more call for the counterfactual class 1 - target go through one
    ``te_eraser_latex_weights`` launch each, and the weights join the batch's one device-to-host copy with the logits of
    the batch's engine forward (the correctness flag: first argmax == target).  A key "latex" holds {j: {"GT": (name,
    text), "CF": (name, text)}} per annotation j in dataset order (``CF`` only for those methods); ``generate_LRP``'s
    batches then hold one token length (its ``[CLS]`` entry, the row minimum, would see the padding)."""
    ks = tuple(int(k) for k in ks)
    gen_name = getattr(getattr(generator_method, "func", generator_method), "__name__", "")
    lat = _Latex(generator_method, gen_name, encodings, evidence_classes) if latex else None
    if tokens_to_flip and not faithfulness:
        raise ValueError("tokens_to_flip needs faithfulness (metrics.py reads it with the classification fields)")
    if tokens_to_flip and not 1 <= int(flip_chunk) <= _lib.ERASER_MAX_SELECTIONS:
        raise ValueError("flip_chunk must lie in 1..%d" % _lib.ERASER_MAX_SELECTIONS)
    docids = [annotation_docid(a) for a in annotations]
    if len(set(docids)) != len(docids):
        raise ValueError("two annotations of the split share a document; the pipeline keys its predictions by docid")
    n_words = [len(documents[d].split()) for d in docids]
    truth = TruthIndex(annotations)
    ranges = {d: word_piece_ranges(documents[d].split(), encodings[d][1]) for d in set(docids)}
    targets = [evidence_classes[a.classification] for a in annotations]
    if device is None:
        owner = getattr(generator_method, "__self__", None)
        model = getattr(owner, "model", None)
        device = next(model.parameters()).device if model is not None else torch.device("cuda")
    n, kmax = len(annotations), max(ks)
    order = np.full((n, kmax), -1, dtype=np.int64)
    counts = np.zeros((n, len(ks), 3 + len(iou_thresholds)), dtype=np.int64)
    if same_length is None:
        same_length = gen_name == "generate_attn_gradcam" or (latex and gen_name == "generate_LRP")
    faith = _Faithfulness(generator_method, annotations, docids, ranges, truth, n_words, evidence_classes,
                          aopc_thresholds, k_fraction, faith_chunk, tokens_to_flip, flip_chunk, kmax,
                          device) if faithfulness else None
    soft = _Soft(truth, annotations, docids, ranges, n_words) if soft_scores else None
    units = [u for u in (lat, soft, faith) if u is not None]            # the order of their device work
    ks_run = ks + ((faith.kfull,) if faith is not None and faith.kfull > kmax else ())
    by_len = sorted(range(n), key=lambda i: len(encodings[docids[i]][0]))
    batches = []
    for i in by_len:
        if not batches or len(batches[-1]) == batch_size or \
                (same_length and len(encodings[docids[i]][0]) != len(encodings[docids[batches[-1][0]]][0])):
            batches.append([])
        batches[-1].append(i)
    for idx in batches:
        b = _batch(idx, docids, encodings, pad_id, device, ranges, truth.spans_by_key)
        b.targets = [targets[i] for i in idx]
        maps = generator_method(input_ids=b.ids, attention_mask=b.mask, index=torch.as_tensor(b.targets, device=device))
        b.maps = maps.reshape(len(idx), b.S).to(torch.float32).contiguous()
        res = ops.eraser_rationales(b.maps, b.ranges, b.woff, b.spans, b.soff, ks_run, iou_thresholds)
        named = {"order": res["order"], "counts": res["counts"]}
        for u in units:
            named.update(u.device(b, res))
        h = dict(zip(named, to_host(*named.values())))
        order[idx] = h["order"][:, :kmax]
        counts[idx] = h["counts"][:, :len(ks)]
        for u in units:
            u.host(b, h)
    lines = rationale_lines(docids, ks=ks, order=order)
    scores = {k: hard_scores(truth, docids, counts[:, i], order, iou_thresholds) for i, k in enumerate(ks)}
    out = {"docids": docids, "word_ranges": [ranges[d] for d in docids], "order": order, "counts": counts,
           "lines": lines, "scores": scores}
    for key, u in (("faithfulness", faith), ("latex", lat), ("soft", soft)):
        if u is not None:
            out[key] = u.result()
    return out


def write_results(results, folder):
    """``identifier_results_{k}.json`` (the pipeline's files) and ``scores_{k}.json`` (``metrics.py``'s ``--score_file``
    layout: indent 4, sorted keys) under ``folder``; with faithfulness results also ``faithfulness_results.jsonl``
    (``metrics.py``'s results format) and ``faithfulness_scores.json`` (its ``classification_scores`` dict), with
    tokens to flip also ``tokens_to_flip.json``; with soft scores ``soft_results.jsonl`` and ``soft_scores.json``
    (``score_soft_tokens``' dict)."""
    os.makedirs(folder, exist_ok=True)
    for k, lines in results["lines"].items():
        with open(os.path.join(folder, "identifier_results_%d.json" % k), "w") as f:
            f.write("".join(line + "\n" for line in lines))
        with open(os.path.join(folder, "scores_%d.json" % k), "w") as f:
            json.dump(results["scores"][k], f, indent=4, sort_keys=True)
    if "faithfulness" in results:
        with open(os.path.join(folder, "faithfulness_results.jsonl"), "w") as f:
            f.write("".join(line + "\n" for line in results["faithfulness"]["lines"]))
        with open(os.path.join(folder, "faithfulness_scores.json"), "w") as f:
            json.dump(results["faithfulness"]["scores"], f, indent=4, sort_keys=True)
        if "flip_scores" in results["faithfulness"]:
            with open(os.path.join(folder, "tokens_to_flip.json"), "w") as f:
                json.dump(results["faithfulness"]["flip_scores"], f, indent=4, sort_keys=True)
    if "soft" in results:
        with open(os.path.join(folder, "soft_results.jsonl"), "w") as f:
            f.write("".join(line + "\n" for line in results["soft"]["lines"]))
        with open(os.path.join(folder, "soft_scores.json"), "w") as f:
            json.dump(results["soft"]["scores"], f, indent=4, sort_keys=True)
    if "latex" in results:
        write_documents({(j, k): v for j, doc in results["latex"].items() for k, v in doc.items()}, folder)


# ---- command line ---------------------------------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description="ERASER rationale evaluation (token F1 at top-k) of the BERT explanation methods")
    p.add_argument("--data_dir", dest="data_dir", required=True, help="directory with {split}.jsonl and docs/ or docs.jsonl")
    p.add_argument("--output_dir", dest="output_dir", required=True)
    p.add_argument("--model_params", dest="model_params", required=True,
                   help="the pipeline's JSON parameters (bert_vocab, bert_dir, max_length, evidence_classifier.classes)")
    p.add_argument("--method", default="transformer_attribution", choices=CHOICES + FIGURE_MODES,
                   help="an explanation method, or one of the pipeline's figure modes: ground_truth (the human "
                        "rationales as LaTeX heat maps) and generate_all (the comparison page of every method's maps)")
    p.add_argument("--split", default="test")
    p.add_argument("--state-dict", dest="state_dict", default=None,
                   help="classifier weights (default: output_dir/classifier/classifier.pt, where the pipeline saves them)")
    p.add_argument("--batch-size", dest="batch_size", type=int, default=8)
    p.add_argument("--iou-thresholds", dest="iou_thresholds", type=float, nargs="+", default=[0.5])
    p.add_argument("--faithfulness", action="store_true",
                   help="also measure comprehensiveness, sufficiency and their AOPC (metrics.py score_classifications)")
    p.add_argument("--aopc-thresholds", dest="aopc_thresholds", type=float, nargs="+", default=list(AOPC_THRESHOLDS),
                   help="fractions of each document's words for the AOPC bins (metrics.py --aopc_thresholds)")
    p.add_argument("--k-fraction", dest="k_fraction", type=float, default=None,
                   help="fraction of words removed / kept for the main comprehensiveness and sufficiency (default: the "
                        "split's mean fraction of words inside a human rationale)")
    p.add_argument("--soft-scores", dest="soft_scores", action="store_true",
                   help="also score the word scores as soft predictions (metrics.py score_soft_tokens: AUPRC, AP, ROC AUC)")
    p.add_argument("--tokens-to-flip", dest="tokens_to_flip", action="store_true",
                   help="also find each document's tokens to flip: the fewest best-ranked words whose removal changes "
                        "the prediction (needs --faithfulness)")
    p.add_argument("--latex", action="store_true",
                   help="also write the pipeline's LaTeX heat maps: {j}_GT_{neg|pos}_{correct}.tex for the gold class and, "
                        "for %s, {j}_CF.tex for the other class (two classes only)" % ", ".join(LATEX_CF_METHODS))
    return p


def parse_args(argv=None):
    p = build_parser()
    args = p.parse_args(argv)
    if args.batch_size < 1:
        p.error("--batch-size must be at least 1")
    if not 1 <= len(args.iou_thresholds) <= 8:
        p.error("--iou-thresholds takes 1 to 8 values")
    if not 1 <= len(args.aopc_thresholds) < _lib.ERASER_MAX_SELECTIONS:
        p.error("--aopc-thresholds takes 1 to %d values" % (_lib.ERASER_MAX_SELECTIONS - 1))
    if any(not 0.0 < f <= 1.0 for f in args.aopc_thresholds) or len(set(args.aopc_thresholds)) != len(args.aopc_thresholds):
        p.error("--aopc-thresholds takes distinct fractions in (0, 1]")
    if args.k_fraction is not None and not 0.0 < args.k_fraction <= 1.0:
        p.error("--k-fraction must lie in (0, 1]")
    if args.tokens_to_flip and not args.faithfulness:
        p.error("--tokens-to-flip needs --faithfulness")
    if args.method in FIGURE_MODES and (args.latex or args.faithfulness or args.soft_scores):
        p.error("--method %s writes only its .tex files" % args.method)
    if args.state_dict is None:
        args.state_dict = os.path.join(args.output_dir, "classifier", "classifier.pt")
    return args


def build_generator(method, bert_dir, num_labels, state_dict=None, device="cuda"):
    """The bound ``Generator`` method of ``method`` on the one façade model it needs (``:422-448``)."""
    import transformers
    from .BERT_explainability.modules.BERT.ExplanationGenerator import Generator
    kind, fn = {**METHOD_GENERATOR, **FOLLOW_UP_GENERATOR}[method]
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
    if args.method == "ground_truth":
        docs = ground_truth_documents(annotations, documents, encodings)
        write_documents(docs, os.path.join(args.output_dir, "ground_truth"))
        return docs
    if args.method == "generate_all":                     # the classifier of transformer_attribution predicts (:467)
        model = _generator_model(build_generator("transformer_attribution", params["bert_dir"], len(classes),
                                                 args.state_dict))
        pred = predictions(model, annotations, encodings, batch_size=args.batch_size)
        docs = comparison_figures(annotations, evidence_classes, pred, args.output_dir)
        write_documents(docs, os.path.join(args.output_dir, "generate_all"))
        return docs
    gen = build_generator(args.method, params["bert_dir"], len(classes), args.state_dict)
    res = eraser_eval(gen, documents, annotations, encodings, evidence_classes, batch_size=args.batch_size,
                      iou_thresholds=args.iou_thresholds, faithfulness=args.faithfulness,
                      aopc_thresholds=args.aopc_thresholds, k_fraction=args.k_fraction, soft_scores=args.soft_scores,
                      tokens_to_flip=args.tokens_to_flip, latex=args.latex)
    write_results(res, os.path.join(args.output_dir, {**METHOD_FOLDER, **FOLLOW_UP_FOLDER}[args.method]))
    for k in KS:
        print("top-%d token F1 %.4f (instance macro %.4f)" % (k, res["scores"][k]["token_prf"]["instance_micro"]["f1"],
                                                              res["scores"][k]["token_prf"]["instance_macro"]["f1"]))
    if args.faithfulness:
        f = res["faithfulness"]["scores"]
        print("k fraction %.4f: comprehensiveness %.4f, sufficiency %.4f" % (res["faithfulness"]["fractions"][0],
                                                                            f["comprehensiveness"], f["sufficiency"]))
        print("AOPC over %s: comprehensiveness %.4f, sufficiency %.4f" % (f["aopc_thresholds"], f["comprehensiveness_aopc"],
                                                                         f["sufficiency_aopc"]))
    if args.tokens_to_flip:
        t = res["faithfulness"]["flip_scores"]
        print("tokens to flip: mean fraction %.4f, %d of %d documents never flipped" % (
            t["tokens_to_flip"], t["never_flipped"], len(t["documents"])))
    if args.soft_scores:
        s = res["soft"]["scores"]
        print("soft tokens: AUPRC %.4f, AP %.4f, ROC AUC %.4f" % (s["auprc"], s["average_precision"], s["roc_auc_score"]))
    return res


if __name__ == "__main__":
    main()
